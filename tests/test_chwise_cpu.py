"""CPU tests of the channel-wise convolution: the float64 restatement (tests/chwise_oracle.py) over
the oracle's kernel map matches the compiled reference's fixtures (tests/golden/ref_chwise_*), the
layer has the reference's parameters, and the ops refuse CPU tensors."""
import numpy as np
import pytest
import torch

import chwise_oracle as CO
from helpers import golden, rel_err, state_digest
from oracle import oracle_np as O
from test_gpu_chwise import CASES, CONVNEXT_CLASSES, CONVNEXT_SEED


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(name):
    spec = CASES[name]
    G = golden(f"ref_chwise_{name}.npz")
    D = spec["D"]
    region = O.HYPER_CROSS if spec.get("region") == "HYPER_CROSS" else O.HYPER_CUBE
    out_coords, _ = O.stride_map_coords(G["in_coords"], [1] * D, [spec["s"]] * D)
    assert (out_coords == G["out_coords"]).all()
    offs = O.region_offsets(region, [spec["k"]] * D, [spec["d"]] * D, [1] * D)
    assert len(offs) == len(G["kernel"])
    im, om = O.kernel_map(G["in_coords"], out_coords, offs)
    bias = G["bias"] if spec["bias"] else None
    y = CO.forward(G["in_feats"], G["kernel"], im, om, len(out_coords), bias)
    assert rel_err(y, G["out_feats"]) < 1e-5
    gi, gk = CO.backward(G["in_feats"], G["grad_out"], G["kernel"], im, om)
    assert rel_err(gi, G["grad_in"]) < 1e-5
    assert rel_err(gk, G["grad_kernel"]) < 1e-5


def test_oracle_tables_and_empty_rows():
    # two offsets, three input rows, four output rows: output row 3 and offset 1's row 0 are empty
    im, om = [np.array([0, 2]), np.array([1])], [np.array([0, 1]), np.array([2])]
    out_nbr, in_nbr = CO.tables(im, om, 3, 4)
    assert out_nbr.tolist() == [[0, 2, -1, -1], [-1, -1, 1, -1]]
    assert in_nbr.tolist() == [[0, -1, 1], [-1, 2, -1]]
    x = np.array([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    W = np.array([[1.0, -1.0], [2.0, 0.5]])
    y, A = CO.gather(x, W, out_nbr)
    assert y.tolist() == [[1, -2], [5, -6], [6, 2], [0, 0]]
    assert A.tolist() == [[1, 2], [5, 6], [6, 2], [0, 0]]
    dW, _ = CO.wgrad(x, np.ones((4, 2)), out_nbr)
    assert dW.tolist() == [[6, 8], [3, 4]]


def test_layer_parameters_match_reference():
    import minkowskiengine_b200 as ME
    layer = ME.MinkowskiChannelwiseConvolution(16, kernel_size=7, stride=2, bias=True, dimension=3)
    assert tuple(layer.kernel.shape) == (343, 16) and layer.kernel.dtype == torch.float32
    assert tuple(layer.bias.shape) == (1, 16)
    assert list(layer.state_dict()) == ["kernel", "bias"]
    assert float(layer.kernel.detach().abs().max()) <= 1 / (16 * 343) ** 0.5
    assert repr(layer) == ("MinkowskiChannelwiseConvolution(in=16, region_type=RegionType.HYPER_CUBE, "
                           "kernel_size=[7, 7, 7], stride=[2, 2, 2], dilation=[1, 1, 1])")
    kg = ME.KernelGenerator(kernel_size=3, region_type=ME.RegionType.HYPER_CROSS, dimension=4)
    assert tuple(ME.MinkowskiChannelwiseConvolution(5, kernel_generator=kg, dimension=4)
                 .kernel.shape) == (9, 5)


def test_convnext_initial_weights_match_reference():
    import minkowskiengine_b200 as ME
    from examples.convnext import convnext
    torch.manual_seed(CONVNEXT_SEED)
    net = convnext(ME, 3, CONVNEXT_CLASSES, 3)
    assert (state_digest(net) == golden("ref_chwise_convnext.npz")["init_digest"]).all()
    assert sum(isinstance(m, ME.MinkowskiChannelwiseConvolution) for m in net.modules()) == 2


def test_ops_reject_cpu_tensors():
    import minkowskiengine_b200 as ME
    from minkowskiengine_b200 import backend as _C
    mgr = _C.CoordinateMapManagerGPU_c10()
    key = ME.CoordinateMapKey([1, 1, 1], "")
    args = ([3] * 3, [1] * 3, [1] * 3, ME.RegionType.HYPER_CUBE, None)
    with pytest.raises(RuntimeError):
        _C.ChannelwiseConvolutionForwardGPU(torch.rand(4, 3), torch.rand(27, 3), *args, key,
                                            ME.CoordinateMapKey(4), mgr)
    with pytest.raises(RuntimeError):
        _C.ChannelwiseConvolutionBackwardGPU(torch.rand(4, 3), torch.rand(4, 3), torch.rand(27, 3),
                                             *args, key, key, mgr)
