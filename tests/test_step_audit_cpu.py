"""The step audit's own pieces without a GPU (tests/step_audit.py): its kernel-map restatement
against oracle_np pair for pair, and the recording handle against the package."""
import numpy as np
import pytest
import torch

from examples.minkunet import minkunet
from helpers import state_digest, unique_cloud
from oracle import oracle_np as O
from step_audit import (RecordingHandle, StepAudit, conv_pairs, offsets_of, strided_coords,
                        wgrad_share_steps)


def _cloud(ts, seed):
    """Unique rows over 3 batches with negative coordinates, at tensor stride ts, shuffled."""
    c = unique_cloud(3000, 12, seed, batches=3, allow_negative=True)
    c[:, 1:] *= ts
    return c


def _assert_same_pairs(got, im, om, what):
    assert len(got) == len(im), what
    for k, (i, o) in enumerate(got):
        assert np.array_equal(i.numpy(), im[k]) and np.array_equal(o.numpy(), om[k]), \
            f"{what}: offset {k} differs"


# (kernel size, stride, tensor stride, transposed): the stem, the K = 27 blocks, the strided and
# transposed layers of every level, and K = 1
LAYERS = [(5, 1, 1, False), (3, 1, 1, False), (3, 1, 4, False), (3, 1, 8, False),
          (1, 1, 1, False), (1, 1, 2, False)] + \
    [(2, 2, ts, False) for ts in (1, 2, 4, 8)] + [(2, 2, ts, True) for ts in (2, 4, 8)]


@pytest.mark.parametrize("ks,stride,ts,transposed", LAYERS,
                         ids=[f"k{c[0]}s{c[1]}ts{c[2]}" + ("tr" if c[3] else "") for c in LAYERS])
def test_map_restatement_matches_oracle(ks, stride, ts, transposed):
    D = 3
    if not transposed:
        cin = _cloud(ts, seed=ks * 10 + ts)
        cin_np = cin.numpy()
        if stride == 1:
            cout_np = cin_np
        else:
            cout_np, out_ts = O.stride_map_coords(cin_np, [ts] * D, [stride] * D)
            got = strided_coords(cin, out_ts)
            assert np.array_equal(got.numpy(), cout_np), "strided coordinates differ"
            cout_np = cout_np[np.random.default_rng(ts).permutation(len(cout_np))]
        offs = offsets_of([ks] * D, [1] * D, [ts] * D)
        im, om = O.kernel_map(cin_np, cout_np, offs)
        got = conv_pairs(cin, torch.from_numpy(np.ascontiguousarray(cout_np)), offs)
    else:
        fine_ts = ts // stride
        fine = _cloud(fine_ts, seed=ts)
        coarse, _ = O.stride_map_coords(fine.numpy(), [fine_ts] * D, [stride] * D)
        coarse = coarse[np.random.default_rng(ts).permutation(len(coarse))]
        offs = offsets_of([ks] * D, [1] * D, [fine_ts] * D)
        im, om = O.transposed_kernel_map(coarse, fine.numpy(), offs)
        got = conv_pairs(torch.from_numpy(np.ascontiguousarray(coarse)), fine, offs, transposed=True)
    assert sum(len(i) for i in im) > 0
    _assert_same_pairs(got, im, om, f"k{ks} s{stride} ts{ts}")


def test_map_restatement_edges():
    """Empty offsets, a query outside the coordinate box, one-row maps and a batch of its own."""
    c = torch.tensor([[0, -5, 0, 7], [2, 100, -100, 3]], dtype=torch.int32)
    offs = offsets_of([3] * 3, [1] * 3, [1] * 3)
    im, om = O.kernel_map(c.numpy(), c.numpy(), offs)
    _assert_same_pairs(conv_pairs(c, c, offs), im, om, "two isolated rows")
    assert sum(len(i) for i in im) == 2
    with pytest.raises(AssertionError, match="int64 key"):
        conv_pairs(torch.tensor([[0, -2 ** 30, 0, 0], [9, 2 ** 30, 0, 0]], dtype=torch.int32),
                   c, offs)


MODELS = ["MinkUNet14", "MinkUNet34C"]


@pytest.mark.parametrize("model", MODELS)
def test_recording_handle_builds_the_same_network(ME, model):
    from minkowskiengine_b200.convolution import MinkowskiConvolutionBase
    torch.manual_seed(0)
    plain = minkunet(model, ME, 3, 20, 3)
    audit = StepAudit(ME)
    handle = RecordingHandle(ME, audit)
    torch.manual_seed(0)
    rec = minkunet(model, handle, 3, 20, 3)
    a, b = plain.state_dict(), rec.state_dict()
    assert list(a) == list(b)
    for k in a:
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
    assert [n for n, _ in plain.named_parameters()] == [n for n, _ in rec.named_parameters()]
    assert np.array_equal(state_digest(plain), state_digest(rec))
    wrapped = (handle.MinkowskiConvolution, handle.MinkowskiConvolutionTranspose,
               handle.MinkowskiBatchNorm)
    n_conv = n_bn = 0
    for m in rec.modules():
        if isinstance(m, MinkowskiConvolutionBase):
            assert isinstance(m, wrapped[:2]), f"{type(m).__name__} is not recorded"
            n_conv += 1
        if isinstance(m, ME.MinkowskiBatchNorm):
            assert isinstance(m, wrapped[2]), f"{type(m).__name__} is not recorded"
            n_bn += 1
    assert n_conv == sum(isinstance(m, MinkowskiConvolutionBase) for m in plain.modules())
    assert n_bn == sum(isinstance(m, ME.MinkowskiBatchNorm) for m in plain.modules())
    assert handle.fused_conv_bn_relu == audit.fused_conv_bn_relu
    assert handle.fused_bn_relu == audit.fused_bn_relu and handle.cat == audit.cat
    audit.names(rec)
    assert audit._name(rec.final) == "final"


def test_wgrad_share_steps():
    """The split plan of run_wgrad on 132 SMs: K = 27 and 96 channels at 800k rows split each
    offset 10 ways (2 waves / 27 offsets) over 4 row chunks; K = 1 over 2048 rows: the workspace,
    sized for 32 stages, holds 8 splits, but 2048 / 192 + 1 = 11 estimated stages plan 2; over
    500 rows the plan is one split."""
    pairs = [800_000] + [100_000] * 26
    assert wgrad_share_steps(pairs, 800_000, 800_000, 96, 132)[:2] == \
        [4 * (-(-(12_500 + 4) // 10) + 4), 4 * (-(-(1_563 + 4) // 10) + 4)]
    assert wgrad_share_steps([2048], 2048, 2048, 64, 132) == [4 * (-(-(32 + 1) // 2) + 1)]
    assert wgrad_share_steps([500], 500, 500, 64, 132) == [4 * (8 + 1 + 1)]
