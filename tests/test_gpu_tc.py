"""wgmma (tensor-core) convolution path: bf16 / fp16 operands, fp32 accumulation.

Every output is checked element by element against a float64 restatement fed the same
bf16 / fp16-rounded features and weights (tests/helpers.py): |y - ref| <= TC_ACC * 2^-20 * A,
A the same reduction over absolute values, plus one rounding when the output is stored in
bf16 / fp16.  Forward and dgrad write every element once and the wgrad adds its row splits in a
fixed order, so every result must also be bit-identical run to run."""
import pytest
import torch

from helpers import (TC_ACC, _pairs, assert_one_rounding, lib_conv_backward, ref_conv, ref_wgrad,
                     unique_cloud)
from oracle import oracle_np as O

pytestmark = pytest.mark.gpu


def _random_table(K, n_out, n_in, density, seed, device):
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, n_in, (K, n_out), generator=g, dtype=torch.int32)
    drop = torch.rand((K, n_out), generator=g) > density
    idx[drop] = -1
    return idx.to(device)


def _tc(fn):
    """fn() with the tensor-core launches it made asserted non-zero."""
    from minkowskiengine_b200 import _lib
    n0 = _lib.tc_launch_count()
    out = fn()
    assert _lib.tc_launch_count() > n0, "did not take the tensor-core path"
    return out


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K", [
    (16, 16, 500, 100, 27),          # single partial tile, BK=16
    (32, 32, 3000, 3001, 27),        # BK=32, R=4 super tiles with a ragged tail
    (64, 128, 5000, 2000, 27),       # BASELINE cfg1 channel shape, BK=64
    (96, 96, 4000, 4000, 27),        # MinkUNet34C stride-1 blocks (BK=32, N=96)
    (128, 96, 4000, 1000, 8),
    (192, 128, 1000, 1000, 27),
    (384, 256, 700, 300, 27),        # widest concat layer, N=256 (R=1)
    (256, 256, 300, 129, 27),
    (32, 64, 90000, 90000, 8),       # more super tiles than SMs: persistent loop + phases
])
def test_tc_forward_matches_fp32_reference(ME, cuda, dtype, cin, cout, n_in, n_out, K):
    """A kernel already in the feature dtype (packed alone, not an fp32 master)."""
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(cin * 1000 + cout)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(dtype).to(cuda)
    nbr = _random_table(K, n_out, n_in, 0.35, seed=K + n_out, device=cuda)
    km = backend._KernelMap(nbr, torch.empty((K, n_in), dtype=torch.int32, device=cuda))
    ref, A = ref_conv(feats, w, _pairs(nbr), n_out)
    out32 = _tc(lambda: backend._conv_forward(feats, w, km, out_dtype=torch.float32))
    assert_one_rounding(out32, ref, A, "forward, fp32 output", TC_ACC)
    out_lp = _tc(lambda: backend._conv_forward(feats, w, km))
    assert out_lp.dtype == dtype
    assert_one_rounding(out_lp, ref, A, "forward", TC_ACC)
    assert torch.equal(out_lp, backend._conv_forward(feats, w, km)), "forward differs run to run"
    assert torch.equal(out32, backend._conv_forward(feats, w, km, out_dtype=torch.float32))


def _to_pairs(im, om, device):
    return [(torch.as_tensor(i, dtype=torch.long, device=device),
             torch.as_tensor(o, dtype=torch.long, device=device)) for i, o in zip(im, om)]


@pytest.mark.parametrize("dtype", [torch.bfloat16])
@pytest.mark.parametrize("cin,cout,ks,stride", [(32, 64, 3, 1), (64, 96, 3, 2), (96, 32, 2, 2)])
def test_tc_layer_vs_oracle(ME, cuda, dtype, cin, cout, ks, stride):
    """Through the public API (SparseTensor + MinkowskiConvolution, bf16 features), forward
    and backward, against float64 on the oracle's kernel maps, fed the same rounded values."""
    D = 3
    coords = unique_cloud(6000, 24, seed=5, allow_negative=True)
    g = torch.Generator().manual_seed(9)
    feats = torch.rand(len(coords), cin, generator=g).to(dtype)
    conv = ME.MinkowskiConvolution(cin, cout, kernel_size=ks, stride=stride, dimension=D).to(cuda)
    gout = None
    runs = []
    for _ in range(2):
        conv.kernel.grad = None
        x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
        y = _tc(lambda: conv(x))
        assert y.F.dtype == dtype
        if gout is None:
            gout = (torch.rand(y.F.shape, generator=g) - 0.5).to(dtype).to(cuda)
        _tc(lambda: y.F.backward(gout))
        runs.append((x, y, x.F.grad.clone(), conv.kernel.grad.clone()))
    (x, y, gi, gw), (_, y2, gi2, gw2) = runs
    assert torch.equal(y.F, y2.F) and torch.equal(gi, gi2) and torch.equal(gw, gw2), \
        "layer differs run to run"
    in_c, out_c = x.C.cpu().numpy(), y.C.cpu().numpy()
    offs = O.region_offsets(O.HYPER_CUBE, [ks] * D, [1] * D, [1] * D)
    pairs = _to_pairs(*O.kernel_map(in_c, out_c, offs), cuda)
    w = conv.kernel.detach().to(dtype)
    y_ref, y_A = ref_conv(x.F.detach(), w, pairs, len(out_c))
    assert_one_rounding(y.F.detach(), y_ref, y_A, "layer forward", TC_ACC)
    gi_ref, gi_A = ref_conv(gout, w.transpose(1, 2), [(o, i) for i, o in pairs], len(in_c))
    assert_one_rounding(gi, gi_ref, gi_A, "layer dgrad (bf16)", TC_ACC)
    gw_ref, gw_A = ref_wgrad(x.F.detach(), gout, pairs)
    assert_one_rounding(gw, gw_ref, gw_A, "layer wgrad (fp32)", TC_ACC)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K", [
    (16, 16, 500, 100, 27),
    (32, 32, 3000, 3001, 27),
    (64, 128, 5000, 2000, 27),
    (96, 96, 4000, 4000, 27),       # N = 96: one and a half 64-channel blocks
    (128, 96, 4000, 1000, 8),
    (192, 128, 1000, 1000, 27),     # two m-tiles (128 + 64 padded)
    (384, 256, 700, 300, 27),       # three m-tiles -> two m-tile groups
    (256, 256, 300, 129, 27),
    (24, 48, 777, 333, 5),          # channel counts that are not multiples of 16 / 64
    (32, 64, 60000, 60000, 8),
])
def test_tc_wgrad_matches_fp32_reference(ME, cuda, dtype, cin, cout, n_in, n_out, K):
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(cin * 77 + cout)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    w = torch.zeros(K, cin, cout, dtype=torch.float32, device=cuda)   # fp32 master weights
    nbr = _random_table(K, n_out, n_in, 0.35, seed=K + n_out + 1, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    _, gw = _tc(lambda: backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True))
    _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    ref, A = ref_wgrad(feats, gout, _pairs(nbr))
    assert gw.dtype == torch.float32
    assert_one_rounding(gw, ref, A, "wgrad", TC_ACC)
    assert torch.equal(gw, gw2), "wgrad differs run to run"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("cin,cout,n_in,n_out,K", [
    (32, 32, 3000, 3001, 27),        # one 32-channel block per stage, R = 4, ragged tail
    (32, 16, 500, 100, 27),          # single partial tile
    (64, 128, 5000, 2000, 27),       # two blocks per stage (128B-swizzled weights)
    (96, 96, 4000, 4000, 27),        # three blocks per stage: the MinkUNet34C stride-1 blocks
    (128, 96, 4000, 1000, 8),        # two stages per (tile, offset)
    (192, 128, 1000, 1000, 27),
    (384, 256, 700, 300, 27),        # four stages per offset, N = 256 (single accumulator set)
    (256, 384, 300, 129, 27),        # output columns split in two launches
    (160, 64, 2000, 1500, 5),        # 160 = 5 blocks of 32 (one block per stage)
    (32, 64, 90000, 90000, 8),       # more super tiles than SMs: persistent loop + phases
    (96, 96, 50000, 50000, 27),
])
def test_ta_forward_and_dgrad_packed_weights(ME, cuda, dtype, cin, cout, n_in, n_out, K):
    """fp32 master weights -> packed operand copies -> k_conv_wg:
    forward over out_nbr and dgrad over in_nbr against float64, in the feature dtype and in fp32."""
    from minkowskiengine_b200 import backend
    g = torch.Generator().manual_seed(cin * 1000 + cout + 7)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).to(dtype).to(cuda)
    w = ((torch.rand(K, cin, cout, generator=g) - 0.5) / (cin ** 0.5)).to(cuda)   # fp32 master
    out_nbr = _random_table(K, n_out, n_in, 0.35, seed=K + n_out, device=cuda)
    in_nbr = _random_table(K, n_in, n_out, 0.3, seed=K + n_in + 3, device=cuda)
    km = backend._KernelMap(out_nbr, in_nbr)
    ref, A = ref_conv(feats, w.to(dtype), _pairs(out_nbr), n_out)
    out32 = _tc(lambda: backend._conv_forward(feats, w, km, out_dtype=torch.float32))
    assert_one_rounding(out32, ref, A, "forward, fp32 output", TC_ACC)
    out_lp = backend._conv_forward(feats, w, km)
    assert out_lp.dtype == dtype
    assert_one_rounding(out_lp, ref, A, "forward", TC_ACC)
    assert torch.equal(out_lp, backend._conv_forward(feats, w, km)), "forward differs run to run"
    # weights modified in place -> the packed copies must be rebuilt
    with torch.no_grad():
        w.mul_(0.5)
    out_half = backend._conv_forward(feats, w, km, out_dtype=torch.float32)
    ref, A = ref_conv(feats, w.to(dtype), _pairs(out_nbr), n_out)
    assert_one_rounding(out_half, ref, A, "forward after an in-place weight update", TC_ACC)
    # dgrad: rows = input rows, reduction over c_out, W_k^T
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).to(dtype).to(cuda)
    ref, A = ref_conv(gout, w.to(dtype).transpose(1, 2), _pairs(in_nbr), n_in)
    gi, _ = _tc(lambda: backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False))
    gi2, _ = backend._conv_backward(feats, gout, w, km, need_in=True, need_w=False)
    assert gi.dtype == dtype
    assert_one_rounding(gi, ref, A, "dgrad", TC_ACC)
    assert torch.equal(gi, gi2), "dgrad differs run to run"
    gi32, _ = _tc(lambda: lib_conv_backward(feats, gout, w, km, grad_in_dtype=torch.float32))
    assert_one_rounding(gi32, ref, A, "dgrad, fp32 output", TC_ACC)
    assert torch.equal(gi32, lib_conv_backward(feats, gout, w, km, grad_in_dtype=torch.float32)[0])


@pytest.mark.parametrize("K,n,density,chunk", [(27, 5000, 0.3, 2048), (8, 70000, 0.125, 65536),
                                               (1, 100, 1.0, 65536), (125, 3001, 0.05, 2048),
                                               (27, 2048, 0.0, 2048), (81, 40000, 0.4, 4096),
                                               (27, 150000, 0.3, 65536)])
def test_pair_lists_match_table(ME, cuda, K, n, density, chunk, monkeypatch):
    """meb200_kernel_map_pairs: compacted (other row, table row) lists in (row chunk, offset)
    order, table-row order inside a segment, every segment padded with -1 to a multiple of the
    stage — against torch.nonzero."""
    from minkowskiengine_b200 import backend
    monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", chunk)
    nbr = _random_table(K, n, 12345, density, seed=K + n, device=cuda)
    km = backend._KernelMap(nbr, torch.empty((K, 1), dtype=torch.int32, device=cuda))
    pin, pout, seg, nch = km.pair_lists()
    S = km.PAIR_STAGE
    seg_h = seg.cpu().tolist()
    assert seg_h[0] == 0 and len(seg_h) == nch * K + 1
    bpc = -(-chunk // 2048)                   # table blocks (2048 rows) per chunk
    assert nch == -(-(-(-n // 2048)) // bpc)
    covered = 0
    for c in range(nch):
        r0, r1 = c * bpc * 2048, min((c + 1) * bpc * 2048, n)
        for k in range(K):
            rows = torch.nonzero(nbr[k, r0:r1] >= 0).flatten() + r0
            cnum = len(rows)
            a, b = seg_h[c * K + k], seg_h[c * K + k + 1]
            assert b - a == (cnum + S - 1) // S * S
            assert torch.equal(pout[a:a + cnum].long(), rows)
            assert torch.equal(pin[a:a + cnum], nbr[k][rows])
            assert bool((pin[a + cnum:b] == -1).all()) and bool((pout[a + cnum:b] == -1).all())
            covered += cnum
    assert covered == int((nbr >= 0).sum())
    # the swapped view exchanges the two sides and shares the storage
    sw = km.swapped()
    sin, sout, sseg, snch = sw.pair_lists()
    assert sin.data_ptr() == pout.data_ptr() and sout.data_ptr() == pin.data_ptr()
    assert sseg.data_ptr() == seg.data_ptr() and snch == nch


def test_wgrad_pairs_many_chunks(ME, cuda, monkeypatch):
    """k_wgrad_wg walking several row chunks of the pair lists (small chunks forced) against float64."""
    from minkowskiengine_b200 import backend
    monkeypatch.setattr(backend._KernelMap, "PAIR_CHUNK_ROWS", 4096)
    K, n_in, n_out, cin, cout = 27, 30000, 33000, 96, 96
    g = torch.Generator().manual_seed(5)
    feats = (torch.rand(n_in, cin, generator=g) - 0.5).bfloat16().to(cuda)
    gout = (torch.rand(n_out, cout, generator=g) - 0.5).bfloat16().to(cuda)
    w = torch.zeros(K, cin, cout, device=cuda)
    nbr = _random_table(K, n_out, n_in, 0.3, seed=11, device=cuda)
    km = backend._KernelMap(nbr, torch.full((K, n_in), -1, dtype=torch.int32, device=cuda))
    _, gw = _tc(lambda: backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True))
    assert km.pair_lists()[3] == 9
    ref, A = ref_wgrad(feats, gout, _pairs(nbr))
    assert_one_rounding(gw, ref, A, "chunked pair-list wgrad", TC_ACC)
    _, gw2 = backend._conv_backward(feats, gout, w, km, need_in=False, need_w=True)
    assert torch.equal(gw, gw2), "wgrad differs run to run"


def test_batched_weight_packing_equals_single_and_cast(ME, cuda):
    """The one-launch re-pack of every registered kernel (backend._PackTable,
    meb200_conv_pack_weights_batched) must leave exactly the bytes the per-kernel packing leaves,
    which are the kernel cast to the feature dtype (and its per-offset transpose), for ragged and
    32-aligned channel counts, and track tensors that die or move."""
    from minkowskiengine_b200 import backend, _lib
    lib = _lib.load()
    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(5)
    shapes = [(27, 32, 64), (8, 96, 96), (1, 5, 7), (27, 48, 20), (125, 64, 32), (3, 256, 128)]
    ks = [torch.nn.Parameter(torch.randn(s, generator=g).to(cuda)) for s in shapes]

    def single(k):
        K, ci, co = k.shape
        buf = torch.empty((2, K * ci * co), dtype=dtype, device=cuda)
        _lib.check(lib.meb200_conv_pack_weights(
            _lib.ptr(k.detach()), K, ci, co, _lib.dtype_code(dtype), _lib.ptr(buf[0]),
            _lib.ptr(buf[1]), _lib.current_stream()))
        return buf

    def check(k):
        got = backend._packed_weights(k, dtype)
        ref = single(k)
        assert torch.equal(got[0].flatten(), ref[0]) and torch.equal(got[1].flatten(), ref[1])
        assert torch.equal(got[0], k.detach().to(dtype))
        assert torch.equal(got[1], k.detach().to(dtype).transpose(1, 2))

    for k in ks:            # first sight: packed one by one, registered
        check(k)
    tbl = backend._PACK_TABLES[(torch.device(cuda).index or 0, dtype)]
    n0 = lib.meb200_launch_count()
    with torch.no_grad():   # "optimizer step": every kernel changes
        for k in ks:
            k.add_(0.5)
    got0 = backend._packed_weights(ks[0], dtype)          # one batched launch re-packs all of them
    assert lib.meb200_launch_count() == n0 + 1
    for k in ks:
        assert backend._PACKED[id(k)][1] == k._version     # all fresh: no further launches
    n1 = lib.meb200_launch_count()
    for k in ks:
        backend._packed_weights(k, dtype)
    assert lib.meb200_launch_count() == n1
    for k in ks:
        check(k)
    # a tensor dies, another is re-allocated: the table is rebuilt, results stay right
    del ks[2]
    with torch.no_grad():
        ks[1].data = ks[1].data.clone()
        for k in ks:
            k.mul_(1.25)
    for k in ks:
        check(k)
    assert all(e[0]() is not None for e in tbl.entries.values()) or True
