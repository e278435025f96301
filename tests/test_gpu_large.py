"""Full-size (BASELINE.json configs) checks through size-independent properties, where the
numpy oracle would take too long:
  * kernel-map symmetry: for an odd kernel at stride 1, pair (k, i, o) exists iff
    (K-1-k, o, i) exists — i.e. out_nbr[K-1-k] is the transpose of out_nbr[k];
  * table consistency: in_nbr is exactly the transpose of out_nbr, pair count = symmetric sum;
  * insert idempotence: inserting the unique coordinates again yields identity maps;
  * stride: every output coordinate is the floor of at least one input, no duplicates;
  * convolution linearity and an fp32 torch restatement on the device (tensor-core bf16 path,
    cfg1: 100k coords, 64 -> 128, k=3, s=2), dgrad/wgrad adjointness <dY, conv(X)> identities;
  * 4-D (cfg4: 200k draws, K = 81) hashing stress against a sort-based torch lookup."""
import pytest
import torch

from oracle.oracle_np import surface_cloud

pytestmark = pytest.mark.gpu


def _maps(ME, coords, cuda, ks, stride, D=3):
    x = ME.SparseTensor(torch.zeros(len(coords), 1), coords, device=cuda)
    mgr = x.coordinate_manager
    out_key = x.coordinate_map_key if stride == 1 else mgr.stride(x.coordinate_map_key, stride)
    km = mgr._manager._kernel_map(x.coordinate_map_key, out_key, [ks] * D, [stride] * D, [1] * D,
                                  ME.RegionType.HYPER_CUBE, torch.IntTensor(), False, False)
    return x, mgr, out_key, km


def test_kernel_map_symmetry_100k(ME, cuda):
    coords = surface_cloud(100_000, seed=0)
    x, mgr, _, km = _maps(ME, coords, cuda, 3, 1)
    K, n = km.out_nbr.shape
    assert K == 27 and n == 100_000
    rows = torch.arange(n, device=cuda, dtype=torch.int32)
    pairs = 0
    for k in range(K):
        o = km.out_nbr[k]
        hit = o >= 0
        pairs += int(hit.sum())
        # (k, i=o[r], o=r) exists  <=>  (K-1-k, i=r, o=o[r]) exists
        back = km.out_nbr[K - 1 - k][o[hit].long()]
        assert torch.equal(back, rows[hit])
        # in_nbr is the transpose table
        assert torch.equal(km.in_nbr[k][o[hit].long()], rows[hit])
    assert pairs == 846_116          # SURVEY.md §8 probe count for surface(100k, seed 0), k=3 s=1
    assert int((km.in_nbr >= 0).sum()) == pairs
    assert torch.equal(km.out_nbr[13], rows)     # centre offset maps every row to itself


def test_insert_idempotent_and_stride_properties_100k(ME, cuda):
    coords = surface_cloud(100_000, seed=0)
    dup = torch.cat([coords, coords[:5000]])                 # 5000 duplicates at the end
    x = ME.SparseTensor(torch.zeros(len(dup), 1), dup, device=cuda)
    assert len(x) == 100_000 and torch.equal(x.C.cpu(), coords)
    assert torch.equal(x.inverse_mapping.cpu()[100_000:], torch.arange(5000))
    mgr = x.coordinate_manager
    key2, (ui, inv) = mgr.insert_and_map(x.C, 1, "again")
    assert len(inv) == 0 and torch.equal(ui.cpu(), torch.arange(100_000))
    s2 = mgr.stride(x.coordinate_map_key, 2)
    c2 = mgr.get_coordinates(s2)
    assert len(torch.unique(c2, dim=0)) == len(c2) == 39_234            # SURVEY.md §8 level size
    assert bool(((c2[:, 1:] % 2) == 0).all())
    fl = x.C.clone()
    fl[:, 1:] = torch.div(fl[:, 1:], 2, rounding_mode="floor") * 2
    assert len(torch.unique(torch.cat([fl, c2]), dim=0)) == len(c2)     # same coordinate set


def _torch_conv(feats, w, out_nbr):
    out = torch.zeros((out_nbr.shape[1], w.shape[2]), dtype=torch.float32, device=feats.device)
    for k in range(out_nbr.shape[0]):
        idx = out_nbr[k].long()
        out += (feats.float()[idx.clamp(min=0)] * (idx >= 0).unsqueeze(1)) @ w[k].float()
    return out


def test_cfg1_single_conv_bf16_100k(ME, cuda):
    """BASELINE configs[1]: k=3 s=2, 100k coords, 64 -> 128, bf16 operands / fp32 accumulate."""
    from minkowskiengine_b200 import _lib, backend
    torch.backends.cuda.matmul.allow_tf32 = False
    coords = surface_cloud(100_000, seed=0)
    x, mgr, out_key, km = _maps(ME, coords, cuda, 3, 2)
    assert km.n_out == 39_234 and int((km.out_nbr >= 0).sum()) == 270_325   # SURVEY.md §8 counts
    g = torch.Generator(device="cpu").manual_seed(0)
    feats = torch.rand(100_000, 64, generator=g).to(torch.bfloat16).to(cuda)
    w = ((torch.rand(27, 64, 128, generator=g) * 2 - 1) / (27 * 64) ** 0.5).to(cuda)
    wl = w.to(torch.bfloat16)
    before = _lib.tc_launch_count()
    y = backend._conv_forward(feats, wl, km, out_dtype=torch.float32)
    assert _lib.tc_launch_count() > before, "forward did not take the tensor-core path"
    ref = _torch_conv(feats, wl, km.out_nbr)
    assert float((y - ref).abs().max() / ref.abs().max()) < 1e-4
    # linearity: conv(a*X1 + X2) == a*conv(X1) + conv(X2) (fp32 output, exact bf16 inputs)
    f2 = torch.rand(100_000, 64, generator=g).to(torch.bfloat16).to(cuda)
    y2 = backend._conv_forward(f2, wl, km, out_dtype=torch.float32)
    ysum = backend._conv_forward((feats.float() * 0.5 + f2.float()).to(torch.bfloat16), wl, km,
                                 out_dtype=torch.float32)
    mixed_ref = _torch_conv((feats.float() * 0.5 + f2.float()).to(torch.bfloat16), wl, km.out_nbr)
    assert float((ysum - mixed_ref).abs().max() / mixed_ref.abs().max()) < 1e-4
    assert float((ysum - (0.5 * y + y2)).abs().max() / ysum.abs().max()) < 2e-2  # bf16 input rounding
    # adjointness: <dY, conv(X)> == <dgrad(dY), X> == <wgrad(X, dY), W>
    dy = (torch.rand(km.n_out, 128, generator=g) - 0.5).to(torch.bfloat16).to(cuda)
    gi, gw = backend._conv_backward(feats, dy, w, km)
    lhs = float((dy.float() * ref).sum())
    assert abs(float((gi.float() * feats.float()).sum()) - lhs) / abs(lhs) < 5e-3   # bf16-stored dgrad
    assert abs(float((gw.float() * wl.float()).sum()) - lhs) / abs(lhs) < 1e-4      # fp32 wgrad


def test_cfg4_4d_hash_stress(ME, cuda):
    """BASELINE configs[4]: 4-D coordinates (b, x, y, z, t), 200k draws, k = 3 (K = 81)."""
    g = torch.Generator().manual_seed(0)
    v = torch.randn(200_000, 3, generator=g)
    v = v / v.norm(dim=1, keepdim=True)
    t = torch.randint(0, 8, (200_000, 1), generator=g)
    c = torch.floor(45 * v + 0.5 * t).int()
    coords = torch.cat([torch.zeros(200_000, 1, dtype=torch.int32), c, t.int()], 1)
    uniq = torch.unique(coords, dim=0)
    assert len(uniq) == 131_897                                   # SURVEY.md §8d probe count
    x, mgr, _, km = _maps(ME, coords, cuda, 3, 1, D=4)
    assert len(x) == 131_897 and km.out_nbr.shape == (81, 131_897)
    assert int((km.out_nbr >= 0).sum()) == 2_378_593              # SURVEY.md §8d pair count
    # spot-check 3 offsets against a sort-based lookup done with torch
    C = x.C.long()
    base = 128
    def key(cc):
        k = cc[:, 0]
        for j in range(1, 5):
            k = k * base + (cc[:, j] + 60)
        return k
    keys = key(C)
    order = torch.argsort(keys)
    sk = keys[order]
    for k in (0, 40, 77):
        off = []
        rem = k
        for _ in range(4):
            off.append(rem % 3 - 1)
            rem //= 3
        q = C.clone()
        q[:, 1:] += torch.tensor(off, device=cuda)
        qk = key(q)
        pos = torch.searchsorted(sk, qk).clamp(max=len(sk) - 1)
        hit = sk[pos] == qk
        exp = torch.where(hit, order[pos], torch.full_like(pos, -1)).int()
        assert torch.equal(km.out_nbr[k], exp)


def _cfg4_cloud(n_draws, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n_draws, 3, generator=g)
    v = v / v.norm(dim=1, keepdim=True)
    t = torch.randint(0, 8, (n_draws, 1), generator=g)
    r = 45.0 * (n_draws / 200_000) ** 0.5
    c = torch.floor(r * v + 0.5 * t).int()
    return torch.unique(torch.cat([torch.zeros(n_draws, 1, dtype=torch.int32), c, t.int()], 1), dim=0)


def test_cfg4_4d_conv_bf16_vs_oracle_20k(ME, cuda):
    """BASELINE configs[4] layer (4-D, k=3 => K=81, C=32 -> 32, bf16) through the public API at
    >= 20k coordinates: kernel map + forward + dgrad + wgrad against the numpy oracle."""
    import numpy as np
    from oracle import oracle_np as O
    coords = _cfg4_cloud(32_000, seed=1)
    assert len(coords) >= 20_000
    g = torch.Generator().manual_seed(4)
    feats = torch.rand(len(coords), 32, generator=g).bfloat16()
    conv = ME.MinkowskiConvolution(32, 32, kernel_size=3, stride=1, dimension=4).to(cuda)
    x = ME.SparseTensor(feats, coords, device=cuda, requires_grad=True)
    y = conv(x)
    in_c = x.C.cpu().numpy()
    im, om = O.kernel_map(in_c, in_c, O.region_offsets(O.HYPER_CUBE, [3] * 4, [1] * 4, [1] * 4))
    km = x.coordinate_manager._manager._kernel_map(
        x.coordinate_map_key, y.coordinate_map_key, [3] * 4, [1] * 4, [1] * 4,
        ME.RegionType.HYPER_CUBE, torch.IntTensor(), False, False)
    nbr = km.out_nbr.cpu().numpy()
    assert int((nbr >= 0).sum()) == sum(len(i) for i in im)
    for k in range(81):                         # bit-exact: pairs of offset k, ordered by out row
        o = np.nonzero(nbr[k] >= 0)[0]
        order = np.argsort(om[k], kind="stable")
        assert (o == om[k][order]).all() and (nbr[k][o] == im[k][order]).all()
    w = conv.kernel.detach().bfloat16().float().cpu().numpy()
    f = feats.float().numpy()
    ref = O.conv_forward(f, w, im, om, len(in_c))
    e = np.abs(y.F.detach().float().cpu().numpy() - ref).max() / np.abs(ref).max()
    assert e < 6e-3, e                          # one bf16 output rounding
    gout = (torch.rand(y.F.shape, generator=g) - 0.5).bfloat16()
    y.F.backward(gout.to(cuda))
    gi, gw = O.conv_backward(f, gout.float().numpy(), w, im, om)
    assert np.abs(x.F.grad.float().cpu().numpy() - gi).max() / np.abs(gi).max() < 6e-3
    assert np.abs(conv.kernel.grad.float().cpu().numpy() - gw).max() / np.abs(gw).max() < 1e-3


def test_cfg4_4d_conv_bf16_full_size_properties(ME, cuda):
    """configs[4] at full size (200k draws -> 131 897 coordinates, K = 81, C = 32): the tensor-core
    path against an fp32 torch restatement on the device, and the adjoint identities."""
    from minkowskiengine_b200 import _lib, backend
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(0)
    v = torch.randn(200_000, 3, generator=g)
    v = v / v.norm(dim=1, keepdim=True)
    t = torch.randint(0, 8, (200_000, 1), generator=g)
    c = torch.floor(45 * v + 0.5 * t).int()
    coords = torch.cat([torch.zeros(200_000, 1, dtype=torch.int32), c, t.int()], 1)
    x, mgr, _, km = _maps(ME, coords, cuda, 3, 1, D=4)
    n = len(x)
    assert n == 131_897
    feats = torch.rand(n, 32, generator=g).bfloat16().to(cuda)
    w = ((torch.rand(81, 32, 32, generator=g) * 2 - 1) / (81 * 32) ** 0.5).to(cuda)
    wl = w.bfloat16()
    before = _lib.tc_launch_count()
    y = backend._conv_forward(feats, wl, km, out_dtype=torch.float32)
    assert _lib.tc_launch_count() > before, "4-D forward did not take the tensor-core path"
    ref = _torch_conv(feats, wl, km.out_nbr)
    assert float((y - ref).abs().max() / ref.abs().max()) < 1e-4
    dy = (torch.rand(n, 32, generator=g) - 0.5).bfloat16().to(cuda)
    gi, gw = backend._conv_backward(feats, dy, w, km)
    lhs = float((dy.float() * ref).sum())
    assert abs(float((gi.float() * feats.float()).sum()) - lhs) / abs(lhs) < 5e-3
    assert abs(float((gw.float() * wl.float()).sum()) - lhs) / abs(lhs) < 1e-4
