"""libmeb200's batch-norm passes (csrc/batchnorm.cu) against float64, over every launch geometry
they take, in fp32, bf16 and fp16.

* The launch geometry (bn_rows_per_cta and the 512-CTA clamp of bn_launch_reduce) is restated in
  Python; a CPU test asserts that the cases below reach every branch of the reduction.
* The library entry points run on inputs whose sums are exact: x = j / 4 with small integers j,
  so every per-thread fp32 partial of x and x^2 is exact, and so is every fp64 sum above it.  The
  statistics must then be the float64 ones bit for bit (the mean: the fp32 rounding of S1 / n;
  invstd and the running statistics within one fp32 ulp).  A row dropped, added twice or credited
  to the wrong channel changes them, however large n is.
* The apply passes run on statistics the test supplies, the modules on random data against
  float64 torch.nn.BatchNorm1d, each element within a bound derived from the arithmetic the
  kernels declare (_stat_bounds, _y_bound, _dx_bound)."""
import zlib
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from helpers import half_ulp

THREADS = 256                    # kBnThreads
MAX_CTAS = 512                   # kBnMaxCtas: one workspace slot per reduction CTA
UNROLL = 4                       # rows per iteration of the reduce and apply loops
SM_COUNTS = {"H100 SXM": 132, "H100 PCIe": 114}
U = 2.0 ** -24                   # unit roundoff of fp32
V = 2.0 ** -53                   # and of fp64
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# the C ABI takes eps and momentum as fp32: every reference uses those values
EPS = float(np.float32(1e-5))
MOM = float(np.float32(0.1))


def cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Geom:
    n: int
    C: int
    rows_per_pass: int           # rows one pass of the CTA covers: THREADS // (C / 8)
    idle: int                    # threads of a CTA without a channel group
    rows: int                    # rows per reduction CTA
    grid: int                    # reduction CTAs
    clamped: bool                # the reduction took the 512-CTA clamp
    J: int                       # threads per total in the last CTA's combine (1: direct loop)
    apply_grid: int              # CTAs of the apply passes (never clamped)

    @property
    def per_thread(self):        # rows one thread sums in every reduction CTA but the last
        return self.rows // self.rows_per_pass

    @property
    def last_rows(self):
        return self.n - (self.grid - 1) * self.rows


def bn_geometry(n, C, sms=None):
    """Launch geometry of the batch-norm passes over [n, C] on `sms` SMs (default: the current
    device's), as bn_rows_per_cta and bn_launch_reduce compute it."""
    if sms is None:
        sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    rpp = THREADS // (C // 8)
    rows = max(cdiv(n, 8 * sms), 8 * rpp)           # ~8 CTAs per SM, at least 8 rows per thread
    rows = cdiv(rows, rpp) * rpp
    grid = cdiv(n, rows)
    apply_grid = grid
    clamped = grid > MAX_CTAS
    if clamped:
        rows = cdiv(cdiv(n, MAX_CTAS), rpp) * rpp
        grid = cdiv(n, rows)
    return Geom(n=n, C=C, rows_per_pass=rpp, idle=THREADS - (C // 8) * rpp, rows=rows,
                grid=max(grid, 1), clamped=clamped,
                J=1 if 2 * C >= THREADS else THREADS // (2 * C),
                apply_grid=apply_grid)


CFG3 = [(800_000, 32), (800_000, 96), (800_000, 256)]   # bench.py cfg3: a MinkUNet34C's widths
CASES = [
    (1, 8), (3, 8),              # one CTA, fewer than the J = 16 combine threads
    (3, 2048),                   # one row per pass
    (200_003, 8),                # 256 rows per pass, J = 16 over 98 CTAs
    (1_200_000, 8),              # clamped: 10 rows per thread
    (40_000, 64),                # J = 2
    (50_001, 24),                # 85 rows per pass, one idle thread, J = 5
    (12_345, 96),                # 21 rows per pass, 4 idle threads, J = 1 although 2C < 256
    (30_001, 200),               # 10 rows per pass, 6 idle threads, 2C >= 256
    (777, 256),
    (5_000, 1024),               # 2 rows per pass
    (60_000, 1024),              # clamped: 59 rows per thread
    (9_000, 2048),               # clamped: 18 rows per thread on one row per pass
] + CFG3
# the exact inputs: j / 4 + a power-of-two offset per channel, |x| <= 48
EXACT_K = 64
OFFSETS = (0.0, 4.0, -8.0, 32.0, -32.0, 1.0, -2.0, 16.0)
EXACT_MAX_X = EXACT_K / 4 + max(abs(o) for o in OFFSETS)


def _case_id(c):
    return f"{c[0]}x{c[1]}"


def _dt(dtype):
    return str(dtype).replace("torch.", "")


@pytest.mark.parametrize("sms", sorted(SM_COUNTS.values()))
def test_geometry_table_reaches_every_branch(sms):
    gs = [bn_geometry(n, C, sms) for n, C in CASES]
    assert {g.rows_per_pass for g in gs} >= {256, 85, 21, 10, 8, 2, 1}
    assert any(g.idle for g in gs)
    # the last CTA's combine: J > 1 (split over threads, then in j order), with fewer CTAs than
    # J and with more; J = 1 (the direct loop) both with 2C >= 256 and with 256 / 2C rounding to 1
    assert any(g.J > 1 and g.grid < g.J for g in gs)
    assert any(g.J > 1 and g.grid > g.J and g.grid % g.J for g in gs)
    assert any(g.J == 1 and 2 * g.C < THREADS for g in gs)
    assert any(2 * g.C >= THREADS for g in gs)
    # unclamped launches sum 8 rows per thread, so the 4-row unroll ends exactly but in the last
    # CTA; clamped ones more, and some end mid-unroll in every CTA
    for g in gs:
        assert g.clamped or g.per_thread == 8
        assert g.grid <= MAX_CTAS and g.last_rows > 0
    assert any(not g.clamped and g.grid > 1 and g.last_rows % g.rows_per_pass for g in gs)
    assert any(g.clamped and g.per_thread % UNROLL for g in gs)
    assert any(g.clamped and g.per_thread % UNROLL == 0 for g in gs)
    assert any(g.apply_grid > MAX_CTAS for g in gs)       # the apply passes are not clamped
    # the cfg3 shapes: all clamped, two of them end mid-unroll in every CTA
    assert [(g.per_thread, g.grid) for g in map(lambda c: bn_geometry(*c, sms), CFG3)] == \
        [(25, 500), (75, 508), (196, 511)]
    # the exact inputs keep every per-thread fp32 partial exact (see _assert_exact_partials)
    for g in gs:
        assert g.per_thread * EXACT_MAX_X ** 2 * 16 < 2 ** 24
        assert 4 * EXACT_MAX_X < 256                     # and are bf16 / fp16 values


# ---- library entry points --------------------------------------------------------------------
def _lib():
    from minkowskiengine_b200 import _lib
    return _lib


def _call(name, *args):
    L = _lib()
    L.check(getattr(L.load(), name)(*args, L.current_stream()))


def _p(t):
    return None if t is None else t.data_ptr()


@pytest.fixture(scope="module")
def ws(cuda):
    """One workspace for every call of this module, as a stream's layers share one."""
    return torch.zeros(int(_lib().load().meb200_bn_workspace_bytes()), dtype=torch.uint8,
                       device=cuda)


def _assert_clean(ws):
    torch.cuda.synchronize()
    nz = int(ws.count_nonzero())
    ws.zero_()
    assert nz == 0, f"the reduction left {nz} nonzero workspace bytes"


def _gen(cuda, *key):
    return torch.Generator(device=cuda).manual_seed(zlib.crc32(repr(key).encode()))


def _exact_x(n, C, dtype, cuda, seed):
    """x = k / 4 + OFFSETS[c % 8], k in [-EXACT_K, EXACT_K]; channel 1 is constant (variance 0)."""
    g = _gen(cuda, "x", n, C, seed)
    k = torch.randint(-EXACT_K, EXACT_K + 1, (n, C), generator=g, device=cuda)
    k[:, 1] = 0
    off = torch.tensor(OFFSETS, dtype=torch.float64, device=cuda).repeat(C // 8)
    x = (k.double() / 4 + off)
    assert torch.equal(x.to(dtype).double(), x)
    return x.to(dtype)


def _assert_exact_partials(geom, terms, quantum, what):
    """Every per-thread fp32 partial over `terms` (multiples of `quantum`) is exact: at most R =
    geom.per_thread terms, so |partial| / quantum <= R · max|term| / quantum < 2^24.  The fp64
    sums of those partials above it are then exact as well."""
    bound = geom.per_thread * float(terms.abs().max()) / quantum
    assert bound < 2 ** 24, f"{what}: fp32 partials of up to {bound:.3g} quanta are not exact"


def _ref_finalize(S1, S2, n, rm0, rv0):
    """float64 restatement of the finalize (numpy, host): mean, invstd, running statistics."""
    S1, S2 = S1.cpu().numpy(), S2.cpu().numpy()
    rm0, rv0 = rm0.double().cpu().numpy(), rv0.double().cpu().numpy()
    mu = S1 / n
    var = np.maximum(S2 / n - mu * mu, 0.0)
    unbiased = var * n / (n - 1) if n > 1 else var
    return dict(mean=mu, invstd=1.0 / np.sqrt(var + EPS),
                running_mean=(1.0 - MOM) * rm0 + MOM * mu,
                running_var=(1.0 - MOM) * rv0 + MOM * unbiased)


def _assert_ulps(got, ref64, what, ulps=1):
    got = got.cpu().numpy()
    r32 = ref64.astype(np.float32)
    err = np.abs(got.astype(np.float64) - r32.astype(np.float64))
    bad = ~(err <= ulps * np.spacing(np.abs(r32)).astype(np.float64))
    assert not bad.any(), (f"{what}: {int(bad.sum())} channels beyond {ulps} fp32 ulp, first "
                           f"{int(np.argmax(bad))}: got {got[bad][0]!r}, float64 {ref64[bad][0]!r}")


def _assert_stats(ref, mean, invstd, running_mean=None, running_var=None):
    m32 = ref["mean"].astype(np.float32)
    got = mean.cpu().numpy()
    assert np.array_equal(got, m32), \
        f"mean: {int((got != m32).sum())} channels differ from fp32(S1 / n)"
    _assert_ulps(invstd, ref["invstd"], "invstd")
    if running_mean is not None:
        _assert_ulps(running_mean, ref["running_mean"], "running_mean")
        _assert_ulps(running_var, ref["running_var"], "running_var")


def _rand_stats(C, cuda, seed):
    g = _gen(cuda, "stats", C, seed)
    rm0 = torch.rand(C, generator=g, device=cuda) * 2 - 1
    rv0 = torch.rand(C, generator=g, device=cuda) + 0.5
    w = torch.rand(C, generator=g, device=cuda) + 0.5
    b = torch.rand(C, generator=g, device=cuda) * 2 - 1
    return rm0, rv0, w, b


def _assert_within(got, ref, bound, what):
    """|got - ref| <= bound element by element; returns the worst ratio |err| / bound."""
    got, ref = got.detach(), ref.detach()
    err = (got.double() - ref.double()).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        j = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(
            f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at flat "
            f"index {j}: got {got.flatten()[j].item()!r}, float64 {ref.flatten()[j].item()!r}, "
            f"|err| {err.flatten()[j].item():.3e} > {bound.flatten()[j].item():.3e}")
    m = bound > 0
    return float((err[m] / bound[m]).max()) if bool(m.any()) else 0.0


def _stored(bound, ref, dtype):
    """A bound on a fp32 result plus its one rounding to the stored dtype."""
    return bound if dtype == torch.float32 else bound + half_ulp(ref.abs() + bound, dtype)


def _y_bound(x, mu, is_, w, b, res, e_mu=0.0, rho=0.0):
    """|y' - y| for y = (x - mu)·is·w + b [+ res] computed as k_bn_apply<T, 0> does, before the
    store: sc = fp32(is·w), sh = fp32(b - fp32(mu·sc)), y = fp32(fmaf(x, sc, sh) [+ res]).  Those
    are at most 5 roundings on terms of A = |x·is·w| + |mu·is·w| + |b| + |res| (6 u·A with one
    spare); the statistics' own errors (mean within e_mu, invstd within the relative rho) add
    |w|·is·(|x - mu|·rho + e_mu·(1 + rho))."""
    A = (x * is_ * w).abs() + (mu * is_ * w).abs() + b.abs() + res.abs()
    stat = w.abs() * is_ * ((x - mu).abs() * rho + e_mu * (1 + rho))
    return stat + 6 * U * (1 + rho) * (A + w.abs() * is_ * e_mu)


def _dx_bound(D, X, K1, K2, isw, rho=0.0, ex=None, ek1=None, ek2=None):
    """|dx' - dx| for dx = (D - K1 - X·K2)·is·w computed as k_bn_apply<T, 1> does, before the
    store: k1 = fp32(K1), k2 = fp32(K2), xhat = fp32(fp32(x - m)·is), fp32((D - k1) - xhat·k2)
    times sc = fp32(is·w).  K1, K2 and xhat as the kernel has them lie within ek1, ek2 and ex of
    the float64 ones (defaults: their roundings alone), invstd within the relative rho.  The
    inner difference takes at most 4 roundings on T = |D| + |K1| + |X·K2| (5 u·T with one
    spare), the scaling 2 and rho."""
    ek1 = (U + 2 * V) * K1.abs() if ek1 is None else ek1
    ek2 = (U + 2 * V) * K2.abs() if ek2 is None else ek2
    ex = 2 * U * (1 + U) * X.abs() if ex is None else ex
    T = D.abs() + K1.abs() + (X * K2).abs()
    inner = ek1 + X.abs() * ek2 + ex * (K2.abs() + ek2) + 5 * U * T
    return isw.abs() * (1 + rho) * (1 + 2 * U) * (inner + T * (rho + 2 * U))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("n,C", CASES, ids=map(_case_id, CASES))
def test_forward_train_statistics_exact(cuda, ws, n, C, dtype):
    """meb200_bn_forward_train: mean bit for bit, invstd and running statistics within one ulp,
    num_batches_tracked + 1, and y from the statistics it returned."""
    geom = bn_geometry(n, C)
    x = _exact_x(n, C, dtype, cuda, 0)
    x64 = x.double()
    _assert_exact_partials(geom, x64, 1 / 4, "x")
    _assert_exact_partials(geom, x64 * x64, 1 / 16, "x^2")
    S1, S2 = x64.sum(0), (x64 * x64).sum(0)           # exact in any order
    rm0, rv0, w, b = _rand_stats(C, cuda, n)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.full((1,), 7, dtype=torch.int64, device=cuda)
    mean = torch.full((C,), float("nan"), device=cuda)
    invstd = torch.full((C,), float("nan"), device=cuda)
    y = torch.empty_like(x)
    L = _lib()
    _call("meb200_bn_forward_train", _p(x), L.dtype_code(dtype), n, C, _p(w), _p(b), None, 0, EPS,
          MOM, _p(rm), _p(rv), _p(nbt), _p(ws), _p(mean), _p(invstd), _p(y))
    _assert_stats(_ref_finalize(S1, S2, n, rm0, rv0), mean, invstd, rm, rv)
    assert int(nbt) == 8
    m, s = mean.double(), invstd.double()
    ref = (x64 - m) * s * w.double() + b.double()
    zero = torch.zeros((), dtype=torch.float64, device=cuda)
    _assert_within(y, ref, _stored(_y_bound(x64, m, s, w.double(), b.double(), zero), ref, dtype),
                   "y")
    _assert_clean(ws)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("n,C", CASES, ids=map(_case_id, CASES))
def test_stats_to_then_finalize_exact(cuda, ws, n, C, dtype):
    """meb200_bn_stats_to, then meb200_bn_finalize on its totals (the path of the NCCL exchange):
    totals bit for bit; finalize from a host count and from a device count."""
    geom = bn_geometry(n, C)
    x = _exact_x(n, C, dtype, cuda, 1)
    x64 = x.double()
    _assert_exact_partials(geom, x64, 1 / 4, "x")
    _assert_exact_partials(geom, x64 * x64, 1 / 16, "x^2")
    sums = torch.full((2 * C,), float("nan"), dtype=torch.float64, device=cuda)
    _call("meb200_bn_stats_to", _p(x), _lib().dtype_code(dtype), n, C, _p(ws), _p(sums))
    S1, S2 = x64.sum(0), (x64 * x64).sum(0)
    assert torch.equal(sums[:C], S1) and torch.equal(sums[C:], S2), "totals differ"
    _assert_clean(ws)
    rm0, rv0, _, _ = _rand_stats(C, cuda, n + 1)
    ref = _ref_finalize(S1, S2, n, rm0, rv0)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd = torch.empty(C, device=cuda), torch.empty(C, device=cuda)
    _call("meb200_bn_finalize", _p(sums), float(n), None, C, EPS, MOM, _p(rm), _p(rv), _p(mean),
          _p(invstd))
    _assert_stats(ref, mean, invstd, rm, rv)
    d_count = torch.tensor([float(n)], dtype=torch.float64, device=cuda)
    mean2, invstd2 = torch.empty(C, device=cuda), torch.empty(C, device=cuda)
    _call("meb200_bn_finalize", _p(sums), 1.0, _p(d_count), C, EPS, MOM, None, None, _p(mean2),
          _p(invstd2))
    assert torch.equal(mean2, mean) and torch.equal(invstd2, invstd)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1.0, 2.0, 3.0, 12_345.0, 800_000.0])
def test_finalize_on_given_sums(cuda, count):
    """meb200_bn_finalize on fp64 totals that are not dyadic (means up to 500, variances from
    1e-3 to 1), and a channel whose totals give a negative variance (clamped to 0)."""
    C = 64
    g = _gen(cuda, "fin", count)
    mu = (torch.rand(C, generator=g, device=cuda, dtype=torch.float64) - 0.5) * \
        10.0 ** torch.arange(C, device=cuda).remainder(4)
    var = torch.rand(C, generator=g, device=cuda, dtype=torch.float64) + 1e-3
    sums = torch.cat([mu * count, (var + mu * mu) * count])
    sums[C + 5] = sums[5] * sums[5] / count * (1 - 1e-12)
    rm0, rv0, _, _ = _rand_stats(C, cuda, int(count))
    ref = _ref_finalize(sums[:C], sums[C:], count, rm0, rv0)
    assert ref["invstd"][5] == 1 / np.sqrt(EPS)
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd = torch.empty(C, device=cuda), torch.empty(C, device=cuda)
    _call("meb200_bn_finalize", _p(sums), count, None, C, EPS, MOM, _p(rm), _p(rv), _p(mean),
          _p(invstd))
    _assert_stats(ref, mean, invstd, rm, rv)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
def test_reductions_of_no_rows(cuda, ws, dtype):
    """n = 0: the totals, and the parameter gradients, are zero (an empty rank's share)."""
    C = 96
    L = _lib()
    x = torch.empty((0, C), dtype=dtype, device=cuda)
    sums = torch.full((2 * C,), float("nan"), dtype=torch.float64, device=cuda)
    _call("meb200_bn_stats_to", _p(x), L.dtype_code(dtype), 0, C, _p(ws), _p(sums))
    assert int(sums.count_nonzero()) == 0
    sums.fill_(float("nan"))
    gw = torch.full((C,), float("nan"), device=cuda)
    gb = torch.full((C,), float("nan"), device=cuda)
    mean, invstd = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    _call("meb200_bn_backward_reduce_to", _p(x), _p(x), None, L.dtype_code(dtype), 0, C, _p(mean),
          _p(invstd), _p(ws), _p(sums), _p(gw), _p(gb))
    assert int(sums.count_nonzero()) == 0 and int(gw.count_nonzero()) == 0
    assert int(gb.count_nonzero()) == 0
    _assert_clean(ws)


def _sign_pattern(n, C, dtype, cuda):
    """y of a fused ReLU layer with a fixed pattern of signs: -1, 0 and +1 (0 masks dy)."""
    r = torch.arange(n, device=cuda).unsqueeze(1)
    c = torch.arange(C, device=cuda).unsqueeze(0)
    return ((r * 7 + c * 5) % 3 - 1).to(dtype)


def _backward_stats(C, cuda):
    """Caller-given mean (the channel's power-of-two offset) and invstd (powers of two)."""
    mean = torch.tensor(OFFSETS, device=cuda).repeat(C // 8)
    invstd = torch.tensor((1.0, 2.0, 0.5, 4.0), device=cuda).repeat(C // 4)
    return mean, invstd


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True], ids=["plain", "ymask"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("n,C", CASES, ids=map(_case_id, CASES))
def test_backward_reduce_exact(cuda, ws, n, C, dtype, masked):
    """meb200_bn_backward_reduce_to on dyadic dy and x and power-of-two statistics: the totals
    are Σdy and Σdy·(x - mean)·invstd bit for bit, the parameter gradients their fp32 roundings."""
    geom = bn_geometry(n, C)
    x = _exact_x(n, C, dtype, cuda, 2)
    g = _gen(cuda, "dy", n, C)
    dy = (torch.randint(-EXACT_K, EXACT_K + 1, (n, C), generator=g, device=cuda).double() / 4)
    dy = dy.to(dtype)
    ymask = _sign_pattern(n, C, dtype, cuda) if masked else None
    mean, invstd = _backward_stats(C, cuda)
    D = dy.double() if ymask is None else torch.where(ymask > 0, dy.double(), 0.0)
    X = (x.double() - mean.double()) * invstd.double()
    _assert_exact_partials(geom, D, 1 / 4, "dy")
    _assert_exact_partials(geom, D * X, 1 / 32, "dy * xhat")     # invstd >= 1/2
    G1, G2 = D.sum(0), (D * X).sum(0)
    sums = torch.full((2 * C,), float("nan"), dtype=torch.float64, device=cuda)
    gw = torch.full((C,), float("nan"), device=cuda)
    gb = torch.full((C,), float("nan"), device=cuda)
    _call("meb200_bn_backward_reduce_to", _p(dy), _p(x), _p(ymask), _lib().dtype_code(dtype), n, C,
          _p(mean), _p(invstd), _p(ws), _p(sums), _p(gw), _p(gb))
    assert torch.equal(sums[:C], G1), "Σdy differs"
    assert torch.equal(sums[C:], G2), "Σdy·xhat differs"
    assert torch.equal(gb, G1.float()) and torch.equal(gw, G2.float())
    _assert_clean(ws)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True], ids=["plain-noaffine", "residual-relu"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("n,C", CASES, ids=map(_case_id, CASES))
def test_apply_forward(cuda, n, C, dtype, fused):
    """meb200_bn_apply_fused on given statistics against y = (x - mean)·invstd·w + b [+ res]
    [ReLU] in float64: plain with a null weight and bias, or affine with residual and ReLU."""
    g = _gen(cuda, "apply", n, C)
    x = (torch.randn(n, C, generator=g, device=cuda) * 3 + 1).to(dtype)
    mean = torch.randn(C, generator=g, device=cuda)
    invstd = torch.rand(C, generator=g, device=cuda) * 2 + 0.1
    w = b = res = None
    if fused:
        w = torch.randn(C, generator=g, device=cuda)
        b = torch.randn(C, generator=g, device=cuda)
        res = torch.randn(n, C, generator=g, device=cuda).to(dtype)
        # elements whose output is exactly zero: x = mean, power-of-two scale, no bias, residual 0
        x[: min(n, 5), :8] = mean[:8].to(dtype)
        mean[:8] = x[0, :8].float()
        invstd[:8] = 2.0
        w[:8] = -0.5
        b[:8] = 0
        res[: min(n, 5), :8] = 0
    y = torch.empty_like(x)
    _call("meb200_bn_apply_fused", _p(x), _lib().dtype_code(dtype), n, C, _p(mean), _p(invstd),
          _p(w), _p(b), _p(res), int(fused), _p(y))
    one = torch.ones((), dtype=torch.float64, device=cuda)
    x64, m, s = x.double(), mean.double(), invstd.double()
    w64 = one if w is None else w.double()
    b64 = one * 0 if b is None else b.double()
    r64 = one * 0 if res is None else res.double()
    ref = (x64 - m) * s * w64 + b64 + r64
    bound = _y_bound(x64, m, s, w64, b64, r64)
    if fused:
        ref = ref.clamp(min=0)          # |relu(a) - relu(b)| <= |a - b|: the bound holds
        assert int(y[: min(n, 5), :8].count_nonzero()) == 0
    _assert_within(y, ref, _stored(bound, ref, dtype), "y")


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True], ids=["plain-noaffine", "ymask-dres"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("n,C", CASES, ids=map(_case_id, CASES))
def test_apply_backward(cuda, n, C, dtype, fused):
    """meb200_bn_backward_apply_fused on given statistics and totals against
    dx = (dy' - G1/n - xhat·G2/n)·invstd·w in float64, dy' = dy where y > 0 (ReLU mask; y = 0
    exactly masks): plain with a null weight and a host count, or with the mask, d_residual (dy'
    exactly) and a device count."""
    g = _gen(cuda, "bwd", n, C)
    dy = torch.randn(n, C, generator=g, device=cuda).to(dtype)
    x = (torch.randn(n, C, generator=g, device=cuda) * 3 + 1).to(dtype)
    mean = torch.randn(C, generator=g, device=cuda)
    invstd = torch.rand(C, generator=g, device=cuda) * 2 + 0.1
    sums = torch.randn(2 * C, generator=g, device=cuda, dtype=torch.float64) * (n ** 0.5)
    w = torch.randn(C, generator=g, device=cuda) if fused else None
    ymask = _sign_pattern(n, C, dtype, cuda) if fused else None
    d_count = torch.tensor([float(n)], dtype=torch.float64, device=cuda) if fused else None
    dx = torch.empty_like(x)
    dres = torch.full_like(x, float("nan")) if fused else None
    _call("meb200_bn_backward_apply_fused", _p(dy), _p(x), _p(ymask), _lib().dtype_code(dtype), n,
          C, _p(mean), _p(invstd), _p(w), _p(sums), 1.0 if fused else float(n), _p(d_count),
          _p(dx), _p(dres))
    D = dy.double() if ymask is None else torch.where(ymask > 0, dy.double(), 0.0)
    if fused:
        assert torch.equal(dres, D.to(dtype)), "d_residual is not the masked dy"
    s = invstd.double()
    X = (x.double() - mean.double()) * s
    K1, K2 = sums[:C] / n, sums[C:] / n
    isw = s if w is None else s * w.double()
    ref = (D - K1 - X * K2) * isw
    _assert_within(dx, ref, _stored(_dx_bound(D, X, K1, K2, isw), ref, dtype), "dx")


# ---- modules against float64 BatchNorm1d, random data -----------------------------------------
def _stat_bounds(x64, geom, training, rm0, rv0):
    """Per channel: how far the statistics the kernels use lie from the float64 ones.

    Training (k_bn_reduce, then the finalize in its last CTA): a thread sums at most
    R = geom.per_thread rows in fp32, S1 by additions and S2 by fmaf(x, x, s), one rounding per
    row; the CTA adds its P = rows_per_pass partials, and the last CTA the B = grid CTAs', in
    fp64.  A recursive sum of m terms errs by at most m·u·Σ|terms| to first order, so
        |S1' - S1| <= e1 = ((R + 1)·u + (P + B + 1)·v)·Σ|x|,   |S2' - S2| <= e2 = (same)·Σx²
    (u = 2^-24, v = 2^-53, one spare rounding each for the second-order terms).  The finalize
    takes mean = S1'/n and var = S2'/n - mean² in fp64 and stores fp32(mean):
        |mean' - μ| <= e_mu  = e1/n + (u + 2v)·|μ|
        |var - σ²|  <= e_var = e2/n + (2|μ| + e1/n)·e1/n + 4v·(Σx²/n + μ²)
    Since Σx²/n = μ² + σ², e_var / σ² carries the factor (μ² + σ²) / σ²: channels far from zero
    lose accuracy with it.  invstd' = fp32((var + eps)^-1/2) lies within the relative rho of the
    float64 value, rho from the interval var ± e_var and two roundings.
    Eval: the mean is the fp32 running mean itself (e_mu = 0); invstd = rsqrt(running_var + eps)
    in fp32: one rounding of the sum and rsqrtf's 2 ulp (4u), rho = 6u with one spare."""
    n = x64.shape[0]
    rm0, rv0 = rm0.double(), rv0.double()
    if not training:
        return dict(mu=rm0, is_=(rv0 + EPS).rsqrt(), e_mu=torch.zeros_like(rm0),
                    rho=torch.full_like(rm0, 6 * U))
    mu = x64.mean(0)
    var = (x64 - mu).square().mean(0)
    k = (geom.per_thread + 1) * U + (geom.rows_per_pass + geom.grid + 1) * V
    e1, e2 = k * x64.abs().sum(0), k * x64.square().sum(0)
    e_mu = e1 / n + (U + 2 * V) * mu.abs()
    e_var = e2 / n + (2 * mu.abs() + e1 / n) * e1 / n + 4 * V * (var + 2 * mu * mu)
    is_ = (var + EPS).rsqrt()
    lo, hi = (var + e_var + EPS).rsqrt(), ((var - e_var).clamp(min=0) + EPS).rsqrt()
    r_iv = torch.maximum(hi / is_ - 1, 1 - lo / is_)
    rho = (r_iv + 2 * V) * (1 + U) + U
    unbiased = var * n / (n - 1)
    rm = (1 - MOM) * rm0 + MOM * mu
    rv = (1 - MOM) * rv0 + MOM * unbiased
    e_rm = MOM * (e1 / n + V * mu.abs()) + 3 * V * ((1 - MOM) * rm0.abs() + MOM * mu.abs())
    e_rv = MOM * (e_var + 3 * V * var) * n / (n - 1) + 3 * V * ((1 - MOM) * rv0 + MOM * unbiased)
    return dict(mu=mu, is_=is_, e_mu=e_mu, rho=rho, var=var, k=k,
                e_rm=e_rm + U * (rm.abs() + e_rm), e_rv=e_rv + U * (rv.abs() + e_rv))


def _grad_bounds(D, x64, st, geom, training):
    """Bounds of the backward reduction's totals as the kernels have them, and of xhat.
    G1 = Σdy' sums like S1; G2 = Σdy'·xhat with xhat = fp32(fp32(x - mean')·invstd') off by
    ex = |x - μ|·is·rho + e_mu·is·(1 + rho) + 2u·|xhat|·(1 + rho), one fmaf per row."""
    mu, is_, e_mu, rho = st["mu"], st["is_"], st["e_mu"], st["rho"]
    X = (x64 - mu) * is_
    ex = ((x64 - mu).abs() * is_ * rho + e_mu * is_) * (1 + rho) + 2 * U * X.abs() * (1 + rho)
    k = (geom.per_thread + 1) * U + (geom.rows_per_pass + geom.grid + 1) * V
    eG1 = k * D.abs().sum(0)
    eG2 = (D.abs() * ex).sum(0) + k * (D.abs() * (X.abs() + ex)).sum(0)
    return X, ex, eG1, eG2


MODULE_CASES = [
    # n, C, dtype, mean/σ of the channels (cycled), affine, training, fused (residual + ReLU)
    pytest.param(40_000, 64, torch.float32, (0, 10, 100), True, True, False, id="f32-offsets"),
    pytest.param(800_000, 32, torch.float32, (0, 10, 100), True, True, True,
                 id="f32-offsets-clamped-fused"),
    pytest.param(40_000, 64, torch.float32, (0, 10, 100), False, False, True,
                 id="f32-offsets-noaffine-eval-fused"),
    pytest.param(12_345, 96, torch.float16, (0, 1), True, True, True, id="f16-fused"),
    pytest.param(12_345, 96, torch.float16, (0, 1), False, True, False, id="f16-noaffine"),
    pytest.param(5_000, 200, torch.float16, (0, 1), True, False, False, id="f16-eval"),
    pytest.param(30_001, 24, torch.bfloat16, (0, 1), False, False, True,
                 id="bf16-noaffine-eval-fused"),
    pytest.param(5_000, 1024, torch.bfloat16, (0, 1), True, True, False, id="bf16-1024"),
] + [pytest.param(n, C, torch.bfloat16, (0, 1), True, True, True, id=f"cfg3-{C}")
     for n, C in CFG3] + [
    pytest.param(800_000, 96, torch.bfloat16, (0, 1), False, True, False, id="cfg3-96-noaffine"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,C,dtype,ratios,affine,training,fused", MODULE_CASES)
def test_module_matches_float64(ME, cuda, n, C, dtype, ratios, affine, training, fused,
                                record_property):
    """MinkowskiBatchNorm / fused_bn_relu against float64 BatchNorm1d on the same rounded inputs:
    y, running statistics, dx, d_residual and the parameter gradients, each element within the
    bound of _stat_bounds / _y_bound / _dx_bound; prints the worst ratio to the bound."""
    g = _gen(cuda, "module", n, C)
    sigma = torch.rand(C, generator=g, device=cuda, dtype=torch.float64) * 1.5 + 0.5
    r = torch.tensor(ratios, dtype=torch.float64, device=cuda).repeat(cdiv(C, len(ratios)))[:C]
    mu = sigma * r * torch.where(torch.arange(C, device=cuda) % 2 == 0, 1.0, -1.0)
    x = (mu + sigma * torch.randn(n, C, generator=g, device=cuda, dtype=torch.float64)).to(dtype)
    res = torch.randn(n, C, generator=g, device=cuda).to(dtype) if fused else None
    dy = torch.randn(n, C, generator=g, device=cuda).to(dtype)
    coords = torch.cat([torch.zeros(n, 1, dtype=torch.int32, device=cuda),
                        torch.arange(n, dtype=torch.int32, device=cuda).unsqueeze(1).repeat(1, 3)],
                       1)
    m = ME.MinkowskiBatchNorm(C, affine=affine).to(cuda)
    with torch.no_grad():
        m.bn.running_mean.copy_(mu + torch.randn(C, generator=g, device=cuda, dtype=torch.float64))
        m.bn.running_var.copy_(sigma.square() * (torch.rand(C, generator=g, device=cuda,
                                                             dtype=torch.float64) + 0.5))
        if affine:
            m.bn.weight.uniform_(0.5, 1.5, generator=g)
            m.bn.bias.uniform_(-1, 1, generator=g)
    ref = torch.nn.BatchNorm1d(C, eps=EPS, momentum=MOM, affine=affine).to(cuda, torch.float64)
    ref.load_state_dict(m.bn.state_dict())
    rm0, rv0 = m.bn.running_mean.clone(), m.bn.running_var.clone()
    m.train(training)
    ref.train(training)

    xs = ME.SparseTensor(x.clone().requires_grad_(True), coords)
    if fused:
        rs = ME.SparseTensor(res.clone().requires_grad_(True),
                             coordinate_map_key=xs.coordinate_map_key,
                             coordinate_manager=xs.coordinate_manager)
        out = ME.fused_bn_relu(m, xs, rs)
    else:
        out = m(xs)
    y = out.F
    y.backward(dy)

    x64 = x.double().requires_grad_(True)
    r64 = res.double() if fused else torch.zeros((), dtype=torch.float64, device=cuda)
    z = ref(x64) + r64
    geom = bn_geometry(n, C)
    st = _stat_bounds(x64.detach(), geom, training, rm0, rv0)
    w64 = ref.weight.detach() if affine else torch.ones((), dtype=torch.float64, device=cuda)
    b64 = ref.bias.detach() if affine else torch.zeros((), dtype=torch.float64, device=cuda)
    x0 = x64.detach()
    yb = _y_bound(x0, st["mu"], st["is_"], w64, b64, r64, st["e_mu"], st["rho"])
    ratios_seen = {}
    zd = z.detach()
    yref = zd.clamp(min=0) if fused else zd
    ratios_seen["y"] = _assert_within(y, yref, _stored(yb, yref, dtype), "y")
    mask = None
    if fused:
        # the ReLU mask backward uses is the kernel's: where it differs from float64's, the
        # pre-activation lies within the forward bound of zero
        mask = y.detach() > 0
        flip = mask != (zd > 0)
        assert bool((zd[flip].abs() <= yb[flip]).all()), "a ReLU decision beyond the bound"
    if training:
        ratios_seen["running_mean"] = _assert_within(m.bn.running_mean, ref.running_mean,
                                                     st["e_rm"], "running_mean")
        ratios_seen["running_var"] = _assert_within(m.bn.running_var, ref.running_var,
                                                    st["e_rv"], "running_var")
        assert int(m.bn.num_batches_tracked) == 1
    else:
        assert torch.equal(m.bn.running_mean, rm0) and torch.equal(m.bn.running_var, rv0)
        assert int(m.bn.num_batches_tracked) == 0

    D = dy.double() if mask is None else torch.where(mask, dy.double(), 0.0)
    z.backward(D)
    if fused:
        assert torch.equal(rs.F.grad, D.to(dtype)), "d_residual is not the masked dy"
    X, ex, eG1, eG2 = _grad_bounds(D, x0, st, geom, training)
    G1, G2 = D.sum(0), (D * X).sum(0)
    if training:
        K1, K2 = G1 / n, G2 / n
        ek1 = eG1 / n + (U + 2 * V) * (K1.abs() + eG1 / n)
        ek2 = eG2 / n + (U + 2 * V) * (K2.abs() + eG2 / n)
    else:                               # the running statistics are constants: dx = dy'·is·w
        K1 = K2 = ek1 = ek2 = torch.zeros_like(G1)
    dxb = _dx_bound(D, X, K1, K2, st["is_"] * w64, st["rho"], ex, ek1, ek2)
    ratios_seen["dx"] = _assert_within(xs.F.grad, x64.grad, _stored(dxb, x64.grad, dtype), "dx")
    if affine:
        assert m.bn.weight.grad.dtype == m.bn.weight.dtype == torch.float32
        ratios_seen["grad_bias"] = _assert_within(m.bn.bias.grad, ref.bias.grad,
                                                  eG1 + U * (G1.abs() + eG1), "grad_bias")
        ratios_seen["grad_weight"] = _assert_within(m.bn.weight.grad, ref.weight.grad,
                                                    eG2 + U * (G2.abs() + eG2), "grad_weight")
    worst = max(ratios_seen.values())
    record_property("worst_ratio_to_bound", worst)
    print(f"[bn fp64] {n}x{C} {_dt(dtype)} mean/σ {ratios} R={geom.per_thread}: " +
          ", ".join(f"{k} {v:.3g}" for k, v in ratios_seen.items()))


@pytest.mark.gpu
def test_eval_backward_uses_its_forward_statistics(ME, cuda):
    """Eval forward, then a training forward of the same module (which moves the running
    statistics), then the backward of the first output: dx and the parameter gradients are those
    of the statistics the first forward used."""
    n, C = 5_000, 64
    g = _gen(cuda, "eval-then-train", n, C)
    x1 = (torch.randn(n, C, generator=g, device=cuda) * 2 + 3)
    x2 = (torch.randn(n, C, generator=g, device=cuda) * 3 - 5)
    dy = torch.randn(n, C, generator=g, device=cuda)
    coords = torch.cat([torch.zeros(n, 1, dtype=torch.int32, device=cuda),
                        torch.arange(n, dtype=torch.int32, device=cuda).unsqueeze(1).repeat(1, 3)],
                       1)
    m = ME.MinkowskiBatchNorm(C).to(cuda)
    with torch.no_grad():
        m.bn.weight.uniform_(0.5, 1.5, generator=g)
        m.bn.bias.uniform_(-1, 1, generator=g)
        m.bn.running_mean.uniform_(2, 4, generator=g)
        m.bn.running_var.uniform_(3, 5, generator=g)
    rm0, rv0 = m.bn.running_mean.clone(), m.bn.running_var.clone()
    m.eval()
    s1 = ME.SparseTensor(x1.clone().requires_grad_(True), coords)
    y1 = m(s1)
    m.train()
    m(ME.SparseTensor(x2, coords))
    assert not torch.equal(m.bn.running_mean, rm0)
    y1.F.backward(dy)

    x64, D = x1.double(), dy.double()
    is_ = (rv0.double() + EPS).rsqrt()
    w64 = m.bn.weight.detach().double()
    X = (x64 - rm0.double()) * is_
    ref_dx = D * is_ * w64
    st = dict(mu=rm0.double(), is_=is_, e_mu=torch.zeros_like(is_), rho=torch.full_like(is_, 6 * U))
    geom = bn_geometry(n, C)
    _, ex, eG1, eG2 = _grad_bounds(D, x64, st, geom, False)
    zero = torch.zeros_like(is_)
    _assert_within(s1.F.grad, ref_dx, _dx_bound(D, X, zero, zero, is_ * w64, 6 * U, ex, zero, zero),
                   "dx")
    G1, G2 = D.sum(0), (D * X).sum(0)
    _assert_within(m.bn.weight.grad, G2, eG2 + U * (G2.abs() + eG2), "grad_weight")
    _assert_within(m.bn.bias.grad, G1, eG1 + U * (G1.abs() + eG1), "grad_bias")
