"""libmeb200's per-cloud kernels (csrc/global.cu: the grouping, the segmented reduction and the
broadcasts) against numpy and float64, over every launch geometry the reduction takes, in fp32,
bf16 and fp16.

* The launch geometry of seg_reduce_t / seg_reduce_launch is restated in Python (seg_geometry);
  a CPU test asserts that the cases below reach every branch of it.
* The grouping (row_seg, order, seg_start, tile_start) must equal numpy's stable counting sort.
* The reduction runs through backend._segment_reduce on real groupings.  On exactly summable
  inputs (see EXACT_RULE) SUM must be the float64 sum bit for bit, AVG fp32(S) / fp32(cnt), MAX
  and its argmax the oracle's (lowest row on ties).  On random inputs every element lies within
  gamma_D * sum|x| of float64, D the rounding depth of the geometry.
* Each broadcast is one fp32 operation and one rounding: bit for bit against numpy.
* The modules (the nine global poolings, the broadcasts, the instance norm) against
  tests/global_oracle.py in float64, each element within a bound derived from their arithmetic."""
import zlib
from dataclasses import dataclass
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import global_oracle as GO
from helpers import half_ulp, one_rounding_bound, one_rounding_ratio

THREADS = 256                    # threads of a k_seg_reduce_tiles CTA
TILE = 512                       # MEB200_SEGMENT_TILE_ROWS: rows per reduction tile
GROUP_TILE = 1024                # kGroupTile: rows per counting-sort tile
SCAN = 1024                      # k_group_scan: counts per iteration of the carry
MAX_B = 12288                    # kMaxSegments
DEFAULT_SMEM = 48 * 1024         # dynamic shared memory a kernel gets without opting in
SUM, AVG, MAX = 0, 1, 2          # MEB200_SEG_*
ADD, MUL, COPY, MAXGRAD = 0, 1, 2, 3   # MEB200_BCAST_*
U = 2.0 ** -24                   # unit roundoff of fp32
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
ITEMSIZE = {torch.float32: 4, torch.bfloat16: 2, torch.float16: 2}


def cdiv(a, b):
    return -(-a // b)


def gamma(d):
    """gamma_d = d·u / (1 - d·u): the relative error of d fp32 roundings in a row."""
    return d * U / (1 - d * U)


def _dt(dtype):
    return str(dtype).replace("torch.", "")


@dataclass(frozen=True)
class SegGeom:
    rows: int                    # rows of the segment
    C: int
    V: int                       # channels per thread and access
    tpr: int                     # threads per row
    rp: int                      # row lanes of the CTA
    col_iters: int               # column vectors one thread loops over
    tiles: int                   # reduction tiles of the segment
    lane_rows: int               # rows of the busiest lane (in a full tile when tiles > 1)
    last_tile_rows: int
    last_lane_rows: int          # rows of the busiest lane of the last tile
    smem: int                    # dynamic shared memory of the launch, bytes

    def depth(self, prod=False, avg=False):
        """Roundings one term of an output element meets at most: its lane's additions, the
        lane combine (rp - 1 additions), the tile sums of the finish, and one each for the
        product (b != NULL) and the AVG division."""
        return self.lane_rows + self.rp - 1 + self.tiles + int(prod) + int(avg)


def seg_geometry(rows, C, dtype=torch.float32, aligned=True, mode=SUM):
    """What seg_reduce_t / seg_reduce_launch choose for a segment of `rows` rows of [*, C]
    features in `dtype` (`aligned`: the buffers are 4 * itemsize aligned)."""
    V = 4 if C % 4 == 0 and aligned else 1
    CV = C // V
    tpr = 1
    while tpr * 2 <= CV and tpr * 2 <= THREADS:
        tpr *= 2
    rp = THREADS // tpr
    tiles = cdiv(rows, TILE)
    last = rows - (tiles - 1) * TILE if rows else 0
    return SegGeom(rows=rows, C=C, V=V, tpr=tpr, rp=rp, col_iters=cdiv(CV, tpr), tiles=tiles,
                   lane_rows=cdiv(min(rows, TILE), rp), last_tile_rows=last,
                   last_lane_rows=cdiv(last, rp), smem=rp * C * (8 if mode == MAX else 4))


# ---- cases -----------------------------------------------------------------------------------------
# Segment sizes per cloud (0: a cloud of the origin map without rows in this map).
LAYOUTS = {
    "edges": [1, 511, 0, 512, 513, 2],       # 1539 rows: every tile edge, crosses a group tile
    "tiles": [3000, 0, 7, 5121],             # 6 and 11 tiles, the last of one row
    "long": [102_437],                       # one cloud over 201 tiles
    "clouds": None,                          # MAX_B clouds of 0..3 rows: the scan's carry
}


def layout_sizes(name):
    s = LAYOUTS[name]
    if s is None:
        s = np.random.default_rng(5).integers(0, 4, MAX_B).tolist()
        s[0], s[-1] = 3, 1
    return s


def layout_rows(name):
    """Cloud (segment) of every row, rows shuffled (seeded)."""
    sizes = layout_sizes(name)
    seg = np.repeat(np.arange(len(sizes)), sizes)
    np.random.default_rng(zlib.crc32(name.encode())).shuffle(seg)
    return seg


# (C, layout, aligned): every tpr, V = 1 and 4, V = 1 with C % 4 == 0 from a misaligned buffer
CASES = [
    (1, "edges", True), (1, "tiles", True), (1, "long", True), (1, "clouds", True),
    (3, "edges", True),
    (4, "edges", True), (4, "tiles", True), (4, "edges", False),
    (5, "edges", True), (5, "tiles", True),
    (12, "edges", True), (12, "long", True), (12, "edges", False),
    (64, "edges", True), (64, "tiles", True), (64, "clouds", True), (64, "tiles", False),
    (96, "tiles", True), (96, "long", True),
    (128, "edges", True),
    (255, "edges", True), (255, "tiles", True),
    (1024, "edges", True), (1024, "tiles", True), (1024, "edges", False),
    (1028, "edges", True),
    (2049, "edges", True),
    (6144, "edges", True),                   # MAX: 48 KB of shared memory exactly
    (6148, "edges", True), (8191, "edges", True), (8192, "edges", True),   # above 48 KB
    (8192, "edges", False),
]


def _case_id(c):
    return f"C{c[0]}-{c[1]}" + ("" if c[2] else "-misaligned")


def _geoms(C, layout, dtype, aligned, mode=SUM):
    return [seg_geometry(m, C, dtype, aligned, mode) for m in layout_sizes(layout) if m]


# Exact inputs: x = j / 4 and y = k / 4 with |j|, |k| <= EXACT_J.  Every partial sum the kernels
# form (in a lane, in the combine, in the finish) is a sum of a subset of one cloud's terms: a
# multiple of the quantum (1/4 for x, 1/16 for x·y) no larger than the cloud's sum of |terms|.
# It is exact in fp32 when that sum is below 2^24 quanta, which _assert_exact checks per case;
# the values are bf16 and fp16 values as well.
EXACT_J = 3
EXACT_RULE = "rows · EXACT_J^2 < 2^24 for x·y / (1/16), rows · EXACT_J < 2^24 for x / (1/4)"


def test_geometry_table_reaches_every_branch():
    seen = []
    for C, layout, aligned in CASES:
        for dtype in DTYPES:
            for mode in (SUM, MAX):
                seen += [(dtype, aligned, mode, g) for g in _geoms(C, layout, dtype, aligned, mode)]
    for dtype in DTYPES:
        assert {g.V for d, _, _, g in seen if d == dtype} == {1, 4}
    assert any(g.V == 1 and g.C % 4 == 0 and not a for _, a, _, g in seen)
    assert {g.tpr for *_, g in seen} == {1 << i for i in range(9)}
    assert any(g.col_iters > 1 and g.V == 4 for *_, g in seen)
    assert any(g.col_iters > 1 and g.V == 1 for *_, g in seen)
    assert any(g.rp == 1 for *_, g in seen)
    assert any(g.tiles > 1 and g.last_tile_rows < g.rp for *_, g in seen)
    assert any(g.tiles == 1 and g.rows < g.rp for *_, g in seen)
    sizes = {g.rows for *_, g in seen}
    assert {1, 511, 512, 513} <= sizes
    assert max(g.tiles for *_, g in seen) > 200
    # MAX on one row lane: 8 C bytes, 48 KB exactly at C = 6144, above it at C > 6144
    max_smem = {g.smem for _, _, m, g in seen if m == MAX}
    assert DEFAULT_SMEM in max_smem and max(max_smem) == 8 * 8192
    assert all(g.smem <= DEFAULT_SMEM for _, _, m, g in seen if m == SUM)
    # depths: from 2 + 255 + tiles at rp = 256 to 512 + tiles at rp = 1
    assert any(g.rp == 256 and g.depth() == 2 + 255 + g.tiles for *_, g in seen)
    assert any(g.rp == 1 and g.depth() == 512 + g.tiles for *_, g in seen)
    # the grouping: segments crossing group tiles, a scan over more than one carry, B = MAX_B
    for name in LAYOUTS:
        seg = layout_rows(name)
        B = len(layout_sizes(name))
        nt = cdiv(len(seg), GROUP_TILE)
        crossing = [s for s in range(min(B, 8))
                    if len(np.unique(np.nonzero(seg == s)[0] // GROUP_TILE)) > 1]
        if name in ("edges", "tiles", "long"):
            assert nt > 1 and crossing, name
    assert cdiv(len(layout_rows("clouds")), GROUP_TILE) * MAX_B > 8 * SCAN
    assert len(layout_sizes("clouds")) == MAX_B and 0 in layout_sizes("clouds")
    # the exact inputs stay exact at every case's largest cloud
    assert max(max(layout_sizes(n)) for n in LAYOUTS) * EXACT_J ** 2 < 2 ** 24


# ---- GPU helpers -----------------------------------------------------------------------------------
def _gen(cuda, *key):
    return torch.Generator(device=cuda).manual_seed(zlib.crc32(repr(key).encode()))


def _batch_of(s):
    """Batch index of cloud s: strictly ascending, with gaps."""
    return 3 * s + s % 3


def _coords(seg):
    """Distinct coordinates, one row per entry of seg (batch = _batch_of(seg))."""
    i = np.zeros(len(seg), np.int64)
    for s in np.unique(seg):
        m = seg == s
        i[m] = np.arange(int(m.sum()))
    return np.stack([_batch_of(seg), i % 64, (i // 64) % 64, i // 4096], 1).astype(np.int32)


_GROUPINGS = {}


def _grouping(ME, cuda, layout):
    """(manager, key, grouping, seg) of `layout`: the origin map holds every cloud of the layout
    (one row each, from a map inserted first), so the empty ones are empty segments."""
    if layout not in _GROUPINGS:
        sizes = layout_sizes(layout)
        seg = layout_rows(layout)
        mgr = ME.CoordinateManager(D=3)
        base = np.zeros((len(sizes), 4), np.int32)
        base[:, 0] = _batch_of(np.arange(len(sizes)))
        mgr.insert_and_map(torch.as_tensor(base).to(cuda), 1, "clouds")
        key, _ = mgr.insert_and_map(torch.as_tensor(_coords(seg)).to(cuda), 1, "rows")
        assert torch.equal(mgr.get_coordinates(key).cpu(), torch.as_tensor(_coords(seg)))
        grp = mgr._manager._origin_grouping(key)
        _GROUPINGS[layout] = (mgr, key, grp, seg)
    return _GROUPINGS[layout]


def _expected_grouping(seg, B):
    cnt = np.bincount(seg, minlength=B)
    seg_start = np.concatenate([[0], np.cumsum(cnt)])
    tile_start = np.concatenate([[0], np.cumsum(-(-cnt // TILE))])
    return np.argsort(seg, kind="stable"), seg_start, tile_start


def _assert_grouping(grp, seg, B):
    order, seg_start, tile_start = _expected_grouping(seg, B)
    assert grp.B == B and grp.n == len(seg)
    assert np.array_equal(grp.row_seg.cpu().numpy(), seg), "row_seg"
    assert np.array_equal(grp.seg_start.cpu().numpy(), seg_start), "seg_start"
    assert np.array_equal(grp.tile_start.cpu().numpy(), tile_start), "tile_start"
    got = grp.order.cpu().numpy()
    bad = np.nonzero(got != order)[0]
    assert len(bad) == 0, f"order differs at {len(bad)} positions, first {bad[:4]}"


def _features(n, C, dtype, cuda, aligned, fill):
    """[n, C] contiguous features in `dtype`; misaligned: the storage starts one element early,
    so the data pointer is not 4 * itemsize aligned."""
    buf = torch.empty(n * C + 1, dtype=dtype, device=cuda)
    t = (buf[1:] if not aligned else buf[:-1]).view(n, C)
    t.copy_(fill)
    assert (t.data_ptr() % (4 * ITEMSIZE[dtype]) == 0) == aligned or C % 4 != 0
    return t


def _seg_sums(v, seg, B):
    """float64 [B, C] sums of the rows of each segment (exact for the exact inputs)."""
    o = np.argsort(seg, kind="stable")
    cnt = np.bincount(seg, minlength=B)
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    out = np.zeros((B, v.shape[1]), np.float64)
    nz = cnt > 0
    if nz.any():
        out[nz] = np.add.reduceat(v[o], starts[nz], axis=0)
    return out, cnt


def _seg_max(v, seg, B):
    """float64 [B, C] maxima and int32 flat argmax row*C + c, lowest row on ties (-1: empty)."""
    n, C = v.shape
    o = np.argsort(seg, kind="stable")
    cnt = np.bincount(seg, minlength=B)
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    nz = cnt > 0
    out = np.zeros((B, C), np.float64)
    idx = np.full((B, C), -1, np.int64)
    vs = v[o]
    out[nz] = np.maximum.reduceat(vs, starts[nz], axis=0)
    seg_sorted = seg[o]
    pos = np.where(vs == out[seg_sorted], np.arange(n)[:, None], n)
    first = np.minimum.reduceat(pos, starts[nz], axis=0)
    idx[nz] = o[first] * C + np.arange(C)
    return out, idx.astype(np.int32)


def _reduce(ME, x, grp, mode, y=None):
    aux = torch.full((grp.B, x.shape[1]) if mode == MAX else (grp.B,), -7,
                     dtype=torch.int32 if mode == MAX else torch.float32, device=x.device)
    out = ME.backend._segment_reduce(x, grp, mode, b=y, aux=aux)
    return out.cpu().numpy(), aux.cpu().numpy()


# ---- grouping --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_origin_grouping_matches_numpy(ME, cuda, layout):
    """row_seg, order, seg_start and tile_start of meb200_origin_group, exactly, on shuffled rows
    with empty clouds between non-empty ones, one-row clouds and B = MAX_B."""
    _, _, grp, seg = _grouping(ME, cuda, layout)
    _assert_grouping(grp, seg, len(layout_sizes(layout)))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2047, 3072, 4097])
@pytest.mark.parametrize("B", [1, 7, MAX_B])
def test_grouping_around_group_tiles(ME, cuda, n, B):
    """Sparse map and tensor field over n rows around multiples of 1024, B clouds (those that get
    no row stay empty segments): the same grouping from both, exactly numpy's."""
    rng = np.random.default_rng(n * 31 + B)
    seg = rng.integers(0, B, n) if B > 1 else np.zeros(n, np.int64)
    if B > 2 and n > 2:
        seg[seg == B // 2] = B // 2 + 1          # an empty cloud between non-empty ones
    mgr = ME.CoordinateManager(D=3)
    base = np.zeros((B, 4), np.int32)
    base[:, 0] = _batch_of(np.arange(B))
    mgr.insert_and_map(torch.as_tensor(base).to(cuda), 1, "clouds")
    coords = _coords(seg)
    key, _ = mgr.insert_and_map(torch.as_tensor(coords).to(cuda), 1, "rows")
    _assert_grouping(mgr._manager._origin_grouping(key), seg, B)
    # the same rows as float points (batch values lroundf rounds to the batch index)
    pts = coords.astype(np.float32)
    pts[:, 0] += rng.choice([-0.49, 0.0, 0.3], n).astype(np.float32)
    tf = ME.TensorField(torch.ones(n, 1, device=cuda), torch.as_tensor(pts).to(cuda),
                        coordinate_manager=mgr)
    _assert_grouping(mgr._manager._field_grouping(tf.coordinate_map_key), seg, B)


# ---- segmented reduction, exact inputs ---------------------------------------------------------------
def _exact(n, C, cuda, seed):
    g = _gen(cuda, "exact", n, C, seed)
    # a handful of values: the maximum repeats in most lanes and tiles of a cloud
    return torch.randint(-EXACT_J, EXACT_J + 1, (n, C), generator=g, device=cuda).double() / 4


def _assert_exact(v, seg, B, quantum, what):
    A, _ = _seg_sums(np.abs(v), seg, B)
    assert A.max() / quantum < 2 ** 24, f"{what}: partial sums are not exact in fp32 ({EXACT_RULE})"


def _assert_equal(got, want, what):
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        j = np.argwhere(bad)[0]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, first at {tuple(j)}: "
                             f"got {got[tuple(j)]!r}, want {want[tuple(j)]!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("C,layout,aligned", CASES, ids=map(_case_id, CASES))
def test_segment_reduce_exact(ME, cuda, C, layout, aligned, dtype):
    """SUM bit for bit, AVG = fp32(S) / fp32(cnt), MAX and argmax the oracle's, the counts in
    aux; for a and for a·b."""
    _, _, grp, seg = _grouping(ME, cuda, layout)
    B, n = grp.B, grp.n
    x64, y64 = _exact(n, C, cuda, 0), _exact(n, C, cuda, 1)
    x = _features(n, C, dtype, cuda, aligned, x64.to(dtype))
    y = _features(n, C, dtype, cuda, aligned, y64.to(dtype))
    assert torch.equal(x.double(), x64) and torch.equal(y.double(), y64)
    xv, yv = x64.cpu().numpy(), y64.cpu().numpy()
    _assert_exact(xv, seg, B, 1 / 4, "x")
    _assert_exact(xv * yv, seg, B, 1 / 16, "x·y")
    for prod in (False, True):
        v = xv * yv if prod else xv
        S, cnt = _seg_sums(v, seg, B)
        what = ("x·y " if prod else "x ") + _dt(dtype)
        out, aux = _reduce(ME, x, grp, SUM, y if prod else None)
        _assert_equal(out, S.astype(np.float32), "SUM " + what)
        _assert_equal(aux, cnt.astype(np.float32), "SUM counts")
        out, aux = _reduce(ME, x, grp, AVG, y if prod else None)
        avg = np.where(cnt[:, None] > 0,
                       S.astype(np.float32) / np.maximum(cnt, 1).astype(np.float32)[:, None], 0)
        _assert_equal(out, avg.astype(np.float32), "AVG " + what)
        _assert_equal(aux, cnt.astype(np.float32), "AVG counts")
    m, idx = _seg_max(xv, seg, B)
    out, aux = _reduce(ME, x, grp, MAX)
    _assert_equal(out, m.astype(np.float32), "MAX " + _dt(dtype))
    _assert_equal(aux, idx, "argmax " + _dt(dtype))


# ---- segmented reduction, random inputs --------------------------------------------------------------
def _seg_bound(geoms_by_seg, B, prod, avg):
    """acc for helpers.one_rounding_bound per segment: gamma_D / 2^-20 (0 for an empty one)."""
    acc = np.zeros(B)
    for s, g in geoms_by_seg.items():
        acc[s] = gamma(g.depth(prod, avg)) * 2.0 ** 20
    return acc


# the widest cases (C >= 6144, where the numpy oracle dominates the time) in fp32 only
RANDOM_CASES = [pytest.param(*c, d, id=f"{_case_id(c)}-{_dt(d)}") for c in CASES for d in DTYPES
                if c[0] < 6144 or d == torch.float32]


@pytest.mark.gpu
@pytest.mark.parametrize("C,layout,aligned,dtype", RANDOM_CASES)
def test_segment_reduce_random(ME, cuda, C, layout, aligned, dtype, record_property):
    """Every element of SUM / AVG (of a and of a·b) within gamma_D · sum|terms| of float64, D the
    depth of its cloud's geometry (one more for the product and for the division); MAX exact."""
    _, _, grp, seg = _grouping(ME, cuda, layout)
    B, n = grp.B, grp.n
    g = _gen(cuda, "random", n, C)
    # mostly positive terms: the rounding errors of a cloud's sum add up instead of cancelling
    x = _features(n, C, dtype, cuda, aligned, (torch.rand(n, C, generator=g, device=cuda) * 2 -
                                               0.25).to(dtype))
    y = _features(n, C, dtype, cuda, aligned, (torch.rand(n, C, generator=g, device=cuda) + 0.5)
                  .to(dtype))
    xv, yv = x.double().cpu().numpy(), y.double().cpu().numpy()
    sizes = layout_sizes(layout)
    geoms = {s: seg_geometry(m, C, dtype, aligned) for s, m in enumerate(sizes) if m}
    ratios = {}
    for prod in (False, True):
        v = xv * yv if prod else xv
        S, cnt = _seg_sums(v, seg, B)
        A, _ = _seg_sums(np.abs(v), seg, B)
        for mode in (SUM, AVG):
            out, _ = _reduce(ME, x, grp, mode, y if prod else None)
            div = np.maximum(cnt, 1)[:, None] if mode == AVG else 1
            acc = torch.as_tensor(_seg_bound(geoms, B, prod, mode == AVG))[:, None]
            ref, Ad = torch.as_tensor(S / div), torch.as_tensor(A / div)
            bound = one_rounding_bound(ref, Ad * acc, torch.float32)
            got = torch.as_tensor(out)
            err = (got.double() - ref).abs()
            bad = ~(err <= bound)
            assert not bool(bad.any()), (
                f"{'AVG' if mode == AVG else 'SUM'}{' x·y' if prod else ''}: {int(bad.sum())} "
                f"elements beyond gamma_D·A, first {torch.nonzero(bad)[0].tolist()}")
            ratios[("avg" if mode == AVG else "sum") + ("-prod" if prod else "")] = \
                one_rounding_ratio(got, ref, Ad * acc)
    m, idx = _seg_max(xv, seg, B)
    out, aux = _reduce(ME, x, grp, MAX)
    _assert_equal(out, m.astype(np.float32), "MAX")
    _assert_equal(aux, idx, "argmax")
    worst = max(ratios.values())
    record_property("worst_ratio_to_bound", worst)
    g0 = max(geoms.values(), key=lambda t: t.depth())
    print(f"[global fp64] C={C} {layout} {_dt(dtype)} V={g0.V} tpr={g0.tpr} rp={g0.rp} "
          f"D<={g0.depth()}: " + ", ".join(f"{k} {r:.3g}" for k, r in ratios.items()))


# ---- broadcast -----------------------------------------------------------------------------------
def _to_out(v32, dtype):
    """A float32 numpy result rounded once to `dtype` (round to nearest even)."""
    return torch.from_numpy(np.ascontiguousarray(v32, np.float32)).to(dtype)


def _bcast_grouping(ME, cuda):
    """The 'edges' grouping's row_seg with some rows outside every segment (-1)."""
    _, _, grp, seg = _grouping(ME, cuda, "edges")
    rs = grp.row_seg.clone()
    rs[::7] = -1
    return SimpleNamespace(row_seg=rs, B=grp.B, n=grp.n), np.where(np.arange(grp.n) % 7 == 0,
                                                                    -1, seg)


BCAST_CASES = [(64, True), (64, False), (5, True)]     # V = 4, V = 1 from x's alignment, C % 4


@pytest.mark.gpu
@pytest.mark.parametrize("out_f32", [False, True], ids=["out-dtype", "out-f32"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("C,aligned", BCAST_CASES, ids=[f"C{c}-{'al' if a else 'mis'}"
                                                        for c, a in BCAST_CASES])
def test_broadcast_bitwise(ME, cuda, C, aligned, dtype, out_f32):
    """ADD, MUL, COPY and MAXGRAD: the fp32 operation rounded once to the output dtype, bit for
    bit; rows with row_seg -1 are zero."""
    grp, seg = _bcast_grouping(ME, cuda)
    B, n = grp.B, grp.n
    g = _gen(cuda, "bcast", C, aligned)
    x = _features(n, C, dtype, cuda, aligned, torch.randn(n, C, generator=g, device=cuda)
                  .to(dtype))
    gl = torch.randn(B, C, generator=g, device=cuda)
    # argmax: a row of the cloud (or -1) per (cloud, channel)
    rows_of = [np.nonzero(seg == s)[0] for s in range(B)]
    rng = np.random.default_rng(C)
    am = np.full((B, C), -1, np.int64)
    for s, r in enumerate(rows_of):
        if len(r):
            pick = r[rng.integers(0, len(r), C)]
            am[s] = np.where(rng.random(C) < 0.9, pick * C + np.arange(C), -1)
    argmax = torch.as_tensor(am.astype(np.int32)).to(cuda)
    out_dtype = torch.float32 if out_f32 else dtype
    xv = x.float().cpu().numpy()
    gv = gl.cpu().numpy()
    inside = seg >= 0
    gs = np.where(inside[:, None], gv[np.maximum(seg, 0)], np.float32(0))
    want = {ADD: np.where(inside[:, None], xv + gs, 0), MUL: np.where(inside[:, None], xv * gs, 0),
            COPY: gs}
    mg = np.zeros((n, C), np.float32).reshape(-1)
    ok = am.reshape(-1) >= 0
    mg[am.reshape(-1)[ok]] = gv.reshape(-1)[ok]
    want[MAXGRAD] = np.where(inside[:, None], mg.reshape(n, C), 0)
    bc = ME.backend._broadcast
    for op in (ADD, MUL, COPY, MAXGRAD):
        if op in (ADD, MUL):
            got = bc(x, gl, grp, op, out_dtype)
        else:
            got = bc(None, gl, grp, op, out_dtype, argmax=argmax if op == MAXGRAD else None,
                     n=n, C=C)
        w = _to_out(want[op].astype(np.float32), out_dtype)
        assert got.dtype == out_dtype
        assert torch.equal(got.cpu(), w), f"op {op}: {int((got.cpu() != w).sum())} differ"
        assert int(got[::7].count_nonzero()) == 0


FMA_CASES = [(zh, k) for zh in (False, True) for k in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("zh,k", FMA_CASES, ids=[f"{'zh' if a else 'nozh'}-{'k' if b else 'nok'}"
                                                 for a, b in FMA_CASES])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("C,aligned", BCAST_CASES, ids=[f"C{c}-{'al' if a else 'mis'}"
                                                        for c, a in BCAST_CASES])
def test_broadcast_fma(ME, cuda, C, aligned, dtype, zh, k):
    """out = x·g[s] + z·h[s] + k[s]: on dyadic inputs (every step exact) the exact value rounded
    once, bit for bit; on random inputs within gamma_3 of sum of |terms| before the store and half
    an ulp of the dtype after it; zero where row_seg is -1."""
    grp, seg = _bcast_grouping(ME, cuda)
    B, n = grp.B, grp.n
    inside = (seg >= 0)[:, None]
    s0 = np.maximum(seg, 0)
    for exact in (True, False):
        g = _gen(cuda, "fma", C, aligned, exact)

        def rnd(*shape, scale=1.0):
            if exact:   # j / 8 with |j| <= 16: products j·k / 64 and their sums stay exact
                return torch.randint(-16, 17, shape, generator=g, device=cuda).float() / 8
            return torch.randn(*shape, generator=g, device=cuda) * scale

        x = _features(n, C, dtype, cuda, aligned, rnd(n, C).to(dtype))
        z = _features(n, C, dtype, cuda, aligned, rnd(n, C).to(dtype)) if zh else None
        gl = rnd(B, C)
        h = rnd(B, C) if zh else None
        kk = rnd(B, C, scale=4.0) if k else None
        got = ME.backend._broadcast_fma(x, gl, grp, z=z, h32=h, k32=kk)
        X, G = x.double().cpu().numpy(), gl.double().cpu().numpy()[s0]
        ref = X * G
        A = np.abs(ref)
        if zh:
            Z, H = z.double().cpu().numpy(), h.double().cpu().numpy()[s0]
            ref, A = ref + Z * H, A + np.abs(Z * H)
        if k:
            K = kk.double().cpu().numpy()[s0]
            ref, A = ref + K, A + np.abs(K)
        ref = np.where(inside, ref, 0.0)
        assert got.dtype == dtype
        if exact:
            w = _to_out(ref.astype(np.float32), dtype)
            assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref)
            assert torch.equal(got.cpu(), w), f"{int((got.cpu() != w).sum())} differ"
        else:
            ref_t = torch.as_tensor(ref)
            A_t = torch.as_tensor(np.where(inside, A, 0.0))
            bound = one_rounding_bound(ref_t, A_t, dtype, acc=gamma(3) * 2.0 ** 20)
            err = (got.cpu().double() - ref_t).abs()
            assert bool((err <= bound).all()), f"{int((err > bound).sum())} beyond the bound"
        assert int(got[::7].count_nonzero()) == 0


# ---- modules against the float64 oracle -------------------------------------------------------------
MODULE_SIZES = [1, 700, 0, 1, 2050, 513]        # one-row clouds, an empty cloud, 5 tiles


def _module_input(ME, cuda, dtype, C, field, sizes=MODULE_SIZES, seed=0, mean=None, std=None):
    """A SparseTensor (or TensorField) over clouds of `sizes` rows (shuffled) whose manager's
    origin holds every cloud; features normal(mean, std) per channel rounded to dtype."""
    rng = np.random.default_rng(seed)
    seg = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(seg)
    n = len(seg)
    mean = np.zeros(C) if mean is None else np.asarray(mean, np.float64)
    std = np.ones(C) if std is None else np.asarray(std, np.float64)
    f = torch.as_tensor(rng.standard_normal((n, C)) * std + mean).to(dtype)
    mgr = ME.CoordinateManager(D=3)
    base = np.zeros((len(sizes), 4), np.int32)
    base[:, 0] = _batch_of(np.arange(len(sizes)))
    mgr.insert_and_map(torch.as_tensor(base).to(cuda), 1, "clouds")
    mgr.origin()
    coords = _coords(seg)
    if field:
        pts = coords.astype(np.float32)
        pts[:, 1:] += 0.25
        x = ME.TensorField(f.to(cuda).requires_grad_(True), torch.as_tensor(pts).to(cuda),
                           coordinate_manager=mgr)
    else:
        key, _ = mgr.insert_and_map(torch.as_tensor(coords).to(cuda), 1, "rows")
        x = ME.SparseTensor(f.to(cuda).requires_grad_(True), coordinate_map_key=key,
                            coordinate_manager=mgr)
    return x, seg, f.double().numpy()


def _within(got, ref, bound, what):
    got = got.detach().double().cpu()
    ref, bound = torch.as_tensor(ref, dtype=torch.float64), torch.as_tensor(bound,
                                                                             dtype=torch.float64)
    err = (got - ref).abs()
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
    """A bound on an fp32 result plus its one rounding to the stored dtype."""
    bound, ref = torch.as_tensor(bound), torch.as_tensor(ref)
    return bound if dtype == torch.float32 else bound + half_ulp(ref.abs() + bound, dtype)


def _depths(sizes, C, dtype, prod=False, avg=False):
    """gamma_D per cloud [B, 1] for the reduction of a module's (aligned) features."""
    return np.array([[gamma(seg_geometry(m, C, dtype).depth(prod, avg)) if m else 0.0]
                     for m in sizes])


GLOBAL_MODE_NAMES = [f"GLOBAL_{k}_POOLING_{v}" for k in ("SUM", "AVG", "MAX")
                     for v in ("DEFAULT", "KERNEL", "PYTORCH_INDEX")]


# every mode on a sparse tensor, one per reduction (the _KERNEL modes) on a tensor field
POOL_CASES = [(m, False) for m in GLOBAL_MODE_NAMES] + \
    [(m, True) for m in GLOBAL_MODE_NAMES if m.endswith("_KERNEL")]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("mode_name,field", POOL_CASES,
                         ids=[m + ("-field" if f else "") for m, f in POOL_CASES])
def test_global_pooling_modules(ME, cuda, mode_name, field, dtype):
    """MinkowskiGlobalPooling in every GLOBAL_* mode, forward and backward, against float64:
    SUM / AVG within gamma_D of sum|x| plus the store's rounding, MAX exactly; the backward
    copies (AVG: divides once in fp32) and rounds once."""
    C = 12
    x, seg, xv = _module_input(ME, cuda, dtype, C, field, seed=3)
    B = len(MODULE_SIZES)
    mode = getattr(ME.PoolingMode, mode_name)
    om = {"SUM": GO.POOL_SUM, "AVG": GO.POOL_AVG, "MAX": GO.POOL_MAX}[mode_name.split("_")[1]]
    y = ME.MinkowskiGlobalPooling(mode)(x)
    assert y.F.dtype == dtype and y.F.shape == (B, C)
    ref, aux = GO.global_pool_forward(xv, seg, B, om)
    if om == GO.POOL_MAX:
        assert np.array_equal(y.F.detach().double().cpu().numpy(), ref)
    else:
        A, cnt = GO.global_pool_forward(np.abs(xv), seg, B, om)
        gam = _depths(MODULE_SIZES, C, dtype, avg=om == GO.POOL_AVG)
        _within(y.F, ref, _stored(gam * A, ref, dtype), mode_name)
    gout = torch.randn(B, C, generator=_gen(cuda, "gout", mode_name), device=cuda).to(dtype)
    x.F.grad = None
    y.F.backward(gout)
    gv = gout.double().cpu().numpy()
    gref = GO.global_pool_backward(gv, seg, len(seg), om, aux)
    if om == GO.POOL_AVG:            # g / cnt in fp32: one rounding, then the store's
        _within(x.F.grad, gref, _stored(U * np.abs(gref), gref, dtype), mode_name + " backward")
    else:
        assert np.array_equal(x.F.grad.double().cpu().numpy(), gref), mode_name + " backward"


@pytest.mark.gpu
@pytest.mark.parametrize("field", [False, True], ids=["sparse", "field"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("op", ["add", "mul", "concat"])
def test_broadcast_modules(ME, cuda, op, dtype, field):
    """MinkowskiBroadcastAddition / Multiplication / Concatenation, forward bit for bit (one fp32
    operation, one rounding), dx exactly or bit for bit, dg within gamma_D of sum|terms| plus the
    store's rounding."""
    C = 12
    x, seg, xv = _module_input(ME, cuda, dtype, C, field, seed=4)
    B = len(MODULE_SIZES)
    mgr = x.coordinate_manager
    g = _gen(cuda, "glob", op)
    gl = torch.randn(B, C, generator=g, device=cuda).to(dtype).requires_grad_(True)
    glob = ME.SparseTensor(gl, coordinate_map_key=mgr.origin(), coordinate_manager=mgr)
    layer = {"add": ME.MinkowskiBroadcastAddition, "mul": ME.MinkowskiBroadcastMultiplication,
             "concat": ME.MinkowskiBroadcastConcatenation}[op]()
    out = layer(x, glob)
    assert isinstance(out, ME.TensorField) == field
    xs, gs = np.float32(xv), gl.detach().float().cpu().numpy()[seg]
    if op == "concat":
        want = np.concatenate([xs, gs], 1)
    else:
        want = xs + gs if op == "add" else xs * gs
    assert torch.equal(out.F.detach().cpu(), _to_out(want, dtype)), op
    dy = torch.randn(out.F.shape, generator=g, device=cuda).to(dtype)
    out.F.backward(dy)
    dyv = dy.double().cpu().numpy()
    if op == "add":
        assert torch.equal(x.F.grad, dy)
        terms = dyv
        gam = _depths(MODULE_SIZES, C, dtype)
    elif op == "mul":
        assert torch.equal(x.F.grad.cpu(), _to_out(np.float32(dyv) * gs, dtype))
        terms = dyv * xv
        gam = _depths(MODULE_SIZES, C, dtype, prod=True)
    else:
        assert torch.equal(x.F.grad, dy[:, :C])
        terms = dyv[:, C:]
        gam = _depths(MODULE_SIZES, C, dtype)
    S, _ = _seg_sums(terms, seg, B)
    A, _ = _seg_sums(np.abs(terms), seg, B)
    _within(gl.grad, S, _stored(gam * A, S, dtype), op + " dg")


def _inorm_bounds(xv, seg, B, C, dtype, sizes):
    """Per-element bounds of MinkowskiInstanceNormFunction's y (before the store) against
    float64, and the pieces the backward bound needs.

    mean' = AVG(x) lies within e_m = gamma_{D+1}·mean|x| of mu.  c' = fp32(x - mean') and
    var' = AVG(c'·c') (depth D + 2 on positive terms) lies in [var_lo, var_hi] with
        var_lo = sigma²·(1 - u)²·(1 - gamma_{D+2}),  var_hi = (sigma² + e_m²)·(1 + u)²·(1 + gamma_{D+2})
    (mean((x - mu - e)²) = sigma² + e²).  inv_std' = rsqrt(fp32(var' + eps)): one rounding of the
    sum, and rsqrtf's 2 ulp (4u); so inv_std' lies within the relative rho of s = (sigma² + eps)^-1/2.
    y' = fp32(fp32(x·is') + fp32(-mean'·is')): three roundings on terms of |x|·is' and |mean'|·is',
        |y' - y| <= s·[(rho + u(1 + rho))·(|x - mu| + e_m) + e_m + u(1 + u)(1 + rho)(|x| + |mu| + e_m)]."""
    eps = float(np.float32(1e-8))
    cnt = np.bincount(seg, minlength=B)
    mu = GO.global_pool_forward(xv, seg, B, GO.POOL_AVG)[0]
    A1 = GO.global_pool_forward(np.abs(xv), seg, B, GO.POOL_AVG)[0]
    g1 = np.array([[gamma(seg_geometry(m, C, dtype).depth(avg=True)) if m else 0.0] for m in sizes])
    g2 = np.array([[gamma(seg_geometry(m, C, torch.float32).depth(prod=True, avg=True)) if m
                    else 0.0] for m in sizes])
    e_m = g1 * A1
    var = GO.global_pool_forward((xv - mu[seg]) ** 2, seg, B, GO.POOL_AVG)[0]
    var_lo = var * (1 - U) ** 2 * (1 - g2)
    var_hi = (var + e_m ** 2) * (1 + U) ** 2 * (1 + g2)
    s = 1 / np.sqrt(var + eps)
    s_lo = (1 - 4 * U) / np.sqrt((var_hi + eps) * (1 + U))
    s_hi = (1 + 4 * U) / np.sqrt((var_lo + eps) * (1 - U))
    rho = np.maximum(s_hi / s - 1, 1 - s_lo / s) * (1 + 1e-12) + 1e-15
    S, M, E, R = s[seg], mu[seg], e_m[seg], rho[seg]
    by = S * ((R + U * (1 + R)) * (np.abs(xv - M) + E) + E +
              U * (1 + U) * (1 + R) * (np.abs(xv) + np.abs(M) + E))
    return dict(s=s, rho=rho, by=by, cnt=cnt)


INORM_CASES = [
    # sizes, C, mean and std per channel (cycled)
    pytest.param(MODULE_SIZES, 12, (0, 1e3, 2.5, -3), (1, 1, 0, 2), id="offsets-constant"),
    pytest.param([102_400, 1, 3], 8, (0, 1e3, 2.5, -3), (1, 1, 0, 2), id="200-tiles"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("sizes,C,means,stds", INORM_CASES)
def test_instance_norm_module(ME, cuda, sizes, C, means, stds, dtype, record_property):
    """MinkowskiInstanceNorm forward and backward against float64 (tests/global_oracle.py), each
    element within the bound of _inorm_bounds and its backward counterpart.  Channel 1 sits at
    10^3 with std 1, channel 2 is the constant 2.5 (output exactly 0), one-row clouds give output
    and input gradient exactly 0."""
    B = len(sizes)
    mean = np.resize(np.asarray(means, np.float64), C)
    std = np.resize(np.asarray(stds, np.float64), C)
    x, seg, xv = _module_input(ME, cuda, dtype, C, False, sizes=sizes, seed=5, mean=mean, std=std)
    layer = ME.MinkowskiInstanceNorm(C).to(cuda)
    out = layer(x)
    eps = float(np.float32(1e-8))
    ref, inv_std = GO.instance_norm_forward(xv, seg, B, eps=eps)
    b = _inorm_bounds(xv, seg, B, C, dtype, sizes)
    ratios = {"y": _within(out.F, ref, _stored(b["by"], ref, dtype), "y")}
    one_row = np.isin(seg, [s for s, m in enumerate(sizes) if m == 1])
    yk = out.F.detach().double().cpu().numpy()
    assert not yk[one_row].any(), "one-row clouds: y is not 0"
    assert not yk[:, 2::4].any(), "a constant channel: y is not 0"
    dy = torch.randn(out.F.shape, generator=_gen(cuda, "dy", C), device=cuda).to(dtype)
    out.F.backward(dy)
    dyv = dy.double().cpu().numpy()
    gref = GO.instance_norm_backward(dyv, ref, inv_std, seg, B)
    # dx = s·(dy - y·a - c), a = mean(dy·y), c = mean(dy); the kernel uses its stored y' (within
    # By of y), a' = AVG(dy·y') (depth D + 2), c' = AVG(dy) (D + 1), is' (rho), and rounds
    # fp32(dy·is'), fmaf(y', fp32(-a'·is'), .), + fp32(-c'·is'): at most 4u·is'·T with one
    # spare, T = |dy| + |y'||a'| + |c'|.
    By = _stored(b["by"], ref, dtype).numpy()
    g1 = np.array([[gamma(seg_geometry(m, C, dtype).depth(avg=True)) if m else 0.0] for m in sizes])
    g2 = np.array([[gamma(seg_geometry(m, C, dtype).depth(prod=True, avg=True)) if m else 0.0]
                   for m in sizes])
    a = GO.global_pool_forward(dyv * ref, seg, B, GO.POOL_AVG)[0]
    c = GO.global_pool_forward(dyv, seg, B, GO.POOL_AVG)[0]
    ad = GO.global_pool_forward(np.abs(dyv), seg, B, GO.POOL_AVG)[0]
    e_a = g2 * GO.global_pool_forward(np.abs(dyv) * (np.abs(ref) + By), seg, B, GO.POOL_AVG)[0] + \
        GO.global_pool_forward(np.abs(dyv) * By, seg, B, GO.POOL_AVG)[0]
    e_c = g1 * ad
    S, R, Ea, Ec = b["s"][seg], b["rho"][seg], e_a[seg], e_c[seg]
    Aa, Ac = np.abs(a[seg]) + Ea, np.abs(c[seg]) + Ec
    T = np.abs(dyv) + (np.abs(ref) + By) * Aa + Ac
    bdx = R * S * T + S * (By * Aa + np.abs(ref) * Ea + Ec) + 4 * U * S * (1 + R) * T
    ratios["dx"] = _within(x.F.grad, gref, _stored(bdx, gref, dtype), "dx")
    gk = x.F.grad.double().cpu().numpy()
    assert not gk[one_row].any(), "one-row clouds: dx is not 0"
    record_property("worst_ratio_to_bound", max(ratios.values()))
    print(f"[inorm fp64] {sizes[0]} rows C={C} {_dt(dtype)}: " +
          ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))


@pytest.mark.gpu
def test_global_max_pooling_above_6144_channels(ME, cuda):
    """MinkowskiGlobalMaxPooling over 6148 and 8192 channels (the reduction's shared memory
    exceeds the default 48 KB there): forward and gradient exactly the oracle's."""
    for C in (6144, 6148, 8192):
        x, seg, xv = _module_input(ME, cuda, torch.float32, C, False, sizes=[3, 40, 0, 1], seed=C)
        y = ME.MinkowskiGlobalMaxPooling()(x)
        ref, aux = GO.global_pool_forward(xv, seg, 4, GO.POOL_MAX)
        assert np.array_equal(y.F.detach().double().cpu().numpy(), ref)
        gout = torch.randn(4, C, generator=_gen(cuda, "max", C), device=cuda)
        y.F.backward(gout)
        gref = GO.global_pool_backward(gout.double().cpu().numpy(), seg, len(seg), GO.POOL_MAX,
                                       aux)
        assert np.array_equal(x.F.grad.double().cpu().numpy(), gref)
