"""Counts (not times) of the (128-row tile, offset) stages the tensor-core forward / dgrad runs on
the bench's clouds, with and without the tile order of meb200_kernel_map.  CPU only (numpy).

    python profiles/tile_order_counts.py [--clouds 8] [--voxels 100000] [--seed 0]

Per stride level of MinkUNet34C, for the k3 table of the level and for the k2s2 tables between
the level and the next: `dense` = every offset for every tile (no order), `natural` = only the
offsets a tile reaches in the map's own row order, `sorted` = the same after the stable sort by
neighbour mask, `sorted, 256 rows` = the same sorted order cut into 256-row tiles, `bound` =
pairs / 128 (every tile full of pairs).  A per-layer table then gives the bytes one forward call
copies from L2 into shared memory: A = the gathered rows (pairs x c_red x 2), B = the offset's
weight slice for all columns, once per stage (stages x c_cols x c_red x 2), at 128- and 256-row
tiles.

A second table counts the pair-mode weight gradient's 64-pair stages on the same tables (pair-list
chunks of 262144 rows, one 128-channel tile, CTA time proportional to its stages, CTAs placed in
launch order on the first free of `--resident` slots): `per offset` = the makespan of the same
number of CTAs for every offset (tc_config.h wgrad_splits, each 1/splits of its offset), `bound` =
total / resident.  An offset above twice the mean sets the makespan: k_wgrad_wg runs its CTAs in
column slices.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TILE = 128


def _keys(c):
    """int64 key of int32 rows (batch, x, y, z), every axis shifted into 16 bits."""
    c = c.astype(np.int64)
    return (c[:, 0] << 48) | ((c[:, 1] + 32768) << 32) | ((c[:, 2] + 32768) << 16) | (c[:, 3] + 32768)


def _strided(coords, ts):
    """The strided map in first-occurrence order (the insert's row numbering)."""
    s = coords.copy()
    s[:, 1:] = np.floor_divide(s[:, 1:], ts) * ts
    _, first = np.unique(_keys(s), return_index=True)
    return s[np.sort(first)]


def _masks(out_c, in_c, offsets):
    """Neighbour mask of every out row: bit k when out + offsets[k] is a row of in."""
    ik = np.sort(_keys(in_c))
    m = np.zeros(len(out_c), dtype=np.int64)
    for k, o in enumerate(offsets):
        q = out_c.copy()
        q[:, 1:] += o
        qk = _keys(q)
        pos = np.minimum(np.searchsorted(ik, qk), len(ik) - 1)
        m |= (ik[pos] == qk).astype(np.int64) << k
    return m


def _stages(masks, tile=TILE):
    t = np.zeros((len(masks) + tile - 1) // tile, dtype=np.int64)
    np.bitwise_or.at(t, np.arange(len(masks)) // tile, masks)
    return int(sum(bin(int(v)).count("1") for v in t))


def _row(name, masks, K):
    n = len(masks)
    pairs = int(sum(bin(int(v)).count("1") for v in masks))
    dense = (n + TILE - 1) // TILE * K
    srt_masks = masks[np.argsort(masks, kind="stable")]
    nat, srt, srt256 = _stages(masks), _stages(srt_masks), _stages(srt_masks, 2 * TILE)
    print(f"| {name} | {n:,} | {pairs / n:.2f} | {dense:,} | {nat:,} | **{srt:,}** | {srt256:,} | "
          f"{pairs / TILE:,.0f} |")
    return pairs, srt, srt256


WG_STAGE, WG_CHUNK, SMS = 64, 262144, 132
# MinkUNet34C k3 layers of the byte table: (name, stride level, c_red, c_cols); a forward reduces
# over c_in into c_out columns (the dgrad of c_in -> c_out reduces over c_out into c_in columns)
LAYER_BYTES = [("block8 96→96", 1, 96, 96), ("block8 128→96", 1, 128, 96),
               ("block7 96→96", 2, 96, 96), ("block4 256→256", 16, 256, 256),
               ("block3 128→128", 8, 128, 128)]


def _wgrad_stages(masks, K):
    """[K] 64-pair stages of every offset's pair list, summed over its row chunks."""
    n = len(masks)
    st = np.zeros(K, dtype=np.int64)
    for c0 in range(0, n, WG_CHUNK):
        m = masks[c0:c0 + WG_CHUNK]
        for k in range(K):
            st[k] += (int(((m >> k) & 1).sum()) + WG_STAGE - 1) // WG_STAGE
    return st


def _makespan(works, slots):
    """CTAs of the given works placed in order on the first free of `slots` slots."""
    free = np.zeros(slots, dtype=np.int64)
    for w in works:
        i = int(np.argmin(free))
        free[i] += w
    return int(free.max())


def _wgrad_row(name, masks, K, resident):
    st = _wgrad_stages(masks, K)
    n = len(masks)
    # wgrad_splits(n / 192 + 1, K, 1, 132) CTAs per offset, share x of offset k taking about
    # 1/splits of its stages; launch order: the shares of an offset, then the next offset
    want = -(-2 * SMS // K)
    splits = max(1, min(want, (n // (3 * WG_STAGE) + 1) // 4))
    works = [int(s) * (x + 1) // splits - int(s) * x // splits for s in st for x in range(splits)]
    today = _makespan(works, resident)
    bound = -(-int(st.sum()) // resident)
    print(f"| {name} | {n:,} | {st.max() / st.mean():.2f} | {splits * K} | {today:,} | "
          f"{bound:,} | {today / max(bound, 1):.2f} |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--resident", type=int, default=264,
                    help="wgrad CTAs the GPU runs at once (2 per SM at c_out <= 96 on 132 SMs)")
    a = ap.parse_args()
    import torch
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(a.voxels, a.seed + j, batch=j) for j in range(a.clouds)])
    coords = coords.numpy()
    k3 = [(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)]
    k2 = [(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)]
    print("| table | rows | nbrs/row | dense | natural | sorted by mask | sorted, 256 rows | bound |")
    print("|---|---|---|---|---|---|---|---|")
    levels = [coords]
    for ts in (2, 4, 8, 16):
        levels.append(_strided(levels[-1], ts))
    tables, counts = [], {}
    for i, c in enumerate(levels):
        ts = 2 ** i
        tables.append((f"k3, stride {ts}", _masks(c, c, np.array(k3) * ts), 27))
        counts[ts] = _row(*tables[-1])
        if i + 1 < len(levels):
            coarse = levels[i + 1]
            # strided k2s2: coarse rows gather fine rows; transposed: fine rows gather one coarse row
            tables.append((f"k2s2 {ts} → {2 * ts}", _masks(coarse, c, np.array(k2) * ts), 8))
            _row(*tables[-1])
            tables.append((f"k2s2 transposed {2 * ts} → {ts}",
                           _masks(c, coarse, -np.array(k2) * ts), 8))
            _row(*tables[-1])
    print()
    print("L2 -> shared-memory bytes of one forward call, GB (16-bit operands):")
    print()
    print("| layer (k3) | stride | c_red → c_cols | A | B, 128-row tiles | B, 256-row tiles |")
    print("|---|---|---|---|---|---|")
    for name, ts, c_red, c_cols in LAYER_BYTES:
        pairs, st128, st256 = counts[ts]
        print(f"| {name} | {ts} | {c_red} → {c_cols} | {pairs * c_red * 2 / 1e9:.2f} | "
              f"{st128 * c_cols * c_red * 2 / 1e9:.2f} | {st256 * c_cols * c_red * 2 / 1e9:.2f} |")
    print()
    print(f"wgrad stages (makespan of the slowest of {a.resident} CTA slots):")
    print()
    print("| table | rows | max / mean stages per offset | CTAs | per offset | bound | ratio |")
    print("|---|---|---|---|---|---|---|")
    for name, masks, K in tables:
        _wgrad_row(name, masks, K, a.resident)


if __name__ == "__main__":
    main()
