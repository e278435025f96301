"""Counts (not times) of the (128-row tile, offset) stages the tensor-core forward / dgrad runs on
the bench's clouds, with and without the tile order of meb200_kernel_map.  CPU only (numpy).

    python profiles/tile_order_counts.py [--clouds 8] [--voxels 100000] [--seed 0]

Per stride level of MinkUNet34C, for the k3 table of the level and for the k2s2 tables between
the level and the next: `dense` = every offset for every tile (no order), `natural` = only the
offsets a tile reaches in the map's own row order, `sorted` = the same after the stable sort by
neighbour mask, `bound` = pairs / 128 (every tile full of pairs).
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


def _stages(masks):
    t = np.zeros((len(masks) + TILE - 1) // TILE, dtype=np.int64)
    np.bitwise_or.at(t, np.arange(len(masks)) // TILE, masks)
    return int(sum(bin(int(v)).count("1") for v in t))


def _row(name, masks, K):
    n = len(masks)
    pairs = int(sum(bin(int(v)).count("1") for v in masks))
    dense = (n + TILE - 1) // TILE * K
    nat, srt = _stages(masks), _stages(masks[np.argsort(masks, kind="stable")])
    print(f"| {name} | {n:,} | {pairs / n:.2f} | {dense:,} | {nat:,} | **{srt:,}** | {pairs / TILE:,.0f} |")
    return dense, srt, pairs / TILE


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=8)
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    from examples.synthetic import surface_cloud
    coords = torch.cat([surface_cloud(a.voxels, a.seed + j, batch=j) for j in range(a.clouds)])
    coords = coords.numpy()
    k3 = [(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)]
    k2 = [(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)]
    print("| table | rows | nbrs/row | dense | natural | sorted by mask | bound |")
    print("|---|---|---|---|---|---|---|")
    levels = [coords]
    for ts in (2, 4, 8, 16):
        levels.append(_strided(levels[-1], ts))
    for i, c in enumerate(levels):
        ts = 2 ** i
        _row(f"k3, stride {ts}", _masks(c, c, np.array(k3) * ts), 27)
        if i + 1 < len(levels):
            coarse = levels[i + 1]
            # strided k2s2: coarse rows gather fine rows; transposed: fine rows gather one coarse row
            _row(f"k2s2 {ts} → {2 * ts}", _masks(coarse, c, np.array(k2) * ts), 8)
            _row(f"k2s2 transposed {2 * ts} → {ts}", _masks(c, coarse, -np.array(k2) * ts), 8)


if __name__ == "__main__":
    main()
