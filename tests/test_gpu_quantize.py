"""GPU voxelisation (SURVEY.md §8(f) row 2: utils/quantization.py:136-333, src/quantization.cpp)
against the compiled reference's CPU sparse_quantize on identical points: kept coordinates,
unique index and inverse map bit-exact, features/labels of the kept points identical.  The
reference's outputs are stored in tests/golden/ref_quantize.npz (digests of the exact values,
tests/golden/make_reference_runs.py)."""
import numpy as np
import pytest
import torch

from helpers import digest, golden

pytestmark = pytest.mark.gpu


def _points(n, seed, extent=40.0, D=3):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, D, generator=g) - 0.5) * extent          # negative halves included
    b = torch.randint(0, 3, (n, 1), generator=g).float()
    return torch.cat([b, pts], 1)


@pytest.mark.parametrize("n,qs", [(20000, 0.5), (50000, 1), (3000, 2.5), (1, 1), (100000, 0.25)])
def test_sparse_quantize_matches_reference(ME, cuda, n, qs):
    G, key = golden("ref_quantize.npz"), f"q_{n}_{qs}"

    def same(t, name):
        return bool((digest(t) == G[f"{key}/{name}"]).all())

    pts = _points(n, seed=n)
    pts[:, 0] *= qs if qs != 1 else 1          # keep the batch column integral after the division
    feats = torch.rand(n, 4, generator=torch.Generator().manual_seed(1))
    gc, gf, gi, ginv = ME.utils.sparse_quantize(pts, feats, return_index=True, return_inverse=True,
                                                quantization_size=qs, device="cuda")
    assert gc.is_cuda and gc.dtype == torch.int32
    assert same(gi.cpu(), "index") and same(gc.cpu(), "coords")
    assert same(gf.cpu(), "feats")
    if int(G[f"{key}/inverse_len"]):                # the reference returns [] when nothing merged
        assert same(ginv.cpu(), "inverse")
    assert torch.equal(gc[ginv].cpu(), torch.floor(pts / qs).int())
    # maps only
    m = ME.utils.sparse_quantize(pts, return_index=True, return_maps_only=True,
                                 quantization_size=qs, device="cuda")
    assert same(m.cpu(), "index")


def test_sparse_quantize_labels_match_reference(ME, cuda):
    G = golden("ref_quantize.npz")
    n = 30000
    pts = _points(n, seed=7, extent=24.0)
    g = torch.Generator().manual_seed(3)
    labels = torch.randint(0, 5, (n,), generator=g, dtype=torch.int32)
    labels[torch.rand(n, generator=g) < 0.02] = -100            # some points already "ignore"
    feats = torch.rand(n, 2, generator=g)
    ri, rinv = G["labels/index"], G["labels/inverse"]
    gc, gf, gl, gi, ginv = ME.utils.sparse_quantize(pts, feats, labels, ignore_label=-100,
                                                    return_index=True, return_inverse=True,
                                                    device="cuda")
    assert (digest(gc.cpu()) == G["labels/coords"]).all() and (digest(gf.cpu()) == G["labels/feats"]).all()
    assert torch.equal(gi.cpu().long(), torch.as_tensor(np.asarray(ri)).long())
    assert torch.equal(ginv.cpu().long(), torch.as_tensor(np.asarray(rinv)).long())
    assert (digest(gl.cpu().int()) == G["labels/labels"]).all()
    assert int((gl == -100).sum()) > 0
    # documented intent (label_mode="consistent"): first label if the voxel's points agree
    gl2 = ME.utils.sparse_quantize(pts, feats, labels, ignore_label=-100, device="cuda",
                                   label_mode="consistent")[2].cpu()
    inv, first = torch.as_tensor(np.asarray(rinv)).long(), labels[torch.as_tensor(np.asarray(ri)).long()]
    for u in range(0, len(first), 97):
        ls = labels[inv == u]
        want = int(first[u]) if bool((ls == first[u]).all()) or int(first[u]) == -100 else -100
        assert int(gl2[u]) == want


def test_collate_then_quantize_on_device(ME, cuda):
    clouds = [(_points(4000, s)[:, 1:] * 3).to(cuda) for s in range(3)]
    feats = [torch.rand(4000, 3, device=cuda) for _ in range(3)]
    bc, bf = ME.utils.sparse_collate(clouds, feats)
    assert bc.is_cuda and bc.shape == (12000, 4) and bf.shape == (12000, 3)
    assert [int((bc[:, 0] == b).sum()) for b in range(3)] == [4000] * 3
    c, f = ME.utils.sparse_quantize(bc, bf, device="cuda")
    x = ME.SparseTensor(f, c)
    assert len(x) == len(c) == len(torch.unique(bc, dim=0))
