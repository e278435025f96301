"""float64 restatement of the COO sparse-times-dense products and of direct max pooling
(tests/test_spmm_cpu.py pins it to the compiled reference's fixtures; tests/test_gpu_spmm.py
compares the GPU against it element by element).

spmm (sparse_matrix_functions.py:32-77): out[r] = sum over the entries p with rows[p] = r of
vals[p] * mat[cols[p]]; duplicates add; a row without entries is 0.  spmm_average (:80-121): the
mean over a row's entries; its COO is stably sorted by row and its values are 1 / count.
Direct max pooling (src/direct_max_pool.cpp): out[o, c] = the maximum of x[i, c] over the pairs
(i, o), the first pair in list order winning a tie, mask[o, c] = i * C + c; this package's
semantics for a row without pairs (0, mask -1) and for all-negative channels (the true maximum).
The backward adds g[o, c] at mask[o, c] once per (o, c)."""
import torch


def _dev(*ts, device=None):
    return [torch.as_tensor(t).to(device) for t in ts]


def spmm(rows, cols, vals, n_rows, mat):
    """(out, A): float64 A @ mat and |A| @ |mat| (the scale of the fp32 accumulation error), on
    mat's device."""
    mat = torch.as_tensor(mat)
    rows, cols, vals = _dev(rows, cols, vals, device=mat.device)
    rows, cols, vals, mat = rows.long(), cols.long(), vals.double(), mat.double()
    out = torch.zeros((n_rows, mat.shape[1]), dtype=torch.float64, device=mat.device)
    A = torch.zeros_like(out)
    if len(rows):
        out.index_add_(0, rows, vals[:, None] * mat[cols])
        A.index_add_(0, rows, vals.abs()[:, None] * mat[cols].abs())
    return out, A


def average_coo(rows, cols, n_rows):
    """(COO int64 [2, P] stably sorted by row, float64 1 / count per entry)."""
    rows, cols = torch.as_tensor(rows).long(), torch.as_tensor(cols).long().to(
        torch.as_tensor(rows).device)
    order = torch.sort(rows, stable=True).indices
    r, c = rows[order], cols[order]
    count = torch.bincount(r, minlength=n_rows).double()
    return torch.stack((r, c)), 1.0 / count[r]


def spmm_average(rows, cols, n_rows, mat):
    """(out, A): the float64 mean of mat[cols[p]] over the entries of each row (0 without any),
    and the same mean over |mat|."""
    mat = torch.as_tensor(mat)
    rows, = _dev(rows, device=mat.device)
    rows = rows.long()
    count = torch.bincount(rows, minlength=n_rows).double().clamp(min=1)[:, None]
    s, A = spmm(rows, cols, torch.ones(len(rows), dtype=torch.float64), n_rows, mat)
    return s / count, A / count


def direct_max(in_map, out_map, x, n_out):
    """(out float64 [n_out, C], mask int64 [n_out, C]) on x's device."""
    x = torch.as_tensor(x)
    im, om = _dev(in_map, out_map, device=x.device)
    im, om, x = im.long(), om.long(), x.double()
    P, C = len(im), x.shape[1]
    v = x[im]
    idx = om[:, None].expand(P, C)
    out = torch.full((n_out, C), -float("inf"), dtype=torch.float64, device=x.device)
    out.scatter_reduce_(0, idx, v, "amax")
    p = torch.arange(P, device=x.device)[:, None].expand(P, C)
    first = torch.full((n_out, C), P, dtype=torch.int64, device=x.device)
    first.scatter_reduce_(0, idx, torch.where(v == out[om], p, P), "amin")   # first pair wins
    has = first < P
    ch = torch.arange(C, device=x.device)[None, :]
    mask = torch.where(has, im[first.clamp(max=max(P - 1, 0))] * C + ch, -1) if P else \
        torch.full((n_out, C), -1, dtype=torch.int64, device=x.device)
    return torch.where(has, out, 0.0), mask


def direct_max_backward(g, mask, n_in):
    """float64 [n_in, C]: g[o, c] added at the flat element mask[o, c] (>= 0) once per (o, c)."""
    g = torch.as_tensor(g).double()
    mask, = _dev(mask, device=g.device)
    mask = mask.long()
    C = g.shape[1]
    out = torch.zeros(n_in * C, dtype=torch.float64, device=g.device)
    m = mask.flatten() >= 0
    out.index_add_(0, mask.flatten()[m], g.flatten()[m])
    return out.view(n_in, C)
