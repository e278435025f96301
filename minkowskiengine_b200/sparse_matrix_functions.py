"""COO sparse matrix times dense matrix (reference: sparse_matrix_functions.py), on the native
grouped reduction (`meb200_group_by_row` + `meb200_field_reduce` with a per-entry source row).

The reference's GPU path is cuSPARSE COO SpMM.  Here the entries are grouped by row with a stable
radix sort and every output row sums its entries in entry order with fp32 accumulation and one
rounding, so results are bit-identical run to run in fp32, bf16 and fp16.  Duplicate entries are
summed; a row without entries is 0.  Every call checks its indices on the device and raises
RuntimeError for one outside the matrix, which costs one host synchronisation.  `is_sorted` and
`cuda_spmm_alg` are accepted for compatibility and ignored: the result depends on neither.  CUDA
tensors only; fp64 raises."""
import torch
from torch.autograd import Function

from . import backend as _C


def _check_indices(rows, cols, mat):
    assert len(rows) == len(cols), "Invalid length"
    assert mat.is_cuda and rows.is_cuda and cols.is_cuda, "All inputs must be on cuda"
    assert rows.device == mat.device and cols.device == mat.device, "device mismatch"


def spmm(rows: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, size: torch.Size,
         mat: torch.Tensor, is_sorted: bool = False, cuda_spmm_alg: int = 1) -> torch.Tensor:
    """[size[0], C] = A @ mat, A the size[0] x size[1] COO matrix with vals[p] at
    (rows[p], cols[p]).  Index tensors may be int32, int64 or float (converted as `.int()`);
    vals has mat's dtype (fp32, bf16 or fp16) and is widened exactly to fp32 weights."""
    assert len(rows) == len(vals), "Invalid length"
    assert vals.dtype == mat.dtype, "dtype mismatch"
    assert vals.device == mat.device, "device mismatch"
    _check_indices(rows, cols, mat)
    assert vals.is_cuda, "All inputs must be on cuda"
    return _C.coo_spmm_int32(rows, cols, vals, size[0], size[1], mat, cuda_spmm_alg, is_sorted)


def spmm_average(rows: torch.Tensor, cols: torch.Tensor, size: torch.Size, mat: torch.Tensor,
                 cuda_spmm_alg: int = 1):
    """(result, COO, vals): result[r] = the mean of mat[cols[p]] over the entries of row r (0 for
    a row without entries); COO = int64 [2, P] of the entries stably sorted by row; vals = 1 /
    (entries of the row) in mat's dtype, the values of the matrix whose product is the result."""
    _check_indices(rows, cols, mat)
    result, coo, vals = _C.coo_spmm_average_int32(rows, cols, size[0], size[1], mat, cuda_spmm_alg)
    return result, coo, vals


class MinkowskiSPMMFunction(Function):
    """spmm with autograd: the gradient of mat is spmm over the transposed matrix; vals and the
    indices get none, as in the reference."""

    @staticmethod
    def forward(ctx, rows: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor, size: torch.Size,
                mat: torch.Tensor, cuda_spmm_alg: int = 1):
        ctx.misc_args = size, cuda_spmm_alg
        ctx.save_for_backward(rows, cols, vals)
        return spmm(rows, cols, vals, size, mat, is_sorted=False, cuda_spmm_alg=cuda_spmm_alg)

    @staticmethod
    def backward(ctx, grad: torch.Tensor):
        size, cuda_spmm_alg = ctx.misc_args
        rows, cols, vals = ctx.saved_tensors
        new_size = torch.Size([size[1], size[0]])
        grad = spmm(cols, rows, vals, new_size, grad.contiguous(), is_sorted=False,
                    cuda_spmm_alg=cuda_spmm_alg)
        return None, None, None, None, grad, None


class MinkowskiSPMMAverageFunction(Function):
    """spmm_average with autograd: the gradient of mat is spmm over the transposed averaging
    matrix (the COO and vals the forward returns)."""

    @staticmethod
    def forward(ctx, rows: torch.Tensor, cols: torch.Tensor, size: torch.Size, mat: torch.Tensor,
                cuda_spmm_alg: int = 1):
        ctx.misc_args = size, cuda_spmm_alg
        result, coo, vals = spmm_average(rows, cols, size, mat, cuda_spmm_alg=cuda_spmm_alg)
        ctx.save_for_backward(coo, vals)
        return result

    @staticmethod
    def backward(ctx, grad: torch.Tensor):
        size, cuda_spmm_alg = ctx.misc_args
        coo, vals = ctx.saved_tensors
        new_size = torch.Size([size[1], size[0]])
        grad = spmm(coo[1], coo[0], vals, new_size, grad.contiguous(), is_sorted=False,
                    cuda_spmm_alg=cuda_spmm_alg)
        return None, None, None, grad, None
