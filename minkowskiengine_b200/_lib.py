"""ctypes binding of the C-ABI library (include/meb200.h).

The product path has NO fallback: if libmeb200.so is missing or an entry point is absent,
loading raises, and every op that needs it raises with it.  Nothing here (or anywhere in
this package) imports `oracle/`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MEB200_LIB=libmeb200_x.so picks an A/B build of the same sources (csrc/build.py)
LIB_PATH = os.path.join(_HERE, "csrc", os.environ.get("MEB200_LIB", "libmeb200.so"))

OK = 0
F32, BF16, F16 = 0, 1, 2
TF32 = 3           # fp32 storage, TF32 tensor-core math (convolutions only)
POOL_SUM, POOL_AVG, POOL_MAX = 0, 1, 2
SEG_SUM, SEG_AVG, SEG_MAX = 0, 1, 2
BCAST_ADD, BCAST_MUL, BCAST_COPY, BCAST_MAXGRAD = 0, 1, 2, 3
UNION_ADD, UNION_SUB, UNION_MUL, UNION_DIV = 0, 1, 2, 3
FIELD_SUM, FIELD_AVG, FIELD_MAX, FIELD_SUBSAMPLE = 0, 1, 2, 3
ERR_DOMAIN = -4

_u32, _u64, _i32, _vp = C.c_uint32, C.c_uint64, C.c_int, C.c_void_p

# name -> (restype, argtypes); must list every symbol include/meb200.h declares
PROTOTYPES = {
    "meb200_last_error": (C.c_char_p, []),
    "meb200_build_arch": (C.c_char_p, []),
    "meb200_cudart_version": (_i32, []),
    "meb200_launch_count": (_u64, []),
    "meb200_tc_launch_count": (_u64, []),
    "meb200_hash_capacity": (_u32, [_u32]),
    "meb200_insert_scratch_bytes": (_u64, [_u32]),
    "meb200_insert_and_map_enqueue": (_i32, [_vp, _vp, _vp, _u32, _u32, _vp, _u32, _vp, _vp, _vp,
                                             _vp, _vp, _vp]),
    "meb200_map_build_table": (_i32, [_vp, _u32, _u32, _vp, _u32, _vp]),
    "meb200_insert_and_map": (_i32, [_vp, _vp, _u32, _u32, _vp, _u32, _vp, _vp, _vp, _vp,
                                     C.POINTER(_u32), _vp]),
    "meb200_stride_coords": (_i32, [_vp, _u32, _u32, C.POINTER(C.c_int32), _vp, _vp]),
    "meb200_region_coords": (_i32, [_vp, _u32, _u32, _vp, _u32, C.POINTER(C.c_int32), _i32,
                                    _vp, _vp, _vp]),
    "meb200_map_find": (_i32, [_vp, _vp, _u32, _u32, _vp, _u32, _vp, _vp]),
    "meb200_kernel_map": (_i32, [_vp, _u32, _vp, _u32, _vp, _u32, _u32, _vp, _u32, _vp, _vp,
                                 _vp, _vp, _vp, _vp, _vp]),
    "meb200_conv_forward": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _u32, _vp,
                                   _i32, _vp, _vp, _vp]),
    "meb200_conv_backward": (_i32, [_vp, _vp, _i32, _u32, _u32, _vp, _u32, _u32, _vp, _vp,
                                    _u32, _vp, _i32, _vp, _vp, _vp, _vp, _u32, _vp, _u64, _vp,
                                    _vp]),
    "meb200_conv_wgrad_uses_pairs": (_i32, [_i32, _u32, _u32, _u32]),
    "meb200_conv_fp8_supported": (_i32, [_u32, _u32]),
    "meb200_conv_forward_fp8": (_i32, [_vp, _vp, _u32, _u32, _vp, _u32, _u32, _vp, _u32, _vp, _i32,
                                       _vp, _vp, _vp]),
    "meb200_conv_pack_weights_e4m3": (_i32, [_vp, _u32, _u32, _u32, _vp, _vp, _vp]),
    "meb200_quantize_e4m3_workspace_bytes": (_u64, []),
    "meb200_quantize_e4m3": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp]),
    "meb200_amax_accumulate": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp]),
    "meb200_e4m3_scales": (_i32, [_vp, _vp, _vp]),
    "meb200_quantize_e4m3_static": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp]),
    "meb200_conv_forward_q": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _u32, _vp,
                                     _i32, _vp, _vp, _vp, _vp, _vp]),
    "meb200_conv_forward_fp8_q": (_i32, [_vp, _vp, _u32, _u32, _vp, _u32, _u32, _vp, _u32, _vp,
                                         _i32, _vp, _vp, _vp, _vp, _vp]),
    "meb200_conv_stem_forward_q": (_i32, [_vp, _i32, _u32, _vp, _u32, _vp, _u32, _vp, _i32, _vp,
                                          _vp, _vp, _vp]),
    "meb200_quantize_e5m2": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp]),
    "meb200_conv_pack_weights_e4m3_dgrad": (_i32, [_vp, _u32, _u32, _u32, _vp, _vp, _vp]),
    "meb200_conv_dgrad_fp8": (_i32, [_vp, _vp, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _u32, _vp,
                                     _i32, _vp, _vp]),
    "meb200_conv_wgrad_fp8_supported": (_i32, [_u32, _u32, _u32]),
    "meb200_conv_wgrad_fp8_workspace_bytes": (_u64, [_u32, _u32, _u32, _u32]),
    "meb200_conv_wgrad_fp8": (_i32, [_vp, _vp, _vp, _vp, _u32, _u32, _u32, _vp, _vp, _vp, _u32,
                                     _u32, _vp, _vp, _u64, _vp]),
    "meb200_conv_pack_weights": (_i32, [_vp, _u32, _u32, _u32, _i32, _vp, _vp, _vp]),
    "meb200_conv_pack_weights_batched": (_i32, [_vp, _u32, _u32, _i32, _vp]),
    "meb200_conv_stem_virtual_channels": (_u32, [_u32]),
    "meb200_conv_stem_supported": (_i32, [_i32, _u32, _u32]),
    "meb200_conv_stem_forward": (_i32, [_vp, _i32, _u32, _vp, _u32, _vp, _u32, _vp, _i32, _vp,
                                        _vp]),
    "meb200_conv_stem_wgrad": (_i32, [_vp, _vp, _i32, _u32, _u32, _vp, _u32, _vp, _vp, _u64, _vp]),
    "meb200_pair_list_chunks": (_u32, [_u32, _u32]),
    "meb200_pair_list_scratch_bytes": (_u64, [_u32, _u32, _u32]),
    "meb200_pair_list_capacity": (_u64, [_u32, _u32, _u32, _u32]),
    "meb200_kernel_map_pairs": (_i32, [_vp, _u32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp]),
    "meb200_conv_workspace_bytes": (_u64, [_u32, _u32, _u32, _u32, _i32]),
    "meb200_chwise_gather": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _vp]),
    "meb200_chwise_wgrad_workspace_bytes": (_u64, [_u32, _u32, _u32, _i32]),
    "meb200_chwise_wgrad": (_i32, [_vp, _vp, _i32, _u32, _u32, _vp, _u32, _u32, _vp, _vp, _u64,
                                   _vp]),
    "meb200_pool_forward":(_i32, [_vp, _i32, _u32, _u32, _vp, _u32, _u32, _i32, _vp, _vp, _vp]),
    "meb200_pool_backward": (_i32, [_vp, _i32, _u32, _u32, _vp, _u32, _u32, _i32, _vp, _vp,
                                    _vp]),
    "meb200_origin_group_scratch_bytes": (_u64, [_u32, _u32]),
    "meb200_origin_group": (_i32, [_vp, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp,
                                   _vp]),
    "meb200_field_origin_group": (_i32, [_vp, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _vp, _vp,
                                         _vp, _vp, _vp, _vp]),
    "meb200_field_origin_insert": (_i32, [_vp, _u32, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp,
                                          C.POINTER(_u32), _vp]),
    "meb200_segment_max_tiles": (_u32, [_u32, _u32]),
    "meb200_segment_workspace_bytes": (_u64, [_u32, _u32, _u32]),
    "meb200_segment_reduce": (_i32, [_vp, _vp, _i32, _u32, _u32, _vp, _vp, _vp, _u32, _i32, _vp, _vp,
                                     _vp, _u64, _vp]),
    "meb200_broadcast": (_i32, [_vp, _i32, _vp, _vp, _vp, _u32, _u32, _i32, _vp, _i32, _vp]),
    "meb200_broadcast_fma": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "meb200_gather_rows": (_i32, [_vp, _i32, _u32, _u32, _vp, _u32, _vp, _vp]),
    "meb200_union_fold_forward": (_i32, [_vp, _u32, _u32, _vp, _u32, _u32, _i32, _i32, _vp, _vp]),
    "meb200_union_fold_backward": (_i32, [_vp, _u32, _u32, _vp, _u32, _u32, _i32, _i32, _vp, _u32,
                                          _vp, _u32, _vp, _vp]),
    "meb200_dense_from_rows": (_i32, [_vp, _i32, _u32, _vp, _vp, _u32, _vp, _vp, _vp]),
    "meb200_dense_to_rows": (_i32, [_vp, _i32, _vp, _vp, _u32, _vp, _vp]),
    "meb200_dense_nonzero_scratch_bytes": (_u64, [_u64]),
    "meb200_dense_nonzero_count": (_i32, [_vp, _i32, _vp, _vp, C.POINTER(_u32), _vp]),
    "meb200_dense_nonzero_coords": (_i32, [_vp, _vp, _vp, _vp]),
    "meb200_quantize_field": (_i32, [_vp, _u32, _u32, C.POINTER(C.c_int32), _vp, _vp, _vp]),
    "meb200_field_insert_and_map": (_i32, [_vp, _u32, _u32, C.POINTER(C.c_int32), _vp, _vp, _u32,
                                           _vp, _vp, _vp, _vp, C.POINTER(_u32), _vp]),
    "meb200_group_by_row_scratch_bytes": (_u64, [_u32, _u32]),
    "meb200_group_by_row": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp, _u64, _vp]),
    "meb200_field_reduce": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _i32, _vp,
                                   _vp, _vp]),
    "meb200_check_pairs": (_i32, [_vp, _vp, _u32, _u32, _u32, _vp, _vp]),
    "meb200_flat_mask": (_i32, [_vp, _vp, _u32, _u32, _u32, _i32, _vp, _vp]),
    "meb200_field_expand": (_i32, [_vp, _i32, _u32, _u32, _vp, _u32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "meb200_interp_map": (_i32, [_vp, _u32, _u32, C.POINTER(C.c_int32), _vp, _vp, _u32, _vp, _vp,
                                 _vp]),
    "meb200_splat_coords": (_i32, [_vp, _u32, _u32, _vp, _vp, _vp]),
    "meb200_interp_forward": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _u32, _u32, _vp, _vp]),
    "meb200_bn_workspace_bytes": (_u64, []),
    "meb200_bn_forward_train": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp, _i32, C.c_float,
                                       C.c_float, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "meb200_bn_stats_to": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp]),
    "meb200_bn_backward_reduce_to": (_i32, [_vp, _vp, _vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp,
                                            _vp, _vp, _vp]),
    "meb200_bn_finalize": (_i32, [_vp, C.c_double, _vp, _u32, C.c_float, C.c_float, _vp, _vp, _vp,
                                  _vp, _vp]),
    "meb200_bn_apply_fused": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "meb200_bn_backward_apply_fused": (_i32, [_vp, _vp, _vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp,
                                              C.c_double, _vp, _vp, _vp, _vp]),
    "meb200_bn_forward_train_peer": (_i32, [_vp, _i32, _u32, _u32, _vp, _vp, _vp, _i32, C.c_float,
                                            C.c_float, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _u32, _u32,
                                            _u32, _vp, _vp, _vp, _vp, _vp]),
    "meb200_bn_backward_reduce_peer": (_i32, [_vp, _vp, _vp, _i32, _u32, _u32, _vp, _vp, _vp, _vp,
                                              C.c_uint64, _u32, _u32, _u32, _vp, _vp, _vp, _vp]),
}

# These calls gained an optional pointer just before the stream: meb200_conv_backward its
# `in_order`, the two forwards their `epi`.  Callers written against the argument list they had
# before (the direct-call test helpers among them) still work: a call one argument short gets NULL
# there (no order: every tile runs every offset; no epilogue).  Any other argument count goes to
# ctypes unchanged and fails there.  The backend passes the full list.
_POINTER_ADDED = ("meb200_conv_backward", "meb200_conv_forward", "meb200_conv_stem_forward")

_lib = None


def _pointer_optional(fn, n_args):
    def call(*args):
        if len(args) == n_args - 1:
            args = args[:-1] + (None, args[-1])
        return fn(*args)
    call.argtypes, call.restype = fn.argtypes, fn.restype
    return call


class BackendError(RuntimeError):
    """Raised for every failure reported by libmeb200 (the reference raises RuntimeError
    from ASSERT/CUDA_CHECK, src/utils.hpp:141-150, src/gpu.cuh:63-163)."""


def load():
    """Loads libmeb200.so once; raises if it is missing (no CPU / eager fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise BackendError(
            f"{LIB_PATH} not found: build it with `python minkowskiengine_b200/csrc/build.py` "
            "(or __graft_entry__.build()). minkowskiengine_b200 has no fallback path.")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError -> loud failure on a stale library
        fn.restype = res
        fn.argtypes = args
    for name in _POINTER_ADDED:
        setattr(lib, name, _pointer_optional(getattr(lib, name), len(PROTOTYPES[name][1])))
    _lib = lib
    return lib


def check(rc):
    if rc != OK:
        msg = load().meb200_last_error().decode("utf-8", "replace")
        raise BackendError(f"libmeb200 error {rc}: {msg}")


def dtype_code(torch_dtype):
    """Code of a feature dtype, or of the convolution operand type "tf32" (backend._operand)."""
    import torch
    try:
        return {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16, "tf32": TF32}[torch_dtype]
    except KeyError:
        raise BackendError(
            f"unsupported feature dtype {torch_dtype}: this backend computes in "
            "float32, bfloat16 or float16") from None


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def current_stream():
    """Raw handle of torch's current CUDA stream on the current device (the fast private
    accessor when this torch has it: the public one builds a Stream object per call and this
    runs once per native launch, ~1000 times per training step)."""
    import torch
    raw = getattr(torch._C, "_cuda_getCurrentRawStream", None)
    if raw is not None:
        return raw(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def launch_count():
    return int(load().meb200_launch_count())


def tc_launch_count():
    return int(load().meb200_tc_launch_count())
