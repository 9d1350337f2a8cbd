"""ctypes binding of the C-ABI library (include/diffdock_b200.h).  No CPU fallback: if the shared library is
missing, or CUDA is not available when a compute entry point is called, this raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdiffdock_b200.so')

_lib = None

_vp, _i32, _i64, _int = C.c_void_p, C.c_int32, C.c_int64, C.c_int

# name -> (restype, argtypes); mirrors include/diffdock_b200.h one to one
SIGNATURES = {
    'ddb200_version': (C.c_char_p, []),
    'ddb200_tp_table_create': (_int, [_vp, _int, _vp, _int, C.POINTER(_vp)]),
    'ddb200_tp_table_destroy': (None, [_vp]),
    'ddb200_tp_table_info': (_int, [_vp, _int]),
    'ddb200_tpconv_accumulate': (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp]),
    'ddb200_tpconv_finalize': (_int, [_vp, _vp, _i64, _int, _int, _vp, _vp, _vp, _i64, _int, _vp, _vp]),
    'ddb200_radius_count': (_int, [_vp, _vp, _vp, _vp, _vp, C.c_float, _i64, _int, _int, _vp, _vp]),
    'ddb200_radius_fill': (_int, [_vp, _vp, _vp, _vp, _vp, C.c_float, _i64, _int, _int, _vp, _vp, _vp, _vp]),
    'ddb200_pose_update': (_int, [_vp, _i64, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _int, _vp,
                                  _vp]),
    'ddb200_pose_update_dev': (_int, [_vp, _i64, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64,
                                      _vp, _int, _vp, _vp]),
    'ddb200_pose_update_packed': (_int, [_vp, _i64, _vp, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64,
                                         _vp, _int, _vp, _vp, _vp]),
    'ddb200_philox_probe': (_int, [C.c_uint64, _i64, C.c_uint32, C.c_uint32, _int, _vp, _vp, _vp]),
    'ddb200_graph_fill': (_int, [_vp, _vp, _vp, _vp, _vp, C.c_float, _i64, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp, _int, _vp, _int, _int, _vp]),
    'ddb200_csr_sort_by_target': (_int, [_vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    'ddb200_edge_embed': (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _int, _int, _vp, C.c_float, _i64, _vp, _vp, _vp]),
    'ddb200_radial_gemm': (_int, [_vp, _i64, _i64, _int, _vp, _vp, _int, _vp, _i64, _vp]),
    'ddb200_radial_mlp': (_int, [_vp, _i64, _int, _vp, _i64, _int, _vp, _vp, _vp, _vp, _int, _vp, _vp, _int, _i64, _vp,
                                 _i64, _vp]),
    'ddb200_fused_conv': (_int, [_vp, _vp]),          # (const ddb200_fused_args*, stream)
    'ddb200_fused_conv_so': (_int, [_vp, _vp]),       # (const ddb200_fused_args*, stream), second-order plans
    'ddb200_fused_debug_read': (_int, [_vp]),
    'ddb200_contact_count': (_int, [_vp, _i32, C.c_float, _i32, _i32, _vp, _vp]),
    'ddb200_contact_fill': (_int, [_vp, _i32, C.c_float, _i32, _i32, _vp, _vp, _vp, _vp]),
    'ddb200_crop_flags': (_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    'ddb200_crop_select_edges': (_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'ddb200_receptor_need': (_int, [_vp, _vp, _i64, _i32, _vp, _vp, _i64, _vp, _i64, _i32, _vp, _vp]),
    'ddb200_confidence_head': (_int, [_vp, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _i32,
                                      _vp, _vp, _vp]),
}

# the deterministic (fixed-point) convolutions of the same library; mirrors include/diffdock_b200_fixed.h one to one
FIXED_SIGNATURES = {
    'ddb200_tpconv_accumulate_fixed': (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    'ddb200_tpconv_finalize_fixed': (_int, [_vp, _vp, _i64, _int, _int, _vp, _vp, _vp, _i64, _int, _vp, _vp]),
    'ddb200_fused_conv_fixed': (_int, [_vp, _vp, _vp, _vp]),      # (args, int64 sum, int32 error word, stream)
    'ddb200_fused_conv_so_fixed': (_int, [_vp, _vp, _vp, _vp]),
}

# the pose metrics of evaluation; mirrors include/diffdock_b200_metrics.h one to one
METRICS_SIGNATURES = {
    'ddb200_pose_metrics': (_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
                f"g.build()').  diffdock_b200 has no CPU fallback.")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in (SIGNATURES | FIXED_SIGNATURES | METRICS_SIGNATURES).items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


def check(rc: int, what: str):
    if rc != 0:
        names = {-1: 'DDB200_EINVAL', -2: 'DDB200_ETABLE', -3: 'DDB200_ESMEM'}
        raise RuntimeError(f"{what} failed: {names.get(rc, f'cudaError {rc}')}")
