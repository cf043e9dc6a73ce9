"""ctypes binding of libdhqr.so (include/dhqr.h).  No fallbacks: if the CUDA library is missing or a
call fails, this raises — the product path never routes through oracle/ or any CPU code."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdhqr.so")

_i64, _int, _vp, _dbl, _u64 = C.c_int64, C.c_int, C.c_void_p, C.c_double, C.c_uint64

# name -> argtypes; every function returns int except the two noted below.  Kept in one table so
# tests can check that the library exports exactly what include/dhqr.h declares.
SIGNATURES = {
    "dhqr_version": [],
    "dhqr_last_error": [],
    "dhqr_create": [C.POINTER(_vp), _int],
    "dhqr_create_dist": [C.POINTER(_vp), _int, _vp, _int, _int],
    "dhqr_nccl_unique_id": [_vp],
    "dhqr_destroy": [_vp],
    "dhqr_set_option": [_vp, C.c_char_p, _i64],
    "dhqr_get_option": [_vp, C.c_char_p, C.POINTER(_i64)],
    "dhqr_launch_count": [_vp, C.POINTER(_i64)],
    "dhqr_profile_reset": [_vp],
    "dhqr_profile_get": [_vp, _int, C.c_char_p, _int, C.POINTER(_dbl), C.POINTER(_i64), C.POINTER(_dbl)],
    "dhqr_plan_host_upload": [_i64, _i64, _int, _int, _int, _int, _int, _int, _int, C.POINTER(_i64), C.POINTER(_int), C.POINTER(_int)],
    "dhqr_qr_f64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _int, _vp],
    "dhqr_apply_qt_f64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _int, _vp],
    "dhqr_apply_q_f64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _int, _vp],
    "dhqr_backsolve_f64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_solve_f64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_qr_c64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _vp],
    "dhqr_apply_qt_c64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _int, _vp],
    "dhqr_backsolve_c64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_solve_c64": [_vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_partialdot_c64": [_vp, _vp, _vp, _i64, _i64, _vp, _vp],
    "dhqr_form_q_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _i64, _vp],
    "dhqr_form_q_c64": [_vp, _i64, _i64, _vp, _i64, _vp, _i64, _vp],
    "dhqr_forwardsolve_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_forwardsolve_c64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_solve_adj_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_solve_adj_c64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _int, _vp],
    "dhqr_qrcp_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp],
    "dhqr_solve_qrcp_f64": [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _int, _vp],
    "dhqr_qr_host_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _int],
    "dhqr_ldiv_host_f64": [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp],
    "dhqr_partialdot_f64": [_vp, _vp, _vp, _i64, _i64, _vp, _vp],
    "dhqr_fill_uniform_f64": [_vp, _u64, _i64, _i64, _i64, _i64, _vp, _i64, _vp],
    "dhqr_k_block_reflector_f64": [_vp, _i64, _int, _vp, _i64, _i64, _int, _vp, _i64, _vp, _vp],
    "dhqr_debug_copy_f64": [_vp, C.c_char_p, _vp, _i64, _vp],
    "dhqr_k_panel_f64": [_vp, _i64, _int, _vp, _i64, _vp, _vp],
    "dhqr_k_wide_panel_f64": [_vp, _i64, _vp, _i64, _vp, C.POINTER(_int), _vp],
}

_lib = None


class DhqrError(RuntimeError):
    def __init__(self, fn: str, code: int, text: str):
        super().__init__(f"{fn} returned {code}: {text}")
        self.code = code


def load() -> C.CDLL:
    """Load libdhqr.so (built in-tree by __graft_entry__.build()).  Fails loudly when absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_char_p if name == "dhqr_last_error" else _int
    _lib = lib
    return lib


def call(name: str, *args) -> None:
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise DhqrError(name, rc, lib.dhqr_last_error().decode(errors="replace"))
