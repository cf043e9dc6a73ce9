"""dhqr_b200 — H100-native (sm_90a) blocked Householder QR behind DistributedHouseholderQR.jl's qr! / \\.

Import as ``import dhqr_b200`` (repo-root shim) — the directory keeps the name the task fixes
(``distributedhouseholderqr.jl_b200``), which is not a valid Python identifier.
"""
from . import _lib
from .api import (ColumnBlockMatrix, DistributedHouseholderQRStruct, Handle, LocalColumnBlock, PivotedHouseholderQRStruct, alphafactor,
                  apply_q_, apply_qt_, backsolve_, balanced_splits, colmajor_empty, default_handle, fill_uniform_, form_q, form_r,
                  forwardsolve_, householder_, init_distributed, ldiv, ldiv_adjoint, partialdot, plan_host_upload, qr_, qr_bang, qrcp_,
                  shutdown_distributed, solve_adjoint_, solve_householder_, solve_qrcp_, splits, to_colmajor)

__all__ = ["ColumnBlockMatrix", "DistributedHouseholderQRStruct", "Handle", "LocalColumnBlock", "PivotedHouseholderQRStruct", "alphafactor",
           "apply_q_", "apply_qt_", "backsolve_", "balanced_splits", "colmajor_empty", "default_handle", "fill_uniform_", "form_q", "form_r",
           "forwardsolve_", "householder_", "init_distributed", "ldiv", "ldiv_adjoint", "partialdot", "plan_host_upload", "qr_", "qr_bang",
           "qrcp_", "shutdown_distributed", "solve_adjoint_", "solve_householder_", "solve_qrcp_", "splits", "to_colmajor", "_lib"]
