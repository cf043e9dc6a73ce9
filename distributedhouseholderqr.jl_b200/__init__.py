"""dhqr_b200 — H100-native (sm_90a) blocked Householder QR behind DistributedHouseholderQR.jl's qr! / \\.

Import as ``import dhqr_b200`` (repo-root shim) — the directory keeps the name the task fixes
(``distributedhouseholderqr.jl_b200``), which is not a valid Python identifier.
"""
from . import _lib
from .api import (AppendedRows, BatchedAppendedRows, BatchedDowndatedRows, BatchedHouseholderQRStruct, BatchedStreamingLeastSquares, ColumnBlockMatrix, CompleteOrthogonalStruct, DistributedHouseholderQRStruct, DowndatedRows, Handle, LocalColumnBlock,
                  PivotedHouseholderQRStruct, StreamingLeastSquares, alphafactor, append_rows_, apply_q_, apply_q_batched_, apply_qt_, apply_qt_batched_, append_rows_batched_, backsolve_, backsolve_batched_, balanced_splits, cod_, colmajor_empty,
                  colmajor_empty_batched, default_handle, downdate_rows_, downdate_rows_batched_, fill_uniform_, form_q, form_r, forwardsolve_, householder_, init_distributed, ldiv,
                  ldiv_adjoint, partialdot, plan_host_upload, qr_, qr_bang, qr_batched_, qrcp_, shutdown_distributed, solve_adjoint_,
                  solve_batched_, solve_cod_, solve_householder_, solve_qrcp_, splits, to_colmajor)

__all__ = ["AppendedRows", "BatchedAppendedRows", "BatchedDowndatedRows", "BatchedHouseholderQRStruct", "BatchedStreamingLeastSquares", "ColumnBlockMatrix", "CompleteOrthogonalStruct", "DistributedHouseholderQRStruct", "DowndatedRows", "Handle", "LocalColumnBlock",
           "PivotedHouseholderQRStruct", "StreamingLeastSquares", "alphafactor", "append_rows_", "apply_q_", "apply_q_batched_", "apply_qt_", "apply_qt_batched_", "append_rows_batched_", "backsolve_", "backsolve_batched_", "balanced_splits", "cod_",
           "colmajor_empty", "colmajor_empty_batched", "default_handle", "downdate_rows_", "downdate_rows_batched_", "fill_uniform_", "form_q", "form_r", "forwardsolve_", "householder_",
           "init_distributed", "ldiv", "ldiv_adjoint", "partialdot", "plan_host_upload", "qr_", "qr_bang", "qr_batched_", "qrcp_",
           "shutdown_distributed", "solve_adjoint_", "solve_batched_", "solve_cod_", "solve_householder_", "solve_qrcp_", "splits", "to_colmajor",
           "_lib"]
