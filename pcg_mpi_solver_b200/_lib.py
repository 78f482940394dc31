"""ctypes binding of libpcgb200.so (include/pcgb200.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C pcg_mpi_solver_b200/csrc`.
There is deliberately NO fallback: if the shared object is missing or a call fails, an
exception is raised - the product path never degrades to a CPU / PyTorch implementation.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_int, c_int32, c_int64, c_ubyte, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libpcgb200.so")

UNIQUE_ID_BYTES = 128
IPC_BLOB_BYTES = 64
TRANSPORT_NCCL, TRANSPORT_PEER = 0, 1
MG_MAX_LEVELS = 32


class PcgbError(RuntimeError):
    pass


class Options(ctypes.Structure):
    _fields_ = [("tol", c_double), ("maxiter", c_int32), ("n_global", c_int64), ("max_stag", c_int32),
                ("check_every", c_int32), ("use_graph", c_int32), ("fixed_iters", c_int32),
                ("record_resvec", c_int32), ("time_kernels", c_int32), ("x0_zero", c_int32)]


class Result(ctypes.Structure):
    _fields_ = [("flag", c_int32), ("iters", c_int32), ("relres", c_double), ("normb", c_double),
                ("imin", c_int32), ("stag", c_int32), ("moresteps", c_int32), ("too_small_tol", c_int32),
                ("matvecs", c_int64), ("launches", c_int64), ("loop_ms", c_double), ("spmv_ms", c_double),
                ("spmv_timed", c_int64), ("loop_iters", c_int64), ("setup_ms", c_double), ("final_ms", c_double), ("phase_ms", c_double * 8)]


class EbeGroup(ctypes.Structure):
    _fields_ = [("nd", c_int32), ("ne", c_int64), ("d_idx", c_void_p), ("d_sign", c_void_p), ("d_ck", c_void_p), ("ke_host", c_void_p)]


class HexBox(ctypes.Structure):
    _fields_ = [("ng", c_int32 * 3), ("e0", c_int32 * 3), ("ne", c_int32 * 3)]


# name -> (restype, argtypes); every symbol declared in include/pcgb200.h
SIGNATURES = {
    "pcgb_version": (c_int, []),
    "pcgb_abi_sizes": (None, [POINTER(c_int32)]),
    "pcgb_last_error": (c_char_p, []),
    "pcgb_device_count": (c_int, []),
    "pcgb_csr_create": (c_int, [c_int64, c_int64, c_int64, c_void_p, c_int, c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    "pcgb_csr_destroy": (c_int, [c_void_p]),
    "pcgb_spmv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_csr_diag": (c_int, [c_void_p, c_void_p, c_void_p]),
    "pcgb_csr_release_col": (c_int, [c_void_p, c_void_p]),
    "pcgb_csr_set_boundary_rows": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "pcgb_spmv_split": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_spmv_bytes": (c_int64, [c_void_p]),
    "pcgb_spmv_stream_bytes": (c_int64, [c_void_p]),
    "pcgb_csr_plan_info": (c_int, [c_void_p, POINTER(c_int64)]),
    "pcgb_csr_value_dict": (c_int, [c_void_p]),
    "pcgb_csr_run_share": (c_double, [c_void_p]),
    "pcgb_csr_vd_plan": (c_int, [c_void_p, POINTER(c_int64)]),
    "pcgb_dot_w": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_axpby": (c_int, [c_int64, c_double, c_void_p, c_double, c_void_p, c_void_p]),
    "pcgb_mul": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_reciprocal": (c_int, [c_int64, c_void_p, c_void_p, c_void_p]),
    "pcgb_comm_unique_id": (c_int, [POINTER(c_ubyte)]),
    "pcgb_comm_create": (c_int, [c_int, c_int, POINTER(c_ubyte), POINTER(c_void_p)]),
    "pcgb_comm_destroy": (c_int, [c_void_p]),
    "pcgb_comm_window_export": (c_int, [c_void_p, POINTER(c_ubyte)]),
    "pcgb_comm_window_import": (c_int, [c_void_p, POINTER(c_ubyte)]),
    "pcgb_comm_transport": (c_int, [c_void_p]),
    "pcgb_comm_set_transport": (c_int, [c_void_p, c_int]),
    "pcgb_comm_status": (c_int, [c_void_p, c_void_p]),
    "pcgb_allreduce_sum": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "pcgb_halo_create": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int64), POINTER(c_int64), c_int64, POINTER(c_void_p)]),
    "pcgb_halo_destroy": (c_int, [c_void_p]),
    "pcgb_halo_blob_bytes": (c_int64, [c_void_p]),
    "pcgb_halo_export": (c_int, [c_void_p, POINTER(c_ubyte)]),
    "pcgb_halo_import": (c_int, [c_void_p, POINTER(c_ubyte)]),
    "pcgb_halo_exchange_add": (c_int, [c_void_p, c_void_p, c_void_p]),
    "pcgb_halo_bytes": (c_int64, [c_void_p]),
    "pcgb_solver_create": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    "pcgb_solver_destroy": (c_int, [c_void_p]),
    "pcgb_solve": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(Options), c_void_p, POINTER(Result), c_void_p]),
    "pcgb_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_solver_set_trace": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "pcgb_trace_record_bytes": (c_int64, []),
    "pcgb_ebe_create": (c_int, [c_int64, c_int, POINTER(EbeGroup), POINTER(c_void_p)]),
    "pcgb_ebe_destroy": (c_int, [c_void_p]),
    "pcgb_ebe_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_ebe_bytes": (c_int64, [c_void_p]),
    "pcgb_solver_create_ebe": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    "pcgb_ebe_ordered_create": (c_int, [c_int64, c_int, POINTER(EbeGroup), POINTER(c_void_p)]),
    "pcgb_ebe_ordered_destroy": (c_int, [c_void_p]),
    "pcgb_ebe_ordered_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_ebe_ordered_bytes": (c_int64, [c_void_p]),
    "pcgb_solver_create_ebe_ordered": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    "pcgb_assemble_symbolic": (c_int, [c_int64, c_int, POINTER(EbeGroup), c_void_p, POINTER(c_int64), c_void_p, POINTER(c_void_p)]),
    "pcgb_assemble_numeric": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_assemble_destroy": (c_int, [c_void_p]),
    "pcgb_ebe2_create": (c_int, [c_int64, c_int, POINTER(EbeGroup), POINTER(c_int32), POINTER(c_void_p)]),
    "pcgb_ebe2_destroy": (c_int, [c_void_p]),
    "pcgb_ebe2_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_ebe2_launches": (c_int, [c_void_p]),
    "pcgb_mg_create": (c_int, [c_void_p, POINTER(HexBox), POINTER(c_double), c_double, c_double, c_void_p, c_int, c_double, POINTER(c_void_p)]),
    "pcgb_mg_destroy": (c_int, [c_void_p]),
    "pcgb_mg_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_info": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_int64), POINTER(c_double), POINTER(c_int64)]),
    "pcgb_mg_restrict": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_prolong_add": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_smooth": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_coarse_solve": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_create_ranks": (c_int, [c_void_p, POINTER(HexBox), c_int, POINTER(c_void_p), c_void_p, POINTER(c_void_p), POINTER(c_double),
                                     c_double, c_double, c_void_p, c_int, c_double, POINTER(c_void_p)]),
    "pcgb_mg_create_field": (c_int, [c_void_p, POINTER(HexBox), POINTER(c_double), c_void_p, c_void_p, c_int, c_double, POINTER(c_void_p)]),
    "pcgb_mg_create_any": (c_int, [c_void_p, POINTER(HexBox), POINTER(c_double), c_void_p, c_double, c_double, c_void_p, c_int, c_double,
                                   POINTER(c_void_p)]),
    "pcgb_mg_level_box": (c_int, [c_void_p, c_int, POINTER(c_int32)]),
    "pcgb_mg_level_csr": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p]),
    "pcgb_mg_create_index_free": (c_int, [c_void_p, POINTER(HexBox), POINTER(c_double), c_double, c_double, c_void_p, c_int, c_double,
                                          POINTER(c_void_p)]),
    "pcgb_mg_create_ranks_index_free": (c_int, [c_void_p, POINTER(HexBox), c_int, POINTER(c_void_p), c_void_p, POINTER(c_void_p),
                                                POINTER(c_double), c_double, c_double, c_void_p, c_int, c_double, POINTER(c_void_p)]),
    "pcgb_mg_create_ranks_field": (c_int, [c_void_p, POINTER(HexBox), c_int, POINTER(c_void_p), c_void_p, c_void_p, POINTER(c_void_p),
                                           POINTER(c_double), c_void_p, c_void_p, c_int, c_double, POINTER(c_void_p)]),
    "pcgb_mg_create_field_rap": (c_int, [c_void_p, POINTER(HexBox), POINTER(c_double), c_void_p, c_void_p, c_int, c_double,
                                         POINTER(c_void_p)]),
    "pcgb_mg_create_ranks_field_rap": (c_int, [c_void_p, POINTER(HexBox), c_int, POINTER(c_void_p), c_void_p, c_void_p,
                                               POINTER(c_void_p), POINTER(c_double), c_void_p, c_void_p, c_int, c_double,
                                               POINTER(c_void_p)]),
    "pcgb_mg_level_dinv": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "pcgb_mg_level_apply": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_setup_info": (c_int, [c_void_p, POINTER(c_double), POINTER(c_int64)]),
    "pcgb_mg_info_ranks": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_int64)]),
    "pcgb_mg_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_mg_scatter": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_solve_mg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(Options), c_void_p, POINTER(Result), c_void_p]),
    "pcgb_hex_nrows": (c_int64, [POINTER(HexBox)]),
    "pcgb_hex_count": (c_int, [POINTER(HexBox), c_void_p, c_void_p]),
    "pcgb_hex_fill": (c_int, [POINTER(HexBox), POINTER(c_double), c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_hex_field_check": (c_int, [POINTER(HexBox), c_void_p, c_void_p]),
    "pcgb_hex_fill_field": (c_int, [POINTER(HexBox), POINTER(c_double), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_hexop_create": (c_int, [POINTER(HexBox), POINTER(c_double), c_double, c_void_p, POINTER(c_void_p)]),
    "pcgb_hexop_destroy": (c_int, [c_void_p]),
    "pcgb_hexop_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_hexop_diag": (c_int, [c_void_p, c_void_p, c_void_p]),
    "pcgb_hexop_bytes": (c_int64, [c_void_p]),
    "pcgb_solver_create_hexop": (c_int, [c_void_p, c_void_p, c_void_p, POINTER(c_void_p)]),
    "pcgb_hexop_create_periodic": (c_int, [POINTER(HexBox), POINTER(c_double), c_double, c_void_p, POINTER(c_void_p)]),
    "pcgb_hexop_periodic_load": (c_int, [c_void_p, POINTER(c_double), c_double, c_void_p, c_void_p]),
    "pcgb_fields_create": (c_int, [POINTER(HexBox), c_double, c_double, c_double, c_void_p, POINTER(c_void_p)]),
    "pcgb_fields_destroy": (c_int, [c_void_p]),
    "pcgb_fields_element": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_fields_nodal": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_fields_create_periodic": (c_int, [POINTER(HexBox), c_double, c_double, c_double, c_void_p, POINTER(c_void_p)]),
    "pcgb_fields_element_periodic": (c_int, [c_void_p, c_void_p, POINTER(c_double), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcgb_fields_average": (c_int, [c_void_p, c_void_p, POINTER(c_double), POINTER(c_double), POINTER(c_double), c_void_p]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load libpcgb200.so; raise loudly if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PcgbError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "or `make -C pcg_mpi_solver_b200/csrc` (there is no CPU/PyTorch fallback)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().pcgb_last_error()
        raise PcgbError(f"{what or 'libpcgb200'} failed ({rc}): {msg.decode() if msg else '?'}")


def ptr(t) -> int:
    """Device (or host) address of a torch tensor / numpy array, 0 for None."""
    if t is None:
        return 0
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def stream_ptr(stream=None) -> int:
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return s.cuda_stream
