"""Device-resident CSR operator: the assembled stiffness matrix A = K[Eff,Eff] of one subdomain.

Reference: the operator of the hot path is calcMatVecProd(..., 'Strain') (pcg_solver.py:242-300),
an element-by-element product that is never assembled; BASELINE.json's north star prescribes the
assembled CSR form, so the subdomain builder (partition.py) assembles exactly
K = sum_e P_e^T (Ck_e S_e Ke S_e) P_e and this class hands it to the merge-path SpMV kernel.

PyTorch tensors are used only as device-memory holders (data_ptr()).
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib


class CsrMatrix:
    """fp64 values, int32 column indices, int32 or int64 row offsets, all on one CUDA device."""

    def __init__(self, rowptr: torch.Tensor, col: torch.Tensor, val: torch.Tensor, shape):
        if not (rowptr.is_cuda and col.is_cuda and val.is_cuda):
            raise _lib.PcgbError("CsrMatrix needs CUDA tensors (libpcgb200 has no CPU path)")
        if rowptr.dtype not in (torch.int32, torch.int64) or col.dtype != torch.int32 or val.dtype != torch.float64:
            raise TypeError("CsrMatrix: rowptr int32/int64, col int32, val float64")
        self.rowptr, self.col, self.val = rowptr.contiguous(), col.contiguous(), val.contiguous()
        self.shape = (int(shape[0]), int(shape[1]))
        self.nnz = int(val.numel())
        self.device = val.device
        self._h = ctypes.c_void_p()
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.pcgb_csr_create(self.shape[0], self.shape[1], self.nnz, _lib.ptr(self.rowptr),
                                           1 if rowptr.dtype == torch.int64 else 0, _lib.ptr(self.col),
                                           _lib.ptr(self.val), _lib.stream_ptr(), ctypes.byref(self._h)),
                       "pcgb_csr_create")

    # ---- construction helpers --------------------------------------------------------------
    @classmethod
    def from_scipy(cls, A, device="cuda", index64=None):
        A = A.tocsr()
        A.sort_indices()
        use64 = bool(index64) if index64 is not None else A.nnz >= 2**31
        rp = torch.from_numpy(A.indptr.astype(np.int64 if use64 else np.int32)).to(device)
        col = torch.from_numpy(A.indices.astype(np.int32)).to(device)
        val = torch.from_numpy(np.ascontiguousarray(A.data, dtype=np.float64)).to(device)
        return cls(rp, col, val, A.shape)

    # ---- operations ------------------------------------------------------------------------
    @property
    def handle(self):
        return self._h

    def spmv(self, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """y = A x through the merge-path kernel."""
        assert x.is_cuda and x.dtype == torch.float64 and x.numel() == self.shape[1]
        y = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_spmv(self._h, _lib.ptr(x), _lib.ptr(y), _lib.stream_ptr()), "pcgb_spmv")
        return y

    def diagonal(self) -> torch.Tensor:
        d = torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_csr_diag(self._h, _lib.ptr(d), _lib.stream_ptr()), "pcgb_csr_diag")
        return d

    def spmv_bytes(self) -> int:
        """Algorithmic bytes of one SpMV (SURVEY 8(d)): 12 nnz + R (n+1) + 8 ncols + 8 nrows."""
        return int(_lib.load().pcgb_spmv_bytes(self._h))

    def stream_bytes(self) -> int:
        """HBM bytes the selected kernel streams per SpMV (10 B/nnz for the staged-x kernel)."""
        return int(_lib.load().pcgb_spmv_stream_bytes(self._h))

    def plan_info(self) -> dict:
        info = (ctypes.c_int64 * 16)()
        _lib.check(_lib.load().pcgb_csr_plan_info(self._h, info))
        # index_mode: 0 = one 16-bit staged position (or 32-bit column) per non-zero, 1 = per column triple, 2 = per 3x3 node block
        keys = ["ntiles", "tile_items", "lanes", "snap", "split_rows", "smem_bytes", "max_row", "tma", "staged", "x_windows",
                "x_cap", "max_windows_per_tile", "index_mode", "interface_tiles", "resident_ctas", "col_released"]
        return dict(zip(keys, [int(v) for v in info]))

    def value_dict_blocks(self) -> int:
        """Distinct 3x3 blocks in the node-block kernel's value dictionary (0: the kernel streams the values)."""
        return int(_lib.load().pcgb_csr_value_dict(self._h))

    def value_dict_run_share(self) -> float:
        """Share of the nodes whose blocks the dictionary kernel reads through the head of a run (consecutive nodes of a
        tile with the same blocks shifted by one node: a structured mesh along x); 0.0 without a dictionary."""
        return float(_lib.load().pcgb_csr_run_share(self._h))

    def value_dict_plan(self) -> dict:
        """The ring of the dictionary kernel (pcgb_csr_vd_plan); every field 0 without a dictionary."""
        out = (ctypes.c_int64 * 8)()
        _lib.check(_lib.load().pcgb_csr_vd_plan(self._h, out))
        keys = ["stages", "group", "producers", "consumers", "cap_words", "nvwords", "cap_nodes", "ctas_per_sm"]
        return dict(zip(keys, [int(v) for v in out]))

    def release_col(self) -> bool:
        """Free the 4-byte column array when the selected SpMV kernel does not read it (the persistent staged-x kernel
        streams its own 16-bit indices): 2 GB at 128^3, 16 GB at 256^3.  The diagonal is cached first.  Returns True
        when the array was released; to_scipy() is not available afterwards."""
        if self.col is None:
            return True
        with torch.cuda.device(self.device):
            rc = _lib.load().pcgb_csr_release_col(self._h, _lib.stream_ptr())
        if rc != 0:
            return False
        self.col = None
        return True

    def set_boundary_rows(self, rows: torch.Tensor) -> None:
        """Register the interface rows (int32 CUDA tensor) for the interface-first split (see pcgb_csr_set_boundary_rows)."""
        assert rows.is_cuda and rows.dtype == torch.int32
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_csr_set_boundary_rows(self._h, _lib.ptr(rows), rows.numel(), _lib.stream_ptr()),
                       "pcgb_csr_set_boundary_rows")

    def spmv_split(self, x: torch.Tensor, with_dot: bool = False, out: torch.Tensor | None = None):
        """y = A x as two launches (interface tiles first); returns y or (y, x.y)."""
        y = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        d = torch.zeros(1, dtype=torch.float64, device=self.device) if with_dot else None
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_spmv_split(self._h, _lib.ptr(x), _lib.ptr(y), _lib.ptr(d), _lib.stream_ptr()), "pcgb_spmv_split")
        return (y, d) if with_dot else y

    def to_scipy(self):
        import scipy.sparse as sp
        if self.col is None:
            raise _lib.PcgbError("CsrMatrix.to_scipy: the column array was released (release_col)")
        return sp.csr_matrix((self.val.cpu().numpy(), self.col.cpu().numpy(), self.rowptr.cpu().numpy()), shape=self.shape)

    def __del__(self):
        try:
            if self._h:
                _lib.load().pcgb_csr_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass
