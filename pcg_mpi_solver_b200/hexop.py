"""Opt-in index-free matrix-free operator of a hex box (csrc/hexop.cuh, pcgb_hexop_*): the reference's element-by-element
product (calcMatVecProd, pcg_solver.py:263-300) on a structured box, with every index computed from the node's
coordinates.  Its products and its diagonal are bit-identical to `EbeMatrixOrdered` on the same box
(`hexmesh.generate_ebe(block, ordered=True)`), so solves on it give the ordered operator's x, residuals and trace; it holds
no index list, slot buffer or position list, only the box, Ke and (with a field) the caller's Ck per element.

`hexmesh.generate_box_operator(block, device, E_field)` builds it; it has the EbeMatrix interface (shape, device, handle,
apply_local / spmv, diagonal, spmv_bytes) and is accepted by `SubdomainOperator` and `multigrid.HexMultigrid`.

`hexmesh.generate_periodic_operator(cell, device, E_field)` builds the same operator on a periodic cell
(`PeriodicCellOperator`, DESIGN §2.13), which `SubdomainOperator` accepts and `HexMultigrid` refuses.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, PeriodicCell, _same_device, field_ck, hex_element_stiffness


class HexBoxOperator:
    """K_i[Eff,Eff] of `block` applied without indices.  E_field: one Young's modulus per element (as generate_matrix);
    Ck = E_field * h, kept on the device for the operator's lifetime (8 bytes per element)."""

    def __init__(self, block: HexBlock, device="cuda", E_field=None):
        self.block = block
        self.device = torch.device(device)
        n = int(block.n)
        self.shape = (n, n)
        self._ck = None if E_field is None else field_ck(E_field, block, self.device)
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        box = block.cbox()
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_hexop_create(ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                     float(block.E * block.h), _lib.ptr(self._ck), ctypes.byref(self._h)),
                       "pcgb_hexop_create")

    @property
    def handle(self):
        return self._h

    def apply_local(self, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """y = K_i x, no interface sum (x and out must not overlap)."""
        y = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_hexop_apply(self._h, _lib.ptr(x), _lib.ptr(y), _lib.stream_ptr()), "pcgb_hexop_apply")
        return y

    spmv = apply_local

    def diagonal(self) -> torch.Tensor:
        """The local diagonal, summed as EbeMatrix does (pcg_solver.py:282-287), computed on the device."""
        d = torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_hexop_diag(self._h, _lib.ptr(d), _lib.stream_ptr()), "pcgb_hexop_diag")
        return d

    def spmv_bytes(self) -> int:
        return int(_lib.load().pcgb_hexop_bytes(self._h))

    def __del__(self):
        try:
            if self._h:
                _lib.load().pcgb_hexop_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass


class PeriodicCellOperator(HexBoxOperator):
    """K of a periodic cell (hexmesh.PeriodicCell) applied without indices: every node free, coordinates wrapped, each row
    in the box operator's order with all 8 elements present (pcgb_hexop_create_periodic).  K is singular: its null space
    is the three rigid translations.  PCG from x0 = 0 on a right-hand side in K's range (as `load` gives, whose entries
    sum to 0 per direction mathematically) converges to a solution determined up to a translation, on which no strain or
    stress depends.  E_field: one Young's modulus per element, shape (ne[2], ne[1], ne[0]); Ck = E_field * h."""

    def __init__(self, cell: PeriodicCell, device="cuda", E_field=None):
        self.block = cell
        self.device = torch.device(device)
        n = int(cell.n)
        self.shape = (n, n)
        self._ck = None if E_field is None else field_ck(E_field, cell, self.device)
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, cell.nu))
        box = cell.cbox()
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_hexop_create_periodic(ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                              float(cell.E * cell.h), _lib.ptr(self._ck), ctypes.byref(self._h)),
                       "pcgb_hexop_create_periodic")

    def load(self, strain, out: torch.Tensor | None = None) -> torch.Tensor:
        """b = -K u_bar for the macroscopic strain `strain` (6 values, Voigt 11, 22, 33, 23, 13, 12 with engineering
        shears), u_bar = strain x taken relative to each node computed (pcgb_hexop_periodic_load)."""
        e = np.ascontiguousarray(strain, dtype=np.float64)
        if e.shape != (6,):
            raise ValueError(f"load: strain must have 6 Voigt components, got shape {e.shape}")
        if out is not None and not (isinstance(out, torch.Tensor) and out.dtype == torch.float64 and out.dim() == 1
                                    and out.numel() == self.shape[0] and out.is_contiguous() and out.device.type == "cuda"
                                    and _same_device(out.device, self.device)):
            raise ValueError(f"load: out must be a contiguous float64 vector of the cell's {self.shape[0]} dofs on {self.device}")
        b = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_hexop_periodic_load(self._h, e.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                            float(self.block.h), _lib.ptr(b), _lib.stream_ptr()),
                       "pcgb_hexop_periodic_load")
        return b
