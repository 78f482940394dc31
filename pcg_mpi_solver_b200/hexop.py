"""Opt-in index-free matrix-free operator of a hex box (csrc/hexop.cuh, pcgb_hexop_*): the reference's element-by-element
product (calcMatVecProd, pcg_solver.py:263-300) on a structured box, with every index computed from the node's
coordinates.  Its products and its diagonal are bit-identical to `EbeMatrixOrdered` on the same box
(`hexmesh.generate_ebe(block, ordered=True)`), so solves on it give the ordered operator's x, residuals and trace; it holds
no index list, slot buffer or position list, only the box, Ke and (with a field) the caller's Ck per element.

`hexmesh.generate_box_operator(block, device, E_field)` builds it; it has the EbeMatrix interface (shape, device, handle,
apply_local / spmv, diagonal, spmv_bytes) and is accepted by `SubdomainOperator` and `multigrid.HexMultigrid`.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, field_ck, hex_element_stiffness


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
