"""Geometric multigrid preconditioner for one-rank hex-box operators (pcgb_mg_*, csrc/gmg.cuh).

`HexMultigrid(op, block)` builds, on the device, the hierarchy of nested boxes under `block` (the box `op`'s operator
was generated from, `hexmesh.generate_matrix` / `generate_ebe`): coarse matrices rediscretised at 2h, 4h, ... (equal to
the Galerkin products P^T A P for nested Q1 spaces), Chebyshev smoothers and a dense Cholesky factor of the coarsest
level.  Passing it as `M` to `SubdomainOperator.solve` / `solve` runs the same PCG loop with z = M r (one symmetric
V-cycle) instead of z = Minv .* r.  Its iteration count does not grow with the mesh, unlike Jacobi-PCG's.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, hex_element_stiffness


class HexMultigrid:
    """z = M r, one V-cycle.  op: a one-rank SubdomainOperator; block: its HexBlock (e0 = 0, ng = ne, every ne even);
    degree / lo: Chebyshev degree and the lower end of its interval as a fraction of the estimated largest eigenvalue of
    D^-1 A (the upper end is 1.1 times it).  minv: the fine level's inverse diagonal (op.jacobi() if omitted)."""

    def __init__(self, op, block: HexBlock, degree: int = 2, lo: float = 0.25, minv: torch.Tensor | None = None):
        self.op, self.block, self.degree, self.lo = op, block, int(degree), float(lo)
        self.n = op.n
        self.device = op.device
        self._h = ctypes.c_void_p()
        minv = op.jacobi() if minv is None else minv.to(self.device, torch.float64).contiguous()
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        box = block.cbox()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_create(op._solver, ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                  float(block.E), float(block.h), _lib.ptr(minv), self.degree, self.lo,
                                                  ctypes.byref(self._h)), "pcgb_mg_create")

    @property
    def handle(self):
        return self._h

    def _vec(self, n):
        return torch.empty(n, dtype=torch.float64, device=self.device)

    def apply(self, r: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """z = M r (one V-cycle)."""
        z = out if out is not None else self._vec(self.n)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_apply(self._h, _lib.ptr(r), _lib.ptr(z), _lib.stream_ptr()), "pcgb_mg_apply")
        return z

    def info(self) -> dict:
        """levels, n per level, largest-eigenvalue estimates of D^-1 A per level (0 for the coarsest), device bytes."""
        nl = ctypes.c_int32()
        n = (ctypes.c_int64 * _lib.MG_MAX_LEVELS)()
        lam = (ctypes.c_double * _lib.MG_MAX_LEVELS)()
        nb = ctypes.c_int64()
        _lib.check(_lib.load().pcgb_mg_info(self._h, ctypes.byref(nl), n, lam, ctypes.byref(nb)), "pcgb_mg_info")
        k = nl.value
        return {"levels": k, "n": [int(v) for v in n[:k]], "lambda": [float(v) for v in lam[:k]], "bytes": int(nb.value)}

    # ---- the V-cycle's parts (tests)
    def restrict(self, level: int, rf: torch.Tensor) -> torch.Tensor:
        rc = self._vec(self.info()["n"][level + 1])
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_restrict(self._h, level, _lib.ptr(rf), _lib.ptr(rc), _lib.stream_ptr()), "pcgb_mg_restrict")
        return rc

    def prolong_add(self, level: int, ec: torch.Tensor, xf: torch.Tensor) -> torch.Tensor:
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_prolong_add(self._h, level, _lib.ptr(ec), _lib.ptr(xf), _lib.stream_ptr()), "pcgb_mg_prolong_add")
        return xf

    def smooth(self, level: int, b: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
        """x += S (b - A x) on `level`, in place."""
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_smooth(self._h, level, _lib.ptr(b), _lib.ptr(x), _lib.stream_ptr()), "pcgb_mg_smooth")
        return x

    def coarse_solve(self, r: torch.Tensor) -> torch.Tensor:
        z = self._vec(r.numel())
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_coarse_solve(self._h, _lib.ptr(r), _lib.ptr(z), _lib.stream_ptr()), "pcgb_mg_coarse_solve")
        return z

    def __del__(self):
        try:
            if self._h:
                _lib.load().pcgb_mg_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass
