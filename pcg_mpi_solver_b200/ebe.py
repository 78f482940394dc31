"""Opt-in matrix-free element-by-element operator (SURVEY.md 8(f1)) - the reference's own operator form
(calcMatVecProd, pcg_solver.py:263-300) on the GPU instead of the assembled CSR matrix.

Status: parity-green (tests/test_gpu_ebe.py: hex vs CSR/oracle, concrete vs the reference's 1085 iterations, several
live operators with different pattern matrices; synthetic pattern groups at every kernel edge - pattern sizes 1..96,
block tails, signs, clamped and high-valence dofs - entrywise against a long-double reference, constant-memory slot
overflow and sharing, the EBE solver against the oracle and generate_ebe on every bench box; tests/test_gpu_multi.py:
the EBE operator across ranks); timing: `bench.py --operator ebe`.  Scatter-adds with fp64 atomics
(reproducible to rounding only); `EbeMatrixColored` is the bit-reproducible coloured variant (3x slower).  `to_operator(kind="ebe")`.

`EbeMatrixOrdered` (`to_operator(kind="ebe_ordered")`) is the same operator in the reference's own two phases - element
products into a slot buffer laid out like `Flat`, then a per-dof sum in ascending slot position (csrc/ebe_ordered.cuh,
include/pcgb200.h) - with no atomics in the arithmetic: bit-reproducible, and usable in the PCG solve like EbeMatrix.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib


class EbeMatrix:
    """Pattern groups of one subdomain on the device, indices in the free-dof numbering (-1 = clamped)."""

    _fn = ("pcgb_ebe_create", "pcgb_ebe_apply", "pcgb_ebe_bytes", "pcgb_ebe_destroy")   # C entry points of this operator
    _symmetric_only = True    # the warp kernel reads column i of Ke for row i

    def __init__(self, groups, loc_dof_eff: np.ndarray, ndof: int, device="cuda"):
        self.device = torch.device(device)
        n = int(len(loc_dof_eff))
        self.shape = (n, n)
        eff_map = np.full(ndof, -1, dtype=np.int32)
        eff_map[loc_dof_eff] = np.arange(n, dtype=np.int32)
        self._keep = []          # device tensors and host arrays the C side points into
        cgroups = (_lib.EbeGroup * len(groups))()
        diag = np.zeros(n)
        self.nnz_equivalent = 0
        for k, g in enumerate(groups):
            nd, ne = g.loc_dof.shape
            idx = eff_map[g.loc_dof].astype(np.int32)                       # (nd, ne)
            ke = np.ascontiguousarray(g.ke, dtype=np.float64)
            if self._symmetric_only and not np.allclose(ke, ke.T, rtol=1e-12, atol=1e-12 * np.abs(ke).max()):
                raise ValueError("EbeMatrix: pattern matrices must be symmetric")
            d_idx = torch.from_numpy(np.ascontiguousarray(idx)).to(self.device)
            d_ck = torch.from_numpy(np.ascontiguousarray(g.ck, dtype=np.float64)).to(self.device)
            d_sign = torch.from_numpy(np.ascontiguousarray(g.sign.astype(np.uint8))).to(self.device) if g.sign.any() else None
            self._keep += [d_idx, d_ck, d_sign, ke]
            cg = cgroups[k]
            cg.nd, cg.ne = nd, ne
            cg.d_idx, cg.d_ck = d_idx.data_ptr(), d_ck.data_ptr()
            cg.d_sign = d_sign.data_ptr() if d_sign is not None else None
            cg.ke_host = ke.ctypes.data
            # diagonal for the Jacobi preconditioner: sum_e Ck * diag(Ke)  (pcg_solver.py:282-287); signs cancel (s_i^2 = 1)
            contrib = (g.ck[None, :] * np.diag(ke)[:, None]).ravel()
            flat = idx.ravel()
            ok = flat >= 0
            diag += np.bincount(flat[ok], weights=contrib[ok], minlength=n)
            self.nnz_equivalent += int(nd) * int(nd) * int(ne)
        self._diag = diag
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.load(), self._fn[0])(n, len(groups), cgroups, ctypes.byref(self._h)), self._fn[0])

    @property
    def handle(self):
        return self._h

    def apply_local(self, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """y = K_i x, no interface sum."""
        y = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.load(), self._fn[1])(self._h, _lib.ptr(x), _lib.ptr(y), _lib.stream_ptr()), self._fn[1])
        return y

    spmv = apply_local

    def diagonal(self) -> torch.Tensor:
        return torch.from_numpy(self._diag).to(self.device)

    def spmv_bytes(self) -> int:
        return int(getattr(_lib.load(), self._fn[2])(self._h))

    def __del__(self):
        try:
            if self._h:
                getattr(_lib.load(), self._fn[3])(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass


class EbeMatrixOrdered(EbeMatrix):
    """The EbeMatrix operator with a fixed summation order: element products into a slot buffer laid out like the
    reference's `Flat` (slot = off_g + a*ne_g + e), then every dof sums its slots in ascending position, i.e. in
    (group, local index, element) order - what np.bincount does (pcg_solver.py:300).  Bit-reproducible; the PCG solve
    accepts it like EbeMatrix.  Pattern matrices need not be symmetric.  Costs 8 B per element slot and 4 B per free slot of device memory on top."""

    _fn = ("pcgb_ebe_ordered_create", "pcgb_ebe_ordered_apply", "pcgb_ebe_ordered_bytes", "pcgb_ebe_ordered_destroy")
    _symmetric_only = False   # both kernels read Ke by rows, as Ke @ (Ck * U) does


class EbeMatrixColored:
    """Operator-level variant (tests/test_gpu_ebe_colored.py, tests/test_gpu_ebe_color_edges.py): the same operator with
    an atomics-free, bit-reproducible scatter.  All elements of the subdomain are coloured together
    (coloring.color_groups: on the node of every local dof, so that no two elements of a colour share a dof), every
    (pattern group, colour) slice becomes its own group, slices are passed in colour order and the kernels of one colour
    use plain `y[dof] += v` (csrc/ebe_color.cuh).

    The result, bit for bit (include/pcgb200.h): every free dof d starts from +0.0; the colours are taken in ascending
    order, and for the one element e of that colour that touches d, every local index i with idx[i] = d, in ascending i,
    does y_d = y_d + v_{e,i}, with u_j = s_j x_j (0.0 for a clamped dof), acc = fma(Ke[i][j], u_j, acc) over j ascending
    from 0.0, and v_{e,i} = round(acc * Ck_e), negated when s_i is set.

    `colors_per_group` (one integer array of ne_g colours per group) replaces the computed colouring.  Either colouring is
    checked before anything reaches the device: ValueError when two different elements of one colour touch the same
    free dof (an element may list a dof more than once), and ValueError for a pattern matrix that is not symmetric, as
    EbeMatrix.  pcgb_ebe2_create itself trusts the phases it is given."""

    def __init__(self, groups, loc_dof_eff: np.ndarray, ndof: int, device="cuda", colors_per_group=None):
        from .coloring import color_conflicts, color_groups
        self.device = torch.device(device)
        n = int(len(loc_dof_eff))
        self.shape = (n, n)
        eff_map = np.full(ndof, -1, dtype=np.int32)
        eff_map[loc_dof_eff] = np.arange(n, dtype=np.int32)
        for g in groups:
            ke = np.asarray(g.ke, dtype=np.float64)
            if not np.allclose(ke, ke.T, rtol=1e-12, atol=1e-12 * np.abs(ke).max()):
                raise ValueError("EbeMatrixColored: pattern matrices must be symmetric")
        if colors_per_group is None:
            colors_per_group, ncolors = color_groups(groups, ndof)
        else:
            colors_per_group = [np.asarray(c) for c in colors_per_group]
            if len(colors_per_group) != len(groups) or any(c.shape != (g.loc_dof.shape[1],) or (c.size and (c.dtype.kind not in "iu" or c.min() < 0))
                                                           for g, c in zip(groups, colors_per_group)):
                raise ValueError("EbeMatrixColored: colors_per_group needs one array of non-negative integer colours per element of every group")
            ncolors = int(max([int(c.max()) for c in colors_per_group if c.size], default=-1) + 1)
        idx_per_group = [eff_map[g.loc_dof] for g in groups]
        bad = color_conflicts(idx_per_group, colors_per_group, n)
        if bad:
            raise ValueError(f"EbeMatrixColored: {bad} free dofs are touched by two elements of one colour")
        self.ncolors = ncolors
        self._keep = []
        entries = []     # (colour, nd, ne, d_idx, d_sign, d_ck, ke)
        for g, col, idx_all in zip(groups, colors_per_group, idx_per_group):
            ke = np.ascontiguousarray(g.ke, dtype=np.float64)   # ONE array per pattern group: its address identifies the pattern
            self._keep.append(ke)
            has_sign = bool(g.sign.any())
            for c in range(ncolors):
                sel = np.nonzero(col == c)[0]
                if sel.size == 0:
                    continue
                d_idx = torch.from_numpy(np.ascontiguousarray(idx_all[:, sel])).to(self.device)
                d_ck = torch.from_numpy(np.ascontiguousarray(g.ck[sel], dtype=np.float64)).to(self.device)
                d_sign = torch.from_numpy(np.ascontiguousarray(g.sign[:, sel].astype(np.uint8))).to(self.device) if has_sign else None
                self._keep += [d_idx, d_ck, d_sign]
                entries.append((c, g.loc_dof.shape[0], sel.size, d_idx, d_sign, d_ck, ke))
        entries.sort(key=lambda t: t[0])                        # stable: colour order, pattern groups in their order inside a colour
        cgroups = (_lib.EbeGroup * len(entries))()
        phase = (ctypes.c_int32 * len(entries))()
        for k, (c, nd, ne, d_idx, d_sign, d_ck, ke) in enumerate(entries):
            cg = cgroups[k]
            cg.nd, cg.ne = nd, ne
            cg.d_idx, cg.d_ck = d_idx.data_ptr(), d_ck.data_ptr()
            cg.d_sign = d_sign.data_ptr() if d_sign is not None else None
            cg.ke_host = ke.ctypes.data
            phase[k] = c
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_ebe2_create(n, len(entries), cgroups, phase, ctypes.byref(self._h)), "pcgb_ebe2_create")

    def apply_local(self, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        y = out if out is not None else torch.empty(self.shape[0], dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_ebe2_apply(self._h, _lib.ptr(x), _lib.ptr(y), _lib.stream_ptr()), "pcgb_ebe2_apply")
        return y

    def launches(self) -> int:
        return int(_lib.load().pcgb_ebe2_launches(self._h))

    def __del__(self):
        try:
            if self._h:
                _lib.load().pcgb_ebe2_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass
