"""Geometric multigrid preconditioner for hex-box operators (pcgb_mg_*, csrc/gmg.cuh), on one rank or across ranks.

`HexMultigrid(op, block)` builds, on the device, the hierarchy of nested boxes under `block` (the box `op`'s operator
was generated from, `hexmesh.generate_matrix` / `generate_ebe`): coarse matrices rediscretised at 2h, 4h, ... (equal to
the Galerkin products P^T A P for nested Q1 spaces), Chebyshev smoothers and a dense Cholesky factor of the coarsest
level.  Passing it as `M` to `SubdomainOperator.solve` / `solve` runs the same PCG loop with z = M r (one symmetric
V-cycle) instead of z = Minv .* r.  Its iteration count does not grow with the mesh, unlike Jacobi-PCG's.

Across ranks (`op` with a communicator of 2 or more ranks, `blocks` = every rank's box as `hexmesh.partition_blocks` returns
them): every rank halves its own box while all ranks can (`rank_levels`), with one halo plan and ownership weights per
level from `hexmesh.interface_lists`; the first level where some rank cannot halve is gathered onto every rank and continues
as the one-rank hierarchy of its global box.  The global boxes are those of the one-rank preconditioner on the global mesh,
so it is the same operator up to rounding.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, hex_element_stiffness, interface_lists

MAX_GATHERED = 1 << 17    # dofs of the largest global box gathered onto every rank (kMgMaxGathered)
MAX_COARSE = 1536         # dofs of the largest coarsest level (kMgMaxCoarse)


def _halve(b: HexBlock) -> HexBlock:
    return HexBlock(tuple(v // 2 for v in b.ng), tuple(v // 2 for v in b.e0), tuple(v // 2 for v in b.ne), h=2 * b.h, E=b.E, nu=b.nu)


def _whole_levels(ne):
    out = [tuple(int(v) for v in ne)]
    while all(v % 2 == 0 and v // 2 >= 2 for v in out[-1]):
        out.append(tuple(v // 2 for v in out[-1]))
    return out


def rank_levels(blocks) -> list:
    """Per-level box lists of a multi-rank hierarchy: [blocks, halved blocks, ...] up to the gathered level la (the last
    entry; la = len - 1).  Raises ValueError, identically on every rank (all hold the same `blocks`), when the boxes do
    not tile one mesh, the fine level cannot coarsen (la = 0), the gathered global box has more than 2^17 dofs or the
    coarsest level of the replicated hierarchy more than 1536."""
    blocks = list(blocks)
    ng = tuple(blocks[0].ng)
    cells = np.zeros(tuple(reversed(ng)), dtype=np.int32)
    for b in blocks:
        if tuple(b.ng) != ng or any(b.ne[a] <= 0 or b.e0[a] < 0 or b.e0[a] + b.ne[a] > ng[a] for a in range(3)):
            raise ValueError("HexMultigrid: every box must lie in the same global mesh")
        cells[b.e0[2]:b.e0[2] + b.ne[2], b.e0[1]:b.e0[1] + b.ne[1], b.e0[0]:b.e0[0] + b.ne[0]] += 1
    if not np.all(cells == 1):
        raise ValueError("HexMultigrid: the boxes do not tile the global mesh")
    levels = [blocks]
    while all(b.ne[a] % 2 == 0 and b.ne[a] >= 4 and b.e0[a] % 2 == 0 for b in levels[-1] for a in range(3)):
        levels.append([_halve(b) for b in levels[-1]])
    if len(levels) < 2:
        raise ValueError("HexMultigrid: the fine level does not coarsen on every rank (every ne even and >= 4, every e0 even)")
    g = levels[-1][0].ng
    n_gathered = 3 * g[0] * (g[1] + 1) * (g[2] + 1)
    if n_gathered > MAX_GATHERED:
        raise ValueError(f"HexMultigrid: the gathered level has {n_gathered} dofs (at most {MAX_GATHERED})")
    c = _whole_levels(g)[-1]
    if 3 * c[0] * (c[1] + 1) * (c[2] + 1) > MAX_COARSE:
        raise ValueError(f"HexMultigrid: the coarsest level has {3 * c[0] * (c[1] + 1) * (c[2] + 1)} dofs (at most {MAX_COARSE})")
    return levels


class HexMultigrid:
    """z = M r, one V-cycle.  op: a SubdomainOperator; block: its HexBlock; degree / lo: Chebyshev degree and the lower end
    of its interval as a fraction of the estimated largest eigenvalue of D^-1 A (the upper end is 1.1 times it).  minv: the
    fine level's inverse diagonal (op.jacobi() if omitted).

    One rank: block is the whole mesh (e0 = 0, ng = ne, every ne even).  Across ranks (op.comm with 2 or more ranks):
    blocks lists every rank's box and block is blocks[op.comm.rank]; construction is collective and refuses (ValueError,
    on every rank alike, before anything is allocated) what `rank_levels` refuses."""

    def __init__(self, op, block: HexBlock, degree: int = 2, lo: float = 0.25, minv: torch.Tensor | None = None, blocks=None):
        self.op, self.block, self.degree, self.lo = op, block, int(degree), float(lo)
        self.n = op.n
        self.device = op.device
        self._h = ctypes.c_void_p()
        self._halos = []
        self.levels = None
        comm = getattr(op, "comm", None)
        ranked = comm is not None and comm.nranks > 1
        if ranked:
            if blocks is None or len(blocks) != comm.nranks:
                raise ValueError("HexMultigrid: a multi-rank operator needs `blocks`, one box per rank")
            if blocks[comm.rank] != block:
                raise ValueError("HexMultigrid: block must be blocks[comm.rank]")
            if block.n != op.n:
                raise ValueError(f"HexMultigrid: the operator has {op.n} rows, the box {block.n}")
            self.levels = rank_levels(blocks)
        minv = op.jacobi() if minv is None else minv.to(self.device, torch.float64).contiguous()
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        box = block.cbox()
        lib = _lib.load()
        with torch.cuda.device(self.device):
            if not ranked:
                _lib.check(lib.pcgb_mg_create(op._solver, ctypes.byref(box), kep, float(block.E), float(block.h), _lib.ptr(minv),
                                              self.degree, self.lo, ctypes.byref(self._h)), "pcgb_mg_create")
                return
            from .solver import make_halo
            la = len(self.levels) - 1
            own = []
            for l, bl in enumerate(self.levels):
                nbr, lists, w = interface_lists(bl, comm.rank)
                own.append(torch.from_numpy(w).to(self.device))
                if l > 0:
                    self._halos.append(make_halo(comm, nbr, lists, bl[comm.rank].n))
            g = self.levels[-1][0].ng
            ngath = 3 * g[0] * (g[1] + 1) * (g[2] + 1)
            others = [r for r in range(comm.nranks) if r != comm.rank]
            all_dofs = np.arange(ngath, dtype=np.int64)
            self._gather = make_halo(comm, others, [all_dofs] * len(others), ngath)
            self._halos.append(self._gather)
            halos = (ctypes.c_void_p * la)(*[h.value for h in self._halos[:la]])
            owns = (ctypes.c_void_p * (la + 1))(*[t.data_ptr() for t in own])
            torch.cuda.synchronize(self.device)
            _lib.check(lib.pcgb_mg_create_ranks(op._solver, ctypes.byref(box), la, halos, self._gather, owns, kep,
                                                float(block.E), float(block.h), _lib.ptr(minv), self.degree, self.lo,
                                                ctypes.byref(self._h)), "pcgb_mg_create_ranks")

    @property
    def handle(self):
        return self._h

    def _vec(self, n):
        return torch.empty(n, dtype=torch.float64, device=self.device)

    def apply(self, r: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """z = M r (one V-cycle; collective across ranks)."""
        z = out if out is not None else self._vec(self.n)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_apply(self._h, _lib.ptr(r), _lib.ptr(z), _lib.stream_ptr()), "pcgb_mg_apply")
        return z

    def info(self) -> dict:
        """levels, n per level, largest-eigenvalue estimates of D^-1 A per level (0 for the coarsest and for the gathered
        level), device bytes; across ranks also gather_level (la, -1 on one rank), n_gathered and global_lambda (the
        estimates of the global hierarchy: ranked levels below la, then the replicated ones)."""
        lib = _lib.load()
        nl = ctypes.c_int32()
        n = (ctypes.c_int64 * _lib.MG_MAX_LEVELS)()
        lam = (ctypes.c_double * _lib.MG_MAX_LEVELS)()
        nb = ctypes.c_int64()
        _lib.check(lib.pcgb_mg_info(self._h, ctypes.byref(nl), n, lam, ctypes.byref(nb)), "pcgb_mg_info")
        la, ng = ctypes.c_int32(), ctypes.c_int64()
        _lib.check(lib.pcgb_mg_info_ranks(self._h, ctypes.byref(la), ctypes.byref(ng)), "pcgb_mg_info_ranks")
        k = nl.value
        lams = [float(v) for v in lam[:k]]
        out = {"levels": k, "n": [int(v) for v in n[:k]], "lambda": lams, "bytes": int(nb.value)}
        if la.value >= 0:
            out.update(gather_level=la.value, n_gathered=int(ng.value), global_lambda=lams[:la.value] + lams[la.value + 1:])
        return out

    # ---- the V-cycle's parts (tests; collective across ranks)
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

    def gather(self, v: torch.Tensor) -> torch.Tensor:
        """The gathered level's ranked vector -> its global box, the same on every rank."""
        out = self._vec(self.info()["n_gathered"])
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_gather(self._h, _lib.ptr(v), _lib.ptr(out), _lib.stream_ptr()), "pcgb_mg_gather")
        return out

    def scatter(self, g: torch.Tensor) -> torch.Tensor:
        """This rank's entries of a global vector of the gathered level."""
        info = self.info()
        out = self._vec(info["n"][info["gather_level"]])
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().pcgb_mg_scatter(self._h, _lib.ptr(g), _lib.ptr(out), _lib.stream_ptr()), "pcgb_mg_scatter")
        return out

    def __del__(self):
        try:
            lib = _lib.load()
            if self._h:
                lib.pcgb_mg_destroy(self._h)
                self._h = ctypes.c_void_p()
            for h in self._halos:          # the handle used them: destroyed after it
                lib.pcgb_halo_destroy(h)
            self._halos = []
        except Exception:
            pass
