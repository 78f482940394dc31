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

`E_field` (a voxel model, one Young's modulus per element) makes every coarse level a Galerkin product of element matrices,
on one rank (pcgb_mg_create_field) and across ranks (pcgb_mg_create_ranks_field).  Across ranks E_field is the field of the
whole mesh: each rank builds the element matrices of its own boxes, the gathered level's matrices are collected onto every
rank (at most MAX_GATHERED_ELEMENTS elements), and the replicated levels are the one-rank field hierarchy's bit for bit.

`coarsening="any"` (one rank) accepts a box of any size: every axis is coarsened on its own (`any_levels`), halved to
(ne + 1) / 2 elements while ne >= 3 and kept once ne <= 2, down to at most 2x2x2 elements, and the coarse levels are always
Galerkin products of element matrices (pcgb_mg_create_any), with or without `E_field`.

`coarse="index_free"` (default coarsening, no `E_field`; one rank or across ranks) builds the same hierarchy with every
smoothed coarse level applied by the index-free hex-box operator (csrc/hexop.cuh) instead of a CSR matrix
(pcgb_mg_create_index_free / pcgb_mg_create_ranks_index_free): the hierarchy then holds only vectors and the coarsest
factor (`index_free_bytes`), which is what lets MG-PCG run a 512^3 box on one 80 GB GPU.

`coarse="rap"` (one rank, default coarsening, with `E_field`) is the field hierarchy with a matrix-free level 1
(pcgb_mg_create_field_rap): level 1 applies P^T A_0 P from the fine Ck field in one kernel (csrc/gmg_rap.cuh) and levels >= 2
are the field hierarchy's CSR levels bit for bit, built from slabs of level-1 element matrices that are never held whole
(`rap_bytes`, `rap_setup_peak_bytes`).  It preconditions a 512^3 voxel model on one 80 GB GPU, where the CSR field
hierarchy's level 1 alone would take about 49 GB.  Across ranks (`blocks` and the global E_field,
pcgb_mg_create_ranks_field_rap) it is the multi-rank field hierarchy with the same matrix-free level 1 on every rank's
level-1 box, from the rank's slice of the field (`rap_rank_bytes`); the rank boxes must halve at least twice.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .hexmesh import HexBlock, PeriodicCell, block_field, check_field, field_ck, hex_element_stiffness, interface_lists

MAX_GATHERED = 1 << 17    # dofs of the largest global box gathered onto every rank (kMgMaxGathered)
MAX_COARSE = 1536         # dofs of the largest coarsest level (kMgMaxCoarse)
MAX_GATHERED_ELEMENTS = 4096   # elements of the gathered global box of a multi-rank field hierarchy (kMgMaxGatheredElements)
RAP_SLAB_BYTES = 1 << 30       # largest slab of level-1 element matrices a rap set-up holds (kMgRapSlabBytes)
ELEMENT_MATRIX_BYTES = 576 * 8


def _halve(b: HexBlock) -> HexBlock:
    return HexBlock(tuple(v // 2 for v in b.ng), tuple(v // 2 for v in b.e0), tuple(v // 2 for v in b.ne), h=2 * b.h, E=b.E, nu=b.nu)


def _whole_levels(ne):
    out = [tuple(int(v) for v in ne)]
    while all(v % 2 == 0 and v // 2 >= 2 for v in out[-1]):
        out.append(tuple(v // 2 for v in out[-1]))
    return out


def any_levels(ne, max_levels: int = _lib.MG_MAX_LEVELS) -> list:
    """Element counts of every level under coarsening="any": an axis with ne >= 3 becomes (ne + 1) / 2 (coarse node j at
    fine node min(2j, ne)), one with ne <= 2 is kept, while some axis has ne >= 3.  Raises ValueError, as pcgb_mg_create_any
    refuses, for a box with nothing to coarsen or a hierarchy of more than `max_levels` levels."""
    out = [tuple(int(v) for v in ne)]
    while any(v >= 3 for v in out[-1]):
        out.append(tuple((v + 1) // 2 if v >= 3 else v for v in out[-1]))
        if len(out) > max_levels:
            raise ValueError(f"HexMultigrid: the box {tuple(ne)} needs more than {max_levels} levels")
    if len(out) < 2:
        raise ValueError(f"HexMultigrid: the box {tuple(ne)} does not coarsen (some ne must be >= 3)")
    return out


def _whole_box_levels(ne):
    """The default coarsening's levels of the whole box ne and their free dofs, refused (ValueError) as pcgb_mg_create
    refuses the box."""
    lv = _whole_levels(ne)
    if len(lv) < 2:
        raise ValueError(f"HexMultigrid: the box {tuple(ne)} does not coarsen (every ne must be even and >= 4)")
    n = [3 * v[0] * (v[1] + 1) * (v[2] + 1) for v in lv]
    if n[-1] > MAX_COARSE:
        raise ValueError(f"HexMultigrid: the coarsest level has {n[-1]} dofs (at most {MAX_COARSE})")
    return lv, n


def index_free_bytes(ne) -> int:
    """Device bytes pcgb_mg_info reports for the one-rank index-free hierarchy of the whole box `ne` (default coarsening):
    8 (5 n_0 + 6 sum n_l over the smoothed coarse levels + 2 n_c + n_c^2) - the fine level's z, D^-1 and three smoother
    vectors, each coarse level's b, x, D^-1 and three smoother vectors, the coarsest b, x and dense factor.  The few
    fixed-size reduction buffers are not counted.  Raises ValueError where pcgb_mg_create_index_free refuses the box."""
    _, n = _whole_box_levels(ne)
    return 8 * (5 * n[0] + 6 * sum(n[1:-1]) + 2 * n[-1] + n[-1] ** 2)


def _rap_levels(ne):
    """The default coarsening's levels and free dofs, refused (ValueError) as pcgb_mg_create_field_rap refuses the box."""
    lv, n = _whole_box_levels(ne)
    if len(lv) < 3:
        raise ValueError(f"HexMultigrid: coarse='rap' needs at least 3 levels, the box {tuple(ne)} has {len(lv)} "
                         "(level 1 would be the coarsest)")
    return lv, n


def hex_csr_nnz(ne, x_lo: int = 1) -> int:
    """Non-zeros of the clamped stiffness matrix of the whole box ne (x = 0 nodes dropped): 9 times the free neighbour pairs,
    which factor per axis into 3 m - 2 for an axis of m free nodes (nx on x, ny + 1 and nz + 1 on y and z).  x_lo = 0: the
    sub-assembled matrix of a rank's box away from x = 0 (HexBlock.x_lo), nx + 1 free nodes on x."""
    return 9 * (3 * (ne[0] + 1 - x_lo) - 2) * (3 * (ne[1] + 1) - 2) * (3 * (ne[2] + 1) - 2)


def _csr_bytes(ne, n, x_lo: int = 1) -> int:
    """Device bytes of a coarse level's CSR: 12 nnz + 4 (n + 1) (8 (n + 1) from 2^31 - 1 non-zeros on, int64 row offsets)."""
    nnz = hex_csr_nnz(ne, x_lo)
    return 12 * nnz + (4 if nnz < 2**31 - 1 else 8) * (n + 1)


def rap_bytes(ne) -> int:
    """Device bytes pcgb_mg_info reports for the rap hierarchy of the whole box `ne`: the vectors of `index_free_bytes`,
    plus levels 2 .. L-2 as CSR, 12 nnz + 4 (n + 1) bytes each (8 (n + 1) from 2^31 - 1 non-zeros on, int64 row offsets).
    Raises ValueError where pcgb_mg_create_field_rap refuses the box."""
    lv, n = _rap_levels(ne)
    return index_free_bytes(ne) + sum(_csr_bytes(lv[l], n[l]) for l in range(2, len(lv) - 1))


def rap_setup_peak_bytes(ne) -> int:
    """Peak bytes of element matrices a rap set-up holds (pcgb_mg_setup_info): level 2's, plus the larger of a slab of level-1
    layers (an even number of layers of 4608 nx_1 ny_1 bytes, at most RAP_SLAB_BYTES, at least 2, at most nz_1) and level
    3's (built from level 2's; 0 when there are only 3 levels).  Raises ValueError where create refuses the box."""
    lv, _ = _rap_levels(ne)
    layer = ELEMENT_MATRIX_BYTES * lv[1][0] * lv[1][1]
    per = min(lv[1][2], max(2, (RAP_SLAB_BYTES // layer) & ~1))
    elems = [v[0] * v[1] * v[2] for v in lv]
    l3 = ELEMENT_MATRIX_BYTES * elems[3] if len(lv) > 3 else 0
    return ELEMENT_MATRIX_BYTES * elems[2] + max(per * layer, l3)


def gathered_elements(levels) -> int:
    """Elements of the global box of the gathered level of `rank_levels`' list, whose element matrices a multi-rank field
    hierarchy gathers onto every rank.  Raises ValueError, as pcgb_mg_create_ranks_field refuses, above MAX_GATHERED_ELEMENTS:
    the matrices take 4608 bytes per element and the gather plan (ranks - 1) * 576 entries per element."""
    g = levels[-1][0].ng
    n = int(g[0]) * int(g[1]) * int(g[2])
    if n > MAX_GATHERED_ELEMENTS:
        raise ValueError(f"HexMultigrid: the gathered level has {n} elements (at most {MAX_GATHERED_ELEMENTS} with E_field across ranks)")
    return n


def check_global_field(E_field, ng, device=None):
    """A Young's modulus per element of the whole mesh ng (shape (ng[2], ng[1], ng[0]), float64, numpy or a tensor on the
    CPU or `device`), every value finite and positive; raises ValueError otherwise.  Checked the same way on every rank,
    since all ranks hold the same field, before any collective step."""
    check_field(E_field, HexBlock(tuple(ng), (0, 0, 0), tuple(ng)), device)
    if isinstance(E_field, torch.Tensor):
        ok = bool(torch.all(torch.isfinite(E_field) & (E_field > 0)))
    else:
        ok = bool(np.all(np.isfinite(E_field) & (E_field > 0)))
    if not ok:
        raise ValueError("E_field: every value must be finite and positive")
    return E_field


def rap_rank_bytes(levels, rank: int) -> int:
    """Device bytes pcgb_mg_info reports on rank `rank` of the multi-rank rap hierarchy of `rank_levels`' list `levels` (la =
    len(levels) - 1 >= 2), in 8-byte entries unless stated: the vectors (the fine level's z, D^-1 and three smoother vectors;
    each ranked smoothed level's b, x, D^-1 and three smoother vectors, level 1 included; the same six per smoothed level of
    the replicated hierarchy of the gathered global box; the coarsest b, x and dense factor), the ownership weights of every
    ranked level 0 .. la, b and x of the gathered level la, and the CSR of ranked levels 2 .. la-1 (the rank's sub-assembled
    box) and of the replicated smoothed levels, as in `rap_bytes`.  Level 1 holds no matrix.  Raises ValueError for la < 2,
    as HexMultigrid refuses it."""
    la = len(levels) - 1
    if la < 2:
        raise ValueError("HexMultigrid: coarse='rap' across ranks needs the rank boxes to halve at least twice "
                         f"(la = {la}: level 1 would be the gathered level, which is not smoothed)")
    mine = [lv[rank] for lv in levels]
    rep = _whole_levels(levels[-1][0].ng)
    nr = [3 * v[0] * (v[1] + 1) * (v[2] + 1) for v in rep]
    vectors = 5 * mine[0].n + 6 * sum(b.n for b in mine[1:la]) + 6 * sum(nr[:-1]) + 2 * nr[-1] + nr[-1] ** 2
    own = sum(b.n for b in mine)
    csr = sum(_csr_bytes(b.ne, b.n, b.x_lo) for b in mine[2:la]) + sum(_csr_bytes(rep[k], nr[k]) for k in range(len(rep) - 1))
    return 8 * (vectors + own + 2 * mine[la].n) + csr


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

    One rank: block is the whole mesh (e0 = 0, ng = ne; under the default coarsening="even" every level halves every ne
    while all are even and the halves stay >= 2, and the coarsest level must have at most 1536 dofs).  Across ranks (op.comm with 2 or more ranks):
    blocks lists every rank's box and block is blocks[op.comm.rank]; construction is collective and refuses (ValueError,
    on every rank alike, before anything is allocated) what `rank_levels` refuses.

    E_field: the per-element Young's modulus `op` was generated with (hexmesh.generate_matrix / generate_ebe /
    generate_box_operator with E_field; float64, a numpy array or a tensor).  The coarse levels are then Galerkin products of
    element matrices instead of rediscretisations with block.E.  One rank: the field of the box, shape (ne[2], ne[1], ne[0])
    (pcgb_mg_create_field, which checks its values on the device).  Across ranks: the field of the WHOLE mesh, shape
    (ng[2], ng[1], ng[0]), the array every rank passes to hexmesh.block_field for its operator (pcgb_mg_create_ranks_field
    with the rank's block_field slice).  Every rank checks the whole field on the host (shape, finite and positive values)
    and the gathered level's element count (`gathered_elements`, at most MAX_GATHERED_ELEMENTS), so a refusal is a ValueError
    on every rank alike, before anything is allocated; a rank's block-shaped slice is refused.  The set-up holds up to two
    levels' element matrices of the rank's boxes, then the gathered level's (setup_info).

    coarsening (one rank only): "even" (the default, above) or "any": a box of any size, each axis halved or kept on its own
    (`any_levels`), Galerkin levels from E_field or, without it, from Ck = block.E * block.h on every element
    (pcgb_mg_create_any).  "any" builds 4608 bytes of element matrices per level-1 element during the set-up and sets up
    slower than the rediscretised default.  Any other string, or "any" with a multi-rank `op`, raises ValueError.

    coarse: "csr" (the default: every smoothed coarse level a device-generated CSR matrix), "index_free" (those levels
    applied by the index-free hex-box operator, Ck = block.E 2^l block.h; `index_free_bytes` gives the one-rank hierarchy's
    device bytes) or "rap" (default coarsening, E_field required: level 1 applied as P^T A_0 P from the fine Ck field
    without a matrix, levels >= 2 the CSR field hierarchy's bit for bit; `rap_bytes` and `rap_setup_peak_bytes` on one
    rank, `rap_rank_bytes` across ranks, where each rank applies level 1 on its own level-1 box from its slice of the field
    and the level's exchange-add completes the product).  "index_free" with E_field or coarsening="any" raises ValueError,
    as does any other string: Galerkin coarse matrices and odd or kept axes are not one Ke on one box.  "rap" raises
    ValueError before any library call without E_field, with coarsening="any", on one rank for a box `rap_bytes` refuses
    (fewer than 3 levels among them), and across ranks without `blocks`, for what the multi-rank field hierarchy refuses,
    and when the rank boxes do not halve at least twice (la < 2: level 1 would be the gathered level).  A rap handle keeps
    the fine Ck field (across ranks the rank's slice) on the device (8 bytes per element) and reads it in every V-cycle."""

    def __init__(self, op, block: HexBlock, degree: int = 2, lo: float = 0.25, minv: torch.Tensor | None = None, blocks=None,
                 E_field=None, coarsening: str = "even", coarse: str = "csr"):
        from .hexop import PeriodicCellOperator
        if isinstance(getattr(op, "A", None), PeriodicCellOperator) or isinstance(block, PeriodicCell):
            raise ValueError("HexMultigrid: periodic cells have no multigrid (their coarse levels and singular coarsest level "
                             "are not built); use Jacobi-PCG")
        self.op, self.block, self.degree, self.lo = op, block, int(degree), float(lo)
        self.n = op.n
        self.device = op.device
        self._h = ctypes.c_void_p()
        self._halos = []
        self.levels = None
        self._ck = None
        comm = getattr(op, "comm", None)
        ranked = comm is not None and comm.nranks > 1
        if coarsening not in ("even", "any"):
            raise ValueError(f"HexMultigrid: coarsening must be 'even' or 'any', not {coarsening!r}")
        self.coarsening = coarsening
        if coarse not in ("csr", "index_free", "rap"):
            raise ValueError(f"HexMultigrid: coarse must be 'csr', 'index_free' or 'rap', not {coarse!r}")
        if coarse == "index_free" and (E_field is not None or coarsening == "any"):
            raise ValueError("HexMultigrid: coarse='index_free' needs the default coarsening and no E_field "
                             "(Galerkin coarse levels are not one element matrix on one box)")
        if coarse == "rap":
            if E_field is None:
                raise ValueError("HexMultigrid: coarse='rap' needs E_field (its level 1 is P^T A P of the fine field)")
            if coarsening != "even":
                raise ValueError("HexMultigrid: coarse='rap' needs the default coarsening")
            if ranked and blocks is None:
                raise ValueError("HexMultigrid: coarse='rap' across ranks needs `blocks`, one box per rank (on one rank it needs none)")
            if not ranked:
                rap_bytes(block.ne)
        self.coarse = coarse
        if coarsening == "any" and ranked:
            raise ValueError("HexMultigrid: coarsening='any' is supported on one rank only")
        if ranked:
            if blocks is None or len(blocks) != comm.nranks:
                raise ValueError("HexMultigrid: a multi-rank operator needs `blocks`, one box per rank")
            if blocks[comm.rank] != block:
                raise ValueError("HexMultigrid: block must be blocks[comm.rank]")
            if block.n != op.n:
                raise ValueError(f"HexMultigrid: the operator has {op.n} rows, the box {block.n}")
            self.levels = rank_levels(blocks)
            if E_field is not None:
                check_global_field(E_field, block.ng, self.device)
                nge = gathered_elements(self.levels)
            if coarse == "rap":
                rap_rank_bytes(self.levels, comm.rank)
        # across ranks the rank's slice of the global field
        ck = None if E_field is None else field_ck(block_field(E_field, block) if ranked else E_field, block, self.device)
        minv = op.jacobi() if minv is None else minv.to(self.device, torch.float64).contiguous()
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        kep = ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        box = ctypes.byref(block.cbox())
        uniform = (float(block.E), float(block.h))
        tail = (_lib.ptr(minv), self.degree, self.lo, ctypes.byref(self._h))
        if coarse == "rap":
            self._ck = ck              # read by every V-cycle: it lives as long as the handle
        # The library synchronises the device before it reads minv, ck or the ownership weights, whatever stream wrote them.
        lib = _lib.load()
        with torch.cuda.device(self.device):
            if not ranked:
                if coarsening == "any":
                    name, args = "pcgb_mg_create_any", (_lib.ptr(ck), *uniform)
                elif ck is not None:
                    name, args = ("pcgb_mg_create_field_rap" if coarse == "rap" else "pcgb_mg_create_field"), (_lib.ptr(ck),)
                else:
                    name, args = ("pcgb_mg_create_index_free" if coarse == "index_free" else "pcgb_mg_create"), uniform
                _lib.check(getattr(lib, name)(op._solver, box, kep, *args, *tail), name)
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
            kg = None
            if ck is not None:
                # a plan over the gathered level's element matrices, used by the set-up only
                kg = make_halo(comm, others, [np.arange(576 * nge, dtype=np.int64)] * len(others), 576 * nge)
                name = "pcgb_mg_create_ranks_field_rap" if coarse == "rap" else "pcgb_mg_create_ranks_field"
                args = (kg, owns, kep, _lib.ptr(ck))
            else:
                name = "pcgb_mg_create_ranks_index_free" if coarse == "index_free" else "pcgb_mg_create_ranks"
                args = (owns, kep, *uniform)
            try:
                _lib.check(getattr(lib, name)(op._solver, box, la, halos, self._gather, *args, *tail), name)
            finally:
                if kg is not None:
                    lib.pcgb_halo_destroy(kg)

    @property
    def handle(self):
        return self._h

    def _vec(self, n):
        return torch.empty(n, dtype=torch.float64, device=self.device)

    def _call(self, name: str, *args):
        """The library's `name`(handle, *args, stream) on the current stream of the handle's device."""
        with torch.cuda.device(self.device):
            _lib.check(getattr(_lib.load(), name)(self._h, *args, _lib.stream_ptr()), name)

    def apply(self, r: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """z = M r (one V-cycle; collective across ranks)."""
        z = out if out is not None else self._vec(self.n)
        self._call("pcgb_mg_apply", _lib.ptr(r), _lib.ptr(z))
        return z

    def info(self) -> dict:
        """levels, n per level, largest-eigenvalue estimates of D^-1 A per level (0 for the coarsest and for the gathered
        level), device bytes, coarse ("csr", "index_free" or "rap"); across ranks also gather_level (la, -1 on one rank),
        n_gathered and global_lambda (the estimates of the global hierarchy: ranked levels below la, then the replicated
        ones)."""
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
        out = {"levels": k, "n": [int(v) for v in n[:k]], "lambda": lams, "bytes": int(nb.value), "coarse": self.coarse}
        if la.value >= 0:
            out.update(gather_level=la.value, n_gathered=int(ng.value), global_lambda=lams[:la.value] + lams[la.value + 1:])
        return out

    def setup_info(self) -> dict:
        """galerkin_ms (device time of the Galerkin kernels) and element_matrix_peak_bytes (element matrices held at once
        during the set-up); both 0 for the default coarsening without E_field."""
        ms, peak = ctypes.c_double(), ctypes.c_int64()
        _lib.check(_lib.load().pcgb_mg_setup_info(self._h, ctypes.byref(ms), ctypes.byref(peak)), "pcgb_mg_setup_info")
        return {"galerkin_ms": float(ms.value), "element_matrix_peak_bytes": int(peak.value)}

    def level_shapes(self) -> list:
        """Element counts (nx, ny, nz) of every level (pcgb_mg_level_box); across ranks the rank's boxes up to the gathered
        level, then the global ones."""
        lib = _lib.load()
        ne = (ctypes.c_int32 * 3)()
        out = []
        for l in range(self.info()["levels"]):
            _lib.check(lib.pcgb_mg_level_box(self._h, l, ne), "pcgb_mg_level_box")
            out.append(tuple(int(v) for v in ne))
        return out

    # ---- the V-cycle's parts (tests; collective across ranks)
    def level_matrix(self, level: int):
        """The CSR of smoothed coarse level `level` (1 .. levels - 2) as (rowptr int64, col int32, val float64) device tensors."""
        nnz = ctypes.c_int64()
        self._call("pcgb_mg_level_csr", level, None, None, None, ctypes.byref(nnz))
        n = self.info()["n"][level]
        rowptr = torch.empty(n + 1, dtype=torch.int64, device=self.device)
        col = torch.empty(nnz.value, dtype=torch.int32, device=self.device)
        val = torch.empty(nnz.value, dtype=torch.float64, device=self.device)
        self._call("pcgb_mg_level_csr", level, _lib.ptr(rowptr), _lib.ptr(col), _lib.ptr(val), ctypes.byref(nnz))
        return rowptr, col, val

    def level_dinv(self, level: int) -> torch.Tensor:
        """D^-1 of smoothed level `level` (0 .. levels - 2, not the gathered level) as a device tensor, any hierarchy kind."""
        d = self._vec(self.info()["n"][level])
        self._call("pcgb_mg_level_dinv", level, _lib.ptr(d))
        return d

    def level_apply(self, level: int, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """y = A_l x on smoothed coarse level `level` (1 .. levels - 2, not the gathered level), either coarse kind: the
        local product, without the level's exchange-add across ranks (x and out must not overlap)."""
        y = out if out is not None else self._vec(self.info()["n"][level])
        self._call("pcgb_mg_level_apply", level, _lib.ptr(x), _lib.ptr(y))
        return y

    def restrict(self, level: int, rf: torch.Tensor) -> torch.Tensor:
        rc = self._vec(self.info()["n"][level + 1])
        self._call("pcgb_mg_restrict", level, _lib.ptr(rf), _lib.ptr(rc))
        return rc

    def prolong_add(self, level: int, ec: torch.Tensor, xf: torch.Tensor) -> torch.Tensor:
        self._call("pcgb_mg_prolong_add", level, _lib.ptr(ec), _lib.ptr(xf))
        return xf

    def smooth(self, level: int, b: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
        """x += S (b - A x) on `level`, in place."""
        self._call("pcgb_mg_smooth", level, _lib.ptr(b), _lib.ptr(x))
        return x

    def coarse_solve(self, r: torch.Tensor) -> torch.Tensor:
        z = self._vec(r.numel())
        self._call("pcgb_mg_coarse_solve", _lib.ptr(r), _lib.ptr(z))
        return z

    def gather(self, v: torch.Tensor) -> torch.Tensor:
        """The gathered level's ranked vector -> its global box, the same on every rank."""
        out = self._vec(self.info()["n_gathered"])
        self._call("pcgb_mg_gather", _lib.ptr(v), _lib.ptr(out))
        return out

    def scatter(self, g: torch.Tensor) -> torch.Tensor:
        """This rank's entries of a global vector of the gathered level."""
        info = self.info()
        out = self._vec(info["n"][info["gather_level"]])
        self._call("pcgb_mg_scatter", _lib.ptr(g), _lib.ptr(out))
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
