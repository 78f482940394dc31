"""Structured hex elastostatic benchmark problem (BASELINE.json configs C2 / C3 / C5).

A unit-size-h trilinear hex mesh of ng[0] x ng[1] x ng[2] elements, clamped on the global x = 0
face, uniform traction in -z on the x = max face (deterministic, no RNG; SURVEY 8(d) C2).  Each rank
owns one box of elements; its sub-assembled stiffness matrix is generated ON DEVICE by
`pcgb_hex_count` / `pcgb_hex_fill` (csrc/hexgen.cuh) because a 256^3 box is 49 GB of CSR.

The data produced for a rank mirrors what the reference's builder exports for a mesh part
(partition_mesh.py:1310-1317), restricted to the free dofs:
    A            K_i[Eff,Eff]                  (calcMatVecProd operator, pcg_solver.py:242-300)
    b            Fext[LocDofEff]               (updateBC, pcg_solver.py:226-238, Ud = 0)
    w            DofWeightVector[LocDofEff]    (partition_mesh.py:867-887)
    nbr / ovrlp  NbrMPIdVector / OvrlpLocalDofVecList (partition_mesh.py:805-830), ascending global node id

Element pattern: the 8-node trilinear (Q1) hexahedron, E = 1, nu = 0.3, unit edge, integrated with
2x2x2 Gauss points; Ck = E*h scales it like ElemList_Ck scales the reference's pattern matrices.
(The reference's own cube pattern Ke[0] of data/concrete.zip is the SBFEM cube; same 27-node x 3 x 3
sparsity.  The Q1 matrix keeps this repository free of reference data.)
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from .csr import CsrMatrix


def hex_element_stiffness(E: float = 1.0, nu: float = 0.3) -> np.ndarray:
    """24x24 stiffness of the unit-edge Q1 hexahedron; local node l sits at (l&1, l>>1&1, l>>2&1);
    dof = 3*l + direction."""
    lam = E * nu / ((1 + nu) * (1 - 2 * nu))
    mu = E / (2 * (1 + nu))
    D = np.zeros((6, 6))
    D[:3, :3] = lam
    D[np.arange(3), np.arange(3)] += 2 * mu
    D[np.arange(3, 6), np.arange(3, 6)] = mu
    corners = np.array([[(l >> 0) & 1, (l >> 1) & 1, (l >> 2) & 1] for l in range(8)], dtype=float) * 2 - 1
    g = 1.0 / np.sqrt(3.0)
    Ke = np.zeros((24, 24))
    for gz in (-g, g):
        for gy in (-g, g):
            for gx in (-g, g):
                xi = np.array([gx, gy, gz])
                # dN/dxi (8x3) in the reference cube [-1,1]^3, then dN/dx with J = 1/2 I (unit edge)
                dN = np.empty((8, 3))
                for a in range(3):
                    f = np.ones(8)
                    for c in range(3):
                        f *= corners[:, c] / 8.0 if c == a else (1 + corners[:, c] * xi[c])
                    dN[:, a] = f
                dN *= 2.0
                B = np.zeros((6, 24))
                B[0, 0::3] = dN[:, 0]
                B[1, 1::3] = dN[:, 1]
                B[2, 2::3] = dN[:, 2]
                B[3, 0::3] = dN[:, 1]; B[3, 1::3] = dN[:, 0]
                B[4, 1::3] = dN[:, 2]; B[4, 2::3] = dN[:, 1]
                B[5, 0::3] = dN[:, 2]; B[5, 2::3] = dN[:, 0]
                Ke += B.T @ D @ B * (1.0 / 8.0)  # det J = (1/2)^3, unit weights
    return 0.5 * (Ke + Ke.T)


@dataclass
class HexBlock:
    """One rank's box of a global hex mesh, in the free-dof numbering used by the kernels."""
    ng: tuple          # global elements per axis
    e0: tuple          # first element of the box per axis
    ne: tuple          # elements in the box per axis
    h: float = 1.0
    E: float = 1.0
    nu: float = 0.3

    @property
    def x_lo(self) -> int:
        return 1 if self.e0[0] == 0 else 0

    @property
    def nfree_nodes(self) -> int:
        return (self.ne[0] + 1 - self.x_lo) * (self.ne[1] + 1) * (self.ne[2] + 1)

    @property
    def n(self) -> int:
        return 3 * self.nfree_nodes

    def cbox(self) -> _lib.HexBox:
        b = _lib.HexBox()
        for a in range(3):
            b.ng[a], b.e0[a], b.ne[a] = int(self.ng[a]), int(self.e0[a]), int(self.ne[a])
        return b

    # ---- node helpers (host, vectorised) ------------------------------------------------------
    def free_index_of_global_nodes(self, gx, gy, gz):
        """Local free-node index of global node coordinates lying inside the box (gx >= 1)."""
        nxf = self.ne[0] + 1 - self.x_lo
        lx = gx - self.e0[0] - self.x_lo
        ly = gy - self.e0[1]
        lz = gz - self.e0[2]
        return (lz * (self.ne[1] + 1) + ly) * nxf + lx

    def node_ranges(self):
        return [(self.e0[a], self.e0[a] + self.ne[a]) for a in range(3)]


@dataclass
class PeriodicCell:
    """A periodic cell of ne[0] x ne[1] x ne[2] hex elements of edge h (homogenisation; DESIGN §2.13): node (lx, ly, lz) is
    identified with (lx mod ne[0], ly mod ne[1], lz mod ne[2]), so the cell has as many nodes as elements and no clamped
    dof; dof = 3 node + dir, node = (lz ne[1] + ly) ne[0] + lx.  Every ne must be >= 2 (the library refuses less)."""
    ne: tuple
    h: float = 1.0
    E: float = 1.0
    nu: float = 0.3

    @property
    def n_elements(self) -> int:
        return int(self.ne[0]) * int(self.ne[1]) * int(self.ne[2])

    @property
    def n(self) -> int:
        return 3 * self.n_elements

    def cbox(self) -> _lib.HexBox:
        """The whole-mesh box (e0 = 0, ng = ne) the periodic entry points take."""
        b = _lib.HexBox()
        for a in range(3):
            b.ng[a], b.e0[a], b.ne[a] = int(self.ne[a]), 0, int(self.ne[a])
        return b


def _same_device(a, b) -> bool:
    """torch devices a and b are one device ('cuda' stands for the current CUDA device)."""
    a, b = torch.device(a), torch.device(b)
    if a.type == "cuda" and a.index is None:
        a = torch.device("cuda", torch.cuda.current_device())
    if b.type == "cuda" and b.index is None:
        b = torch.device("cuda", torch.cuda.current_device())
    return a == b


def check_field(E_field, block: HexBlock, device=None) -> np.ndarray | torch.Tensor:
    """A per-element Young's modulus of `block`: float64, shape (ne[2], ne[1], ne[0]) (x fastest in memory), a numpy array,
    a CPU tensor or a tensor on `device` (device None: a tensor on any device).  Raises ValueError otherwise.  Its values
    (finite, positive) are checked on the device by the kernels that read it."""
    shape = tuple(int(v) for v in reversed(block.ne))
    if isinstance(E_field, torch.Tensor):
        if E_field.dtype != torch.float64:
            raise ValueError(f"E_field: float64 required, got {E_field.dtype}")
        if device is not None and E_field.device.type != "cpu" and not _same_device(E_field.device, device):
            raise ValueError(f"E_field: on {E_field.device}, expected the CPU or {device}")
    elif isinstance(E_field, np.ndarray):
        if E_field.dtype != np.float64:
            raise ValueError(f"E_field: float64 required, got {E_field.dtype}")
    else:
        raise ValueError("E_field: a numpy array or a torch tensor required")
    if tuple(E_field.shape) != shape:
        raise ValueError(f"E_field: shape {tuple(E_field.shape)}, the box has {shape} elements (ne[2], ne[1], ne[0])")
    return E_field


def field_ck(E_field, block: HexBlock, device) -> torch.Tensor:
    """Ck = E_e * h per element of the box, as a contiguous float64 device vector in element order."""
    check_field(E_field, block, device)
    t = torch.from_numpy(E_field) if isinstance(E_field, np.ndarray) else E_field
    return (t.reshape(-1).to(device, torch.float64) * float(block.h)).contiguous()


def generate_matrix(block: HexBlock, device="cuda", E_field=None) -> CsrMatrix:
    """Sub-assembled K_i[Eff,Eff] of the box, generated on the device.  E_field: one Young's modulus per element of the box
    (shape (ne[2], ne[1], ne[0]), float64; see block_field), replacing block.E: a voxel model (pcgb_hex_fill_field)."""
    lib = _lib.load()
    box = block.cbox()
    n = int(lib.pcgb_hex_nrows(ctypes.byref(box)))
    assert n == block.n
    ck = None if E_field is None else field_ck(E_field, block, device)
    with torch.cuda.device(device):
        if ck is not None:   # refuse a bad field before the CSR arrays are allocated
            _lib.check(lib.pcgb_hex_field_check(ctypes.byref(box), _lib.ptr(ck), _lib.stream_ptr()), "pcgb_hex_field_check")
        counts = torch.empty(n + 1, dtype=torch.int64, device=device)
        _lib.check(lib.pcgb_hex_count(ctypes.byref(box), _lib.ptr(counts), _lib.stream_ptr()), "pcgb_hex_count")
        rowptr = torch.cumsum(counts, 0)  # plumbing: inclusive scan of the per-row counts
        del counts
        nnz = int(rowptr[-1].item())
        col = torch.empty(nnz, dtype=torch.int32, device=device)
        val = torch.empty(nnz, dtype=torch.float64, device=device)
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        if ck is None:
            _lib.check(lib.pcgb_hex_fill(ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                         float(block.E * block.h), _lib.ptr(rowptr), _lib.ptr(col), _lib.ptr(val),
                                         _lib.stream_ptr()), "pcgb_hex_fill")
        else:
            _lib.check(lib.pcgb_hex_fill_field(ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                               _lib.ptr(ck), _lib.ptr(rowptr), _lib.ptr(col), _lib.ptr(val),
                                               _lib.stream_ptr()), "pcgb_hex_fill_field")
        torch.cuda.current_stream().synchronize()
        if nnz < 2**31:
            rowptr = rowptr.to(torch.int32)
    return CsrMatrix(rowptr, col, val, (n, n))


def hex_type_group(block: HexBlock, E_field=None, device=None):
    """The box as the reference would hold it: ONE pattern type group (the Q1 hexahedron, no sign flips,
    Ck = E*h; partition_mesh.py:443-491) in the local all-dof numbering 3*node + dir (x fastest), plus LocDofEff.
    E_field (shape (ne[2], ne[1], ne[0])): Ck = E_field * h per element instead (a tensor on the CPU or on `device`; any
    device when `device` is None).
    Returns (TypeGroup, loc_dof_eff, ndof)."""
    from .partition import TypeGroup
    nx, ny, nz = block.ne
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    dofs = np.empty((24, ex.size), dtype=np.int64)
    for l in range(8):
        node = ((ez + ((l >> 2) & 1)) * (ny + 1) + (ey + ((l >> 1) & 1))) * (nx + 1) + (ex + (l & 1))
        for d in range(3):
            dofs[3 * l + d] = 3 * node + d
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    free_nodes = np.nonzero(lx.ravel() >= block.x_lo)[0]     # ascending -> the free numbering of generate_matrix
    eff = (3 * free_nodes[:, None] + np.arange(3)[None, :]).ravel()
    if E_field is None:
        ck = np.full(ex.size, block.E * block.h)
    else:
        check_field(E_field, block, device)
        f = E_field.detach().cpu().numpy() if isinstance(E_field, torch.Tensor) else E_field
        ck = np.ascontiguousarray(f, dtype=np.float64).reshape(-1) * block.h
    grp = TypeGroup(0, dofs, np.zeros(dofs.shape, dtype=bool), ck, hex_element_stiffness(1.0, block.nu), None)
    return grp, eff, 3 * (nx + 1) * (ny + 1) * (nz + 1)


def generate_ebe(block: HexBlock, device="cuda", ordered: bool = False, E_field=None):
    """The same box as a matrix-free EBE operator (ebe.EbeMatrix); opt-in companion of generate_matrix (SURVEY 8(f1)).
    ordered=True builds ebe.EbeMatrixOrdered, the bit-reproducible variant with a fixed summation order.  E_field: as in
    generate_matrix."""
    from .ebe import EbeMatrix, EbeMatrixOrdered
    grp, eff, ndof = hex_type_group(block, E_field, device)
    return (EbeMatrixOrdered if ordered else EbeMatrix)([grp], eff, ndof, device=device)


def generate_box_operator(block: HexBlock, device="cuda", E_field=None):
    """The same box as the index-free matrix-free operator (hexop.HexBoxOperator): the products and the diagonal of
    generate_ebe(block, ordered=True, E_field=E_field) bit for bit, with no index arrays on the device.  E_field: as in
    generate_matrix."""
    from .hexop import HexBoxOperator
    return HexBoxOperator(block, device=device, E_field=E_field)


def generate_periodic_operator(cell: PeriodicCell, device="cuda", E_field=None):
    """The index-free operator of a periodic cell (hexop.PeriodicCellOperator): the HexBoxOperator interface, accepted by
    SubdomainOperator (Jacobi-PCG), refused by multigrid.HexMultigrid.  E_field: as in generate_matrix, shape
    (ne[2], ne[1], ne[0])."""
    from .hexop import PeriodicCellOperator
    return PeriodicCellOperator(cell, device=device, E_field=E_field)


def hex_mdf_model(ng, E: float = 1.0, nu: float = 0.3, h: float | None = None, traction: float = 1.0, E_field=None):
    """The structured hex problem as an in-memory `MdfModel` (the reference's model-definition schema, SURVEY
    Appendix A) so that the general pipeline - `partition_mesh(model, nparts)` with METIS, the subdomain builder,
    device assembly / EBE - can run on it (config C3: the 128^3 mesh partitioned 8-way by METIS).
    Global numbering: node = (gz*(ny+1)+gy)*(nx+1)+gx, dof = 3*node+dir; one pattern type (the Q1 hexahedron).
    E_field (shape (ng[2], ng[1], ng[0])): one Young's modulus per element, Ck = E_field * h in element order, as the
    reference's concrete model carries one ElemList_Ck per element."""
    from .model import MdfModel
    nx, ny, nz = ng
    h = 1.0 / nx if h is None else h
    ne = nx * ny * nz
    if E_field is None:
        ck = np.full(ne, E * h)
    else:
        check_field(E_field, HexBlock(tuple(ng), (0, 0, 0), tuple(ng)))
        f = E_field.detach().cpu().numpy() if isinstance(E_field, torch.Tensor) else E_field
        ck = np.ascontiguousarray(f, dtype=np.float64).reshape(-1) * h
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    nodes = np.empty((ne, 8), dtype=np.int64)
    for l in range(8):
        nodes[:, l] = ((ez + ((l >> 2) & 1)) * (ny + 1) + (ey + ((l >> 1) & 1))) * (nx + 1) + (ex + (l & 1))
    dofs = (3 * nodes[:, :, None] + np.arange(3)[None, None, :]).reshape(ne, 24)

    def offsets(per):
        s = np.arange(ne, dtype=np.int64) * per
        return np.stack([s, s + per - 1], axis=1)             # INCLUSIVE ends, like the reference's *Offset arrays

    gz, gy, gx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    gx, gy, gz = gx.ravel(), gy.ravel(), gz.ravel()
    ndof = 3 * gx.size
    F = np.zeros(ndof)
    face = gx == nx
    cy = np.where((gy == 0) | (gy == ny), 0.5, 1.0)
    cz = np.where((gz == 0) | (gz == nz), 0.5, 1.0)
    F[3 * np.nonzero(face)[0] + 2] = (-traction * h * h * cy * cz)[face]
    fixed = np.sort((3 * np.nonzero(gx == 0)[0][:, None] + np.arange(3)[None, :]).ravel())
    eff = np.setdiff1d(np.arange(ndof), fixed)
    return MdfModel(name=f"hex{nx}x{ny}x{nz}", n_elem=ne, n_dof=ndof, n_dof_eff=eff.size,
                    node_flat=nodes.ravel().astype(np.int32), node_offset=offsets(8),
                    dof_flat=dofs.ravel().astype(np.int32), dof_offset=offsets(24),
                    sign_flat=np.zeros(ne * 24, dtype=bool), sign_offset=offsets(24),
                    etype=np.zeros(ne, dtype=np.int32), ck=ck, F=F, Ud=np.zeros(ndof),
                    dof_eff=eff.astype(np.int64), fixed_dof=fixed.astype(np.int64), ke=[hex_element_stiffness(1.0, nu)], dt=0.0)


def load_vector(block: HexBlock, traction: float = 1.0, device="cuda") -> torch.Tensor:
    """b = Fext[LocDofEff]: consistent nodal loads of a uniform -z traction on the global x = max face
    (assembled values, identical on every copy of a shared dof, like RefLoadVector = F[DofVector])."""
    b = torch.zeros(block.n, dtype=torch.float64, device=device)
    (x0, x1), (y0, y1), (z0, z1) = block.node_ranges()
    if x1 != block.ng[0]:
        return b
    gy = torch.arange(y0, y1 + 1, device=device)
    gz = torch.arange(z0, z1 + 1, device=device)
    cy = torch.where((gy == 0) | (gy == block.ng[1]), 0.5, 1.0).to(torch.float64)
    cz = torch.where((gz == 0) | (gz == block.ng[2]), 0.5, 1.0).to(torch.float64)
    GZ, GY = torch.meshgrid(gz, gy, indexing="ij")
    node = block.free_index_of_global_nodes(torch.full_like(GY, x1), GY, GZ)
    b[3 * node.reshape(-1) + 2] = (-traction * block.h * block.h * (cz[:, None] * cy[None, :])).reshape(-1)
    return b


def block_field(global_field, block: HexBlock):
    """The box's slice of a field of the whole mesh (shape (ng[2], ng[1], ng[0])): what generate_matrix / generate_ebe take
    as E_field for that box, so every rank builds its own operator without communication."""
    ng = tuple(int(v) for v in reversed(block.ng))
    if tuple(global_field.shape) != ng:
        raise ValueError(f"block_field: the field has shape {tuple(global_field.shape)}, the mesh {ng}")
    (x0, x1), (y0, y1), (z0, z1) = block.node_ranges()
    out = global_field[z0:z1, y0:y1, x0:x1]
    return out.contiguous() if isinstance(out, torch.Tensor) else np.ascontiguousarray(out)


def inclusion_field(ng, fraction: float = 0.4, radii=(2.0, 6.0), E_matrix: float = 1.0, E_inclusion: float = 10.0,
                    seed: int = 0) -> np.ndarray:
    """A two-phase voxel field of spherical inclusions in a matrix (a synthetic stand-in for aggregate in mortar), shape
    (ng[2], ng[1], ng[0]), float64, values E_matrix and E_inclusion only.  Spheres with centres uniform in the box and
    radii uniform in `radii` (element edges) are drawn from numpy's default_rng(seed) one by one; an element (centre at
    i + 1/2) inside one becomes inclusion; drawing stops once the inclusion fraction reaches `fraction`, so it overshoots
    by at most one sphere.  Deterministic: equal arguments give identical bytes."""
    nx, ny, nz = (int(v) for v in ng)
    if not 0.0 <= fraction < 1.0 or not (0 < radii[0] <= radii[1]):
        raise ValueError("inclusion_field: 0 <= fraction < 1 and 0 < radii[0] <= radii[1] required")
    rng = np.random.default_rng(seed)
    inc = np.zeros((nz, ny, nx), dtype=bool)
    target = fraction * inc.size
    count = 0
    while count < target:
        c = rng.uniform(0.0, 1.0, 3) * (nx, ny, nz)
        r = rng.uniform(radii[0], radii[1])
        lo = [max(int(np.floor(c[a] - r)), 0) for a in range(3)]
        hi = [min(int(np.ceil(c[a] + r)) + 1, (nx, ny, nz)[a]) for a in range(3)]
        if any(lo[a] >= hi[a] for a in range(3)):
            continue
        z, y, x = np.meshgrid(np.arange(lo[2], hi[2]) + 0.5, np.arange(lo[1], hi[1]) + 0.5, np.arange(lo[0], hi[0]) + 0.5, indexing="ij")
        inside = (x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2 <= r * r
        sub = inc[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]]
        count += int(np.count_nonzero(inside & ~sub))
        sub |= inside
    return np.where(inc, float(E_inclusion), float(E_matrix))


def block_grid(nranks: int):
    """Process grid used for the weak-scaling stacks of config C5: 1x1x1, 2x1x1, 2x2x1, 2x2x2, ..."""
    p = [1, 1, 1]
    a = 0
    r = nranks
    while r > 1:
        if r % 2:
            raise ValueError("block_grid: rank count must be a power of two")
        p[a % 3] *= 2
        r //= 2
        a += 1
    return tuple(p)


def partition_blocks(ng, pgrid):
    """Split a global mesh into a pgrid[0] x pgrid[1] x pgrid[2] grid of boxes (rank = x fastest)."""
    blocks = []
    cuts = [np.linspace(0, ng[a], pgrid[a] + 1).astype(int) for a in range(3)]
    for pz in range(pgrid[2]):
        for py in range(pgrid[1]):
            for px in range(pgrid[0]):
                e0 = (cuts[0][px], cuts[1][py], cuts[2][pz])
                ne = (cuts[0][px + 1] - e0[0], cuts[1][py + 1] - e0[1], cuts[2][pz + 1] - e0[2])
                blocks.append(HexBlock(tuple(ng), tuple(int(v) for v in e0), tuple(int(v) for v in ne)))
    return blocks


def interface_lists(blocks, rank):
    """Neighbour ranks, shared free-dof index lists (ascending global node id, 3 dofs per node; the
    ordering rule of partition_mesh.py:822-827) and 0/1 ownership weights (partition_mesh.py:867-887)
    of box `rank`."""
    me = blocks[rank]
    ng = me.ng
    nbr, lists = [], []
    w = np.ones(me.n)
    mine = me.node_ranges()
    for other_id, other in enumerate(blocks):
        if other_id == rank:
            continue
        theirs = other.node_ranges()
        lo = [max(mine[a][0], theirs[a][0]) for a in range(3)]
        hi = [min(mine[a][1], theirs[a][1]) for a in range(3)]
        lo[0] = max(lo[0], 1)  # clamped nodes (global x index 0) carry no free dofs
        if any(lo[a] > hi[a] for a in range(3)):
            continue
        gz, gy, gx = np.meshgrid(np.arange(lo[2], hi[2] + 1), np.arange(lo[1], hi[1] + 1), np.arange(lo[0], hi[0] + 1), indexing="ij")
        node = me.free_index_of_global_nodes(gx.ravel(), gy.ravel(), gz.ravel())  # ascending global node id
        dofs = (3 * node[:, None] + np.arange(3)[None, :]).ravel()
        nbr.append(other_id)
        lists.append(dofs.astype(np.int64))
        if rank > other_id:
            w[dofs] = 0.0
    del ng
    return nbr, lists, w


def interface_node_lists(blocks, rank):
    """Neighbour ranks and, per neighbour, the box nodes `rank` shares with it (local numbering of all the box's nodes,
    node = (lz * (ne[1] + 1) + ly) * (ne[0] + 1) + lx, clamped line included) in ascending global node id: the rule of
    interface_lists over every node, as the reference's OvrlpLocalNodeIdVecList covers them (getNodalPS,
    pcg_solver.py:784-809).  The list of rank a for b and that of b for a name the same global nodes in the same order."""
    me = blocks[rank]
    mine = me.node_ranges()
    nbr, lists = [], []
    for other_id, other in enumerate(blocks):
        if other_id == rank:
            continue
        theirs = other.node_ranges()
        lo = [max(mine[a][0], theirs[a][0]) for a in range(3)]
        hi = [min(mine[a][1], theirs[a][1]) for a in range(3)]
        if any(lo[a] > hi[a] for a in range(3)):
            continue
        gz, gy, gx = np.meshgrid(np.arange(lo[2], hi[2] + 1), np.arange(lo[1], hi[1] + 1), np.arange(lo[0], hi[0] + 1), indexing="ij")
        node = ((gz.ravel() - me.e0[2]) * (me.ne[1] + 1) + (gy.ravel() - me.e0[1])) * (me.ne[0] + 1) + (gx.ravel() - me.e0[0])
        nbr.append(other_id)
        lists.append(node.astype(np.int64))
    return nbr, lists
