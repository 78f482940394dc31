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


def generate_matrix(block: HexBlock, device="cuda") -> CsrMatrix:
    """Sub-assembled K_i[Eff,Eff] of the box, generated on the device."""
    lib = _lib.load()
    box = block.cbox()
    n = int(lib.pcgb_hex_nrows(ctypes.byref(box)))
    assert n == block.n
    with torch.cuda.device(device):
        counts = torch.empty(n + 1, dtype=torch.int64, device=device)
        _lib.check(lib.pcgb_hex_count(ctypes.byref(box), _lib.ptr(counts), _lib.stream_ptr()), "pcgb_hex_count")
        rowptr = torch.cumsum(counts, 0)  # plumbing: inclusive scan of the per-row counts
        del counts
        nnz = int(rowptr[-1].item())
        col = torch.empty(nnz, dtype=torch.int32, device=device)
        val = torch.empty(nnz, dtype=torch.float64, device=device)
        ke = np.ascontiguousarray(hex_element_stiffness(1.0, block.nu))
        _lib.check(lib.pcgb_hex_fill(ctypes.byref(box), ke.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                     float(block.E * block.h), _lib.ptr(rowptr), _lib.ptr(col), _lib.ptr(val),
                                     _lib.stream_ptr()), "pcgb_hex_fill")
        torch.cuda.current_stream().synchronize()
        if nnz < 2**31:
            rowptr = rowptr.to(torch.int32)
    return CsrMatrix(rowptr, col, val, (n, n))


def hex_type_group(block: HexBlock):
    """The box as the reference would hold it: ONE pattern type group (the Q1 hexahedron, no sign flips,
    Ck = E*h; partition_mesh.py:443-491) in the local all-dof numbering 3*node + dir (x fastest), plus LocDofEff.
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
    grp = TypeGroup(0, dofs, np.zeros(dofs.shape, dtype=bool), np.full(ex.size, block.E * block.h), hex_element_stiffness(1.0, block.nu), None)
    return grp, eff, 3 * (nx + 1) * (ny + 1) * (nz + 1)


def generate_ebe(block: HexBlock, device="cuda", ordered: bool = False):
    """The same box as a matrix-free EBE operator (ebe.EbeMatrix); opt-in companion of generate_matrix (SURVEY 8(f1)).
    ordered=True builds ebe.EbeMatrixOrdered, the bit-reproducible variant with a fixed summation order."""
    from .ebe import EbeMatrix, EbeMatrixOrdered
    grp, eff, ndof = hex_type_group(block)
    return (EbeMatrixOrdered if ordered else EbeMatrix)([grp], eff, ndof, device=device)


def hex_mdf_model(ng, E: float = 1.0, nu: float = 0.3, h: float | None = None, traction: float = 1.0):
    """The structured hex problem as an in-memory `MdfModel` (the reference's model-definition schema, SURVEY
    Appendix A) so that the general pipeline - `partition_mesh(model, nparts)` with METIS, the subdomain builder,
    device assembly / EBE - can run on it (config C3: the 128^3 mesh partitioned 8-way by METIS).
    Global numbering: node = (gz*(ny+1)+gy)*(nx+1)+gx, dof = 3*node+dir; one pattern type (the Q1 hexahedron)."""
    from .model import MdfModel
    nx, ny, nz = ng
    h = 1.0 / nx if h is None else h
    ne = nx * ny * nz
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
                    etype=np.zeros(ne, dtype=np.int32), ck=np.full(ne, E * h), F=F, Ud=np.zeros(ndof),
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
