"""Host restatement of the index-free hex-box operator (csrc/hexop.cuh, HexBoxOperator).

`node_slots` enumerates, for every free dof, the (local index la, element) pairs the kernel visits, from the node's
coordinates alone; `ref_rows` is the long-double product of chosen rows with the rounding scale of each, which the kernel
must meet within (k + 2) 2^-53 sum |terms| (k = terms summed)."""
import numpy as np

from pcg_mpi_solver_b200.hexmesh import HexBlock, hex_element_stiffness

EPS = 2.0 ** -53

# boxes (ng, e0, ne): with and without the clamped face, e0 != 0 on every axis, ne = 1 / 2 / odd / even per axis, 1x1x1
BOXES = [
    ((1, 1, 1), (0, 0, 0), (1, 1, 1)),
    ((3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ((2, 2, 2), (0, 0, 0), (2, 2, 2)),
    ((5, 4, 3), (0, 0, 0), (5, 4, 3)),
    ((9, 8, 7), (2, 3, 1), (5, 2, 3)),
    ((9, 8, 7), (0, 1, 2), (4, 5, 1)),
    ((6, 7, 8), (3, 2, 4), (2, 3, 4)),
    ((7, 6, 5), (0, 4, 0), (7, 1, 2)),
]


def free_nodes(block: HexBlock):
    """(lx, ly, lz) of every free node in the free numbering (x fastest; lx counts the clamped line)."""
    nx, ny, nz = block.ne
    lz, ly, lx = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(block.x_lo, nx + 1), indexing="ij")
    return lx.ravel(), ly.ravel(), lz.ravel()


def node_slots(block: HexBlock):
    """{free dof: [(a, e), ...]} with a = 3 la + d, la ascending, e the element around the node at local index la."""
    nx, ny, nz = block.ne
    lx, ly, lz = free_nodes(block)
    out = {}
    for node in range(lx.size):
        for d in range(3):
            lst = []
            for la in range(8):
                ox, oy, oz = lx[node] - (la & 1), ly[node] - ((la >> 1) & 1), lz[node] - (la >> 2)
                if 0 <= ox < nx and 0 <= oy < ny and 0 <= oz < nz:
                    lst.append((3 * la + d, int((oz * ny + oy) * nx + ox)))
            out[3 * node + d] = lst
    return out


def group_slots(grp, eff, ndof):
    """{free dof: [(a, e), ...]} from the ordered operator's slot positions a * ne + e of hex_type_group, ascending."""
    em = np.full(ndof, -1, dtype=np.int64)
    em[eff] = np.arange(len(eff))
    idx = em[grp.loc_dof]
    nd, ne = idx.shape
    out = {int(i): [] for i in range(len(eff))}
    for pos in range(nd * ne):           # ascending slot position
        a, e = divmod(pos, ne)
        if idx[a, e] >= 0:
            out[int(idx[a, e])].append((a, e))
    return out


def ref_rows(block: HexBlock, rows, xfetch, ckfetch):
    """(y, abs_sum, count) in long double for free dofs `rows`.  xfetch(free dofs) -> float64 values of x, ckfetch(elements)
    -> Ck.  Only the rows' neighbourhoods are fetched, so a sample of a huge box stays cheap."""
    nx, ny, nz = block.ne
    nxf = nx + 1 - block.x_lo
    ke = hex_element_stiffness(1.0, block.nu).astype(np.longdouble)
    rows = np.asarray(rows, dtype=np.int64)
    node, d = rows // 3, rows % 3
    fx, ly, lz = node % nxf, (node // nxf) % (ny + 1), node // (nxf * (ny + 1))
    lx = fx + block.x_lo
    y = np.zeros(rows.size, dtype=np.longdouble)
    s = np.zeros(rows.size, dtype=np.longdouble)
    k = np.zeros(rows.size, dtype=np.int64)
    for la in range(8):
        ox, oy, oz = lx - (la & 1), ly - ((la >> 1) & 1), lz - (la >> 2)
        ok = (ox >= 0) & (ox < nx) & (oy >= 0) & (oy < ny) & (oz >= 0) & (oz < nz)
        if not ok.any():
            continue
        sel = np.nonzero(ok)[0]
        e = (oz[sel] * ny + oy[sel]) * nx + ox[sel]
        c = np.asarray(ckfetch(e), dtype=np.longdouble)
        for lb in range(8):
            bx, by, bz = ox[sel] + (lb & 1), oy[sel] + ((lb >> 1) & 1), oz[sel] + (lb >> 2)
            free = bx >= block.x_lo
            bnode = (bz * (ny + 1) + by) * nxf + (bx - block.x_lo)
            for dd in range(3):
                xv = np.zeros(sel.size, dtype=np.longdouble)
                if free.any():
                    xv[free] = np.asarray(xfetch(3 * bnode[free] + dd), dtype=np.longdouble)
                t = ke[3 * la + d[sel], 3 * lb + dd] * (c * xv)
                y[sel] += t
                s[sel] += np.abs(t)
        k[sel] += 25
    return y, s, k


def assert_rows(yrows, block, rows, xfetch, ckfetch):
    ref, s, k = ref_rows(block, rows, xfetch, ckfetch)
    yrows = np.asarray(yrows)
    assert not np.isnan(yrows).any(), f"{int(np.isnan(yrows).sum())} rows never written"
    err = np.abs(yrows.astype(np.longdouble) - ref)
    bad = np.nonzero(err > (k + 2) * EPS * s)[0]
    assert bad.size == 0, f"{bad.size} rows off, first {np.asarray(rows)[bad[:5]]}: err {err[bad[:5]]}"


def hard_x(n, rng):
    """x with signed zeros and entries over many decades."""
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-150, 150, n)
    x[rng.random(n) < 0.1] = 0.0
    x[rng.random(n) < 0.1] = -0.0
    return x
