"""Host restatement of the periodic-cell homogenisation (DESIGN §2.13): periodic assembly of K from hex_element_stiffness,
the macroscopic-strain load, a solve with node 0 pinned (scipy), centroid strain, stress and their volume average; plus the
long-double row restatement of the device operator and load (the style of hexop_cases) and the exact restatement of the
device average's reduction order."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from pcg_mpi_solver_b200.hexmesh import hex_element_stiffness

EPS = 2.0 ** -53
CORNERS = np.array([[(l >> 0) & 1, (l >> 1) & 1, (l >> 2) & 1] for l in range(8)], dtype=float)


def elem_dofs(ne):
    """(n_elements, 24) periodic dofs of every element, e = (oz ny + oy) nx + ox, local node l at (l&1, l>>1&1, l>>2&1)."""
    nx, ny, nz = ne
    oz, oy, ox = (a.ravel() for a in np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij"))
    d = np.empty((ox.size, 24), dtype=np.int64)
    for l in range(8):
        node = (((oz + (l >> 2)) % nz) * ny + (oy + ((l >> 1) & 1)) % ny) * nx + (ox + (l & 1)) % nx
        for c in range(3):
            d[:, 3 * l + c] = 3 * node + c
    return d


def ck_of(ne, h, E, E_field):
    return (np.full(int(np.prod(ne)), E * h) if E_field is None else np.ascontiguousarray(E_field, dtype=np.float64).reshape(-1) * h)


def tensor(strain):
    """3x3 tensor strain of a Voigt strain (11, 22, 33, 23, 13, 12) with engineering shears."""
    e = np.asarray(strain, dtype=float)
    return np.array([[e[0], e[5] / 2, e[4] / 2], [e[5] / 2, e[1], e[3] / 2], [e[4] / 2, e[3] / 2, e[2]]])


def ubar_local(strain, h):
    """(24,) u_bar = eps_bar x at the 8 corners of an element, x relative to its first corner."""
    return (h * CORNERS @ tensor(strain).T).ravel()


def assemble(ne, h=1.0, E=1.0, nu=0.3, E_field=None):
    """Periodic K (scipy CSR, n = 3 nx ny nz)."""
    dofs = elem_dofs(ne)
    ke = hex_element_stiffness(1.0, nu)
    ck = ck_of(ne, h, E, E_field)
    n = 3 * int(np.prod(ne))
    vals = ck[:, None, None] * ke[None]
    rows = np.repeat(dofs[:, :, None], 24, axis=2)
    cols = np.repeat(dofs[:, None, :], 24, axis=1)
    return sp.csr_matrix((vals.ravel(), (rows.ravel(), cols.ravel())), shape=(n, n))


def load(ne, strain, h=1.0, E=1.0, nu=0.3, E_field=None):
    """b = -sum_e P_e^T Ck_e Ke u_bar_e with u_bar_e the element's own (continuous) corner values."""
    dofs = elem_dofs(ne)
    fe = hex_element_stiffness(1.0, nu) @ ubar_local(strain, h)
    ck = ck_of(ne, h, E, E_field)
    b = np.zeros(3 * int(np.prod(ne)))
    np.add.at(b, dofs.ravel(), -(ck[:, None] * fe[None, :]).ravel())
    return b


def solve(K, b):
    """u~ with node 0 pinned (u~ = 0 there): K is singular by the three translations."""
    keep = np.arange(3, K.shape[0])
    x = np.zeros(K.shape[0])
    x[keep] = spla.spsolve(K[keep][:, keep].tocsc(), b[keep])
    return x


def d_matrix(nu):
    """E = 1 Voigt stiffness (engineering shears) with the lambda, mu of hex_element_stiffness."""
    lam = nu / ((1 + nu) * (1 - 2 * nu))
    mu = 1.0 / (2 * (1 + nu))
    D = np.zeros((6, 6))
    D[:3, :3] = lam
    D[np.arange(3), np.arange(3)] += 2 * mu
    D[np.arange(3, 6), np.arange(3, 6)] = mu
    return D


def element_fields(ne, x, strain, h=1.0, E=1.0, nu=0.3, E_field=None):
    """(strain, stress) per element, (n_elements, 6) each: the centroid Q1 strain of u~ plus eps_bar (tensor shears),
    sigma = E_e D eps."""
    dofs = elem_dofs(ne)
    u = x[dofs].reshape(-1, 8, 3)
    s = CORNERS * 2 - 1                                   # signs s_a(l)
    g = np.einsum("la,eli->eai", s, u) * (0.25 / h)       # g[e, a, i] = d u_i / d x_a
    eps = np.stack([g[:, 0, 0], g[:, 1, 1], g[:, 2, 2], 0.5 * (g[:, 1, 2] + g[:, 2, 1]), 0.5 * (g[:, 0, 2] + g[:, 2, 0]),
                    0.5 * (g[:, 0, 1] + g[:, 1, 0])], axis=1)
    e = np.asarray(strain, dtype=float)
    eps = eps + np.concatenate([e[:3], 0.5 * e[3:]])[None, :]
    Ee = ck_of(ne, h, E, E_field) / h
    eng = eps.copy()
    eng[:, 3:] *= 2
    return eps, Ee[:, None] * (eng @ d_matrix(nu).T)


def effective_stiffness(ne, h=1.0, E=1.0, nu=0.3, E_field=None, return_u=False):
    """C (6x6, column j = <sigma> under unit strain j) and, with return_u, the 6 fluctuations."""
    K = assemble(ne, h, E, nu, E_field)
    C = np.empty((6, 6))
    us = []
    for j in range(6):
        strain = np.eye(6)[j]
        x = solve(K, load(ne, strain, h, E, nu, E_field))
        C[:, j] = element_fields(ne, x, strain, h, E, nu, E_field)[1].mean(axis=0)
        us.append(x)
    return (C, us) if return_u else C


def energy(ne, x, strain_i, xj, strain_j, h=1.0, E=1.0, nu=0.3, E_field=None):
    """(1/V) sum_e Ck_e (u_bar_i + u~_i)_e^T Ke (u_bar_j + u~_j)_e over each element's own 24 dofs."""
    dofs = elem_dofs(ne)
    ke = hex_element_stiffness(1.0, nu)
    ck = ck_of(ne, h, E, E_field)
    ui = x[dofs] + ubar_local(strain_i, h)[None, :]
    uj = xj[dofs] + ubar_local(strain_j, h)[None, :]
    return float(np.sum(ck * np.einsum("ea,ab,eb->e", ui, ke, uj))) / (int(np.prod(ne)) * h ** 3)


def laminate(E_layers, fractions, nu):
    """Closed-form effective stiffness (Voigt, engineering shears) of isotropic layers normal to z: traction components
    t = (33, 23, 13) continuous, in-plane strains p = (11, 22, 12) continuous."""
    t, p = [2, 3, 4], [0, 1, 5]
    D = d_matrix(nu)
    inv_tt = sum(f * np.linalg.inv(E * D[np.ix_(t, t)]) for E, f in zip(E_layers, fractions))
    a_tp = sum(f * np.linalg.solve(E * D[np.ix_(t, t)], E * D[np.ix_(t, p)]) for E, f in zip(E_layers, fractions))
    s_pp = sum(f * (E * D[np.ix_(p, p)] - E * D[np.ix_(p, t)] @ np.linalg.solve(E * D[np.ix_(t, t)], E * D[np.ix_(t, p)]))
               for E, f in zip(E_layers, fractions))
    Ctt = np.linalg.inv(inv_tt)
    Ctp = Ctt @ a_tp
    C = np.zeros((6, 6))
    C[np.ix_(t, t)] = Ctt
    C[np.ix_(t, p)] = Ctp
    C[np.ix_(p, t)] = Ctp.T
    C[np.ix_(p, p)] = s_pp + a_tp.T @ Ctt @ a_tp
    return C


VOIGT = [(0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1)]


def rotate_voigt(C, Q):
    """C (Voigt, engineering shears) of the material rotated by Q: C'_ijkl = Q_ia Q_jb Q_kc Q_ld C_abcd."""
    T = np.zeros((3, 3, 3, 3))
    for I, (i, j) in enumerate(VOIGT):
        for J, (k, l) in enumerate(VOIGT):
            for a, b in ((i, j), (j, i)):
                for c, d in ((k, l), (l, k)):
                    T[a, b, c, d] = C[I, J]
    R = np.einsum("ia,jb,kc,ld,abcd->ijkl", Q, Q, Q, Q, T)
    return np.array([[R[i, j, k, l] for (k, l) in VOIGT] for (i, j) in VOIGT])


# ---- restatements of the device kernels -----------------------------------------------------------------------------

def node_coords(ne, nodes):
    nx, ny, _ = ne
    nodes = np.asarray(nodes, dtype=np.int64)
    return nodes % nx, (nodes // nx) % ny, nodes // (nx * ny)


def ref_rows(ne, rows, xval, ck, nu=0.3):
    """(y, abs_sum, count) in long double for dofs `rows` of the periodic operator's per-node sum: la ascending over the 8
    elements around the node (wrapped), Ck_e Ke[3 la + d][3 lb + dd] x(node, lb - la, dd).  xval(nodes, dx, dy, dz, dd) ->
    float64 values of x at node + (dx, dy, dz); ck (n_elements,) the Ck field."""
    nx, ny, nz = ne
    ke = hex_element_stiffness(1.0, nu).astype(np.longdouble)
    rows = np.asarray(rows, dtype=np.int64)
    node, d = rows // 3, rows % 3
    lx, ly, lz = node_coords(ne, node)
    y = np.zeros(rows.size, dtype=np.longdouble)
    s = np.zeros(rows.size, dtype=np.longdouble)
    for la in range(8):
        ax, ay, az = la & 1, (la >> 1) & 1, la >> 2
        e = (((lz - az) % nz) * ny + (ly - ay) % ny) * nx + (lx - ax) % nx
        c = np.asarray(ck[e], dtype=np.longdouble)
        for lb in range(8):
            dx, dy, dz = (lb & 1) - ax, ((lb >> 1) & 1) - ay, (lb >> 2) - az
            for dd in range(3):
                t = ke[3 * la + d, 3 * lb + dd] * (c * np.asarray(xval(node, dx, dy, dz, dd), dtype=np.longdouble))
                y += t
                s += np.abs(t)
    return y, s, np.full(rows.size, 8 * 25)


def x_fetch(ne, x):
    nx, ny, nz = ne

    def f(node, dx, dy, dz, dd):
        lx, ly, lz = node_coords(ne, node)
        return x[3 * ((((lz + dz) % nz) * ny + (ly + dy) % ny) * nx + (lx + dx) % nx) + dd]
    return f


def ubar_table(strain, h):
    """u_bar(node + d) - u_bar(node) = eps_bar h d as the device computes it: (E_i0 h d0 + E_i1 h d1) + E_i2 h d2."""
    Et = tensor(strain)
    eh = Et * h

    def f(node, dx, dy, dz, dd):
        return np.full(np.shape(node), (dx * eh[dd, 0] + dy * eh[dd, 1]) + dz * eh[dd, 2])
    return f


def assert_rows(yrows, ref):
    y, s, k = ref
    yrows = np.asarray(yrows)
    assert not np.isnan(yrows).any(), f"{int(np.isnan(yrows).sum())} rows never written"
    err = np.abs(yrows.astype(np.longdouble) - y)
    bad = np.nonzero(err > (k + 2) * EPS * s)[0]
    assert bad.size == 0, f"{bad.size} rows off, first {bad[:5]}: err {err[bad[:5]]}"


def ref_diag(ne, ck, nu=0.3):
    """The periodic diagonal bit for bit: d = 0.0; d = d + Ck_e Ke[3la+dir][3la+dir] over the 8 elements, ascending la."""
    nx, ny, nz = ne
    kd = np.diag(hex_element_stiffness(1.0, nu))
    lx, ly, lz = node_coords(ne, np.arange(int(np.prod(ne))))
    d = np.zeros((lx.size, 3))
    for la in range(8):
        e = (((lz - (la >> 2)) % nz) * ny + (ly - ((la >> 1) & 1)) % ny) * nx + (lx - (la & 1)) % nx
        d = d + ck[e][:, None] * kd[3 * la: 3 * la + 3][None, :]
    return d.ravel()


BRICK = (32, 4, 2)


def ref_average(ne, vals):
    """The device average's order applied to per-element values vals (n_elements, k): bricks of 32 x 4 x 2 elements,
    thread t = tx + 32 ty + 128 tz (0.0 outside the cell), a halving tree v[t] + v[t + w] per brick, then c = ceil(nb /
    256) consecutive partials per thread from 0.0 in ascending order, the same tree over the 256 sums, / n_elements."""
    nx, ny, nz = ne
    bx, by, bz = BRICK
    nbx, nby, nbz = -(-nx // bx), -(-ny // by), -(-nz // bz)
    k = vals.shape[1]
    grid = np.zeros((nbz * bz, nby * by, nbx * bx, k))
    grid[:nz, :ny, :nx] = vals.reshape(nz, ny, nx, k)
    v = grid.reshape(nbz, bz, nby, by, nbx, bx, k).transpose(0, 2, 4, 1, 3, 5, 6).reshape(nbz * nby * nbx, bz * by * bx, k)

    def tree(a):
        while a.shape[1] > 1:
            w = a.shape[1] // 2
            a = a[:, :w] + a[:, w:]
        return a[:, 0]
    part = tree(v)
    nb = part.shape[0]
    c = -(-nb // 256)
    acc = np.zeros((256, k))
    for i in range(c):
        idx = np.arange(256) * c + i
        ok = (idx < nb) & (idx < (np.arange(256) + 1) * c)
        acc[ok] = acc[ok] + part[idx[ok]]
    return tree(acc[None])[0] / float(nx * ny * nz)
