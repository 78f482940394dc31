"""CPU ORACLE (test infrastructure - never imported by the product path).

A numpy restatement of the reference's hot path, each function citing the reference lines it follows
(all paths relative to the reference repository):

    ref_pcg            <- PCG(RefMeshPart)                     src/solver/pcg_solver.py:356-598
    EbePart.matvec     <- calcMatVecProd(...,'Strain')         src/solver/pcg_solver.py:242-300
    EbePart.diag       <- calcMatVecProd(...,'Preconditioner') src/solver/pcg_solver.py:282-287
    exchange_add       <- interface exchange                   src/solver/pcg_solver.py:303-334
    jacobi             <- updatePreconditioner                 src/solver/pcg_solver.py:346-352
    update_bc          <- updateBC                             src/solver/pcg_solver.py:226-238

The reference runs one MPI rank per mesh part; here the parts of a run are advanced in lock-step inside
one process ("SPMD emulation"): every per-rank vector is a list with one numpy array per part, a
local dot followed by MPI_SUM (pcg_solver.py:622-628) becomes a Python sum over the parts in rank
order, and the Isend/Recv pairs become direct reads of the neighbour's array.

PINNING (see tests/test_oracle_golden.py): the restatement is checked against golden vectors produced
by the UNMODIFIED reference run under oracle/fake_mpi (oracle/make_golden_*.py): a structured hex
model in the reference's own MDF format (full solution vectors, 1/2/4 parts) and data/concrete.zip
(Flag / Iter / RelRes / norms / sampled solution, 1 and 8 parts).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

EPS = np.finfo(float).eps  # pcg_solver.py:972


# ----------------------------------------------------------------------------------------- operators
class CsrPart:
    """One mesh part with its operator assembled to CSR on the free dofs (A = K_i[Eff,Eff])."""

    def __init__(self, A, b, nbr=(), ovrlp=(), w=None, x0=None, part_id=0):
        self.A = sp.csr_matrix(A)
        self.n = self.A.shape[0]
        self.b = np.asarray(b, dtype=float)
        self.nbr = list(nbr)
        self.ovrlp = [np.asarray(v, dtype=np.int64) for v in ovrlp]
        self.w = np.ones(self.n) if w is None else np.asarray(w, dtype=float)
        self.x0 = np.zeros(self.n) if x0 is None else np.asarray(x0, dtype=float)
        self.id = part_id

    def matvec(self, x):
        return self.A @ x

    def diag(self):
        return self.A.diagonal()


class EbePart:
    """One mesh part in the reference's own element-by-element form (a decoded N_<id>.mpidat dict or the
    output of the product's subdomain builder).  Vectors handed in/out live on the free dofs; the
    scatter to / gather from the full local dof vector is pcg_solver.py:482-484."""

    def __init__(self, mp, time_step_delta=1.0):
        self.mp = mp
        self.id = int(mp["Id"])
        self.ndof = int(mp["NDOF"])
        self.eff = np.asarray(mp["LocDofEff"], dtype=np.int64)
        self.n = len(self.eff)
        self.nbr = [int(v) for v in mp["NbrMPIdVector"]]
        self.ovrlp_full = [np.asarray(v, dtype=np.int64) for v in mp["OvrlpLocalDofVecList"]]
        self.w = np.asarray(mp["DofWeightVector"], dtype=float)[self.eff]  # pcg_solver.py:997
        self.groups = mp["SubDomainData"]["StrucDataList"]
        self.flat = np.asarray(mp["Flat_ElemLocDof"], dtype=np.int64)
        self.ncount = int(mp["NCountDof"])
        self.delta = time_step_delta
        self.x0 = np.zeros(self.n)
        self.b = None  # filled by update_bc

    # calcMatVecProd 'Strain', FintCalcMode 'outbin' (pcg_solver.py:256-300), full local vectors
    def matvec_full(self, x_full):
        flat = np.zeros(self.ncount)
        i = 0
        for g in self.groups:
            dofs = g["ElemList_LocDofVector"]
            sign = g["ElemList_SignVector"]
            u = x_full[dofs]                       # :277
            u[sign] *= -1.0                        # :278
            v = g["ElemStiffMat"] @ (g["ElemList_Ck"] * u)  # :279
            v[sign] *= -1.0                        # :280
            n = dofs.size
            flat[i:i + n] = v.ravel()              # :294-297
            i += n
        return np.bincount(self.flat, weights=flat, minlength=self.ndof)  # :300

    def diag_full(self):
        flat = np.zeros(self.ncount)
        i = 0
        for g in self.groups:
            v = g["ElemList_Ck"] * g["ElemDiagStiffMat"][np.newaxis].T  # :287
            n = v.size
            flat[i:i + n] = v.ravel()
            i += n
        return np.bincount(self.flat, weights=flat, minlength=self.ndof)


def exchange_add_full(parts, ys):
    """pcg_solver.py:303-334 on full local vectors: y[Ovrlp_j] += (neighbour j's y[its Ovrlp towards me])."""
    byid = {p.id: k for k, p in enumerate(parts)}
    sends = [[y[idx].copy() for idx in p.ovrlp_full] for p, y in zip(parts, ys)]  # :307-309
    for k, p in enumerate(parts):
        for j, nb in enumerate(p.nbr):  # :332-334, neighbour order
            q = parts[byid[nb]]
            ys[k][p.ovrlp_full[j]] += sends[byid[nb]][q.nbr.index(p.id)]
    return ys


def exchange_add(parts, ys):
    """Same exchange for parts whose vectors live on the free dofs (CsrPart)."""
    byid = {p.id: k for k, p in enumerate(parts)}
    sends = [[y[idx].copy() for idx in p.ovrlp] for p, y in zip(parts, ys)]
    for k, p in enumerate(parts):
        for j, nb in enumerate(p.nbr):
            q = parts[byid[nb]]
            ys[k][p.ovrlp[j]] += sends[byid[nb]][q.nbr.index(p.id)]
    return ys


class Operator:
    """calcMPFint (pcg_solver.py:339-342) over all parts, on free-dof vectors."""

    def __init__(self, parts, comm=None):
        self.parts = parts
        self.ebe = isinstance(parts[0], EbePart)
        self.matvecs = 0
        self.comm = comm   # SPMD mode (oracle/spmd.py): this process holds ONE part, neighbours live in other processes

    def apply(self, xs):
        self.matvecs += 1
        if self.ebe:
            fulls = []
            for p, x in zip(self.parts, xs):
                xf = np.zeros(p.ndof)
                xf[p.eff] = x                      # :482  (fixed dofs stay zero)
                fulls.append(p.matvec_full(xf))
            fulls = self.comm.exchange_add_full(self.parts[0], fulls[0]) if self.comm else exchange_add_full(self.parts, fulls)
            fulls = [fulls] if self.comm else fulls
            return [f[p.eff] for p, f in zip(self.parts, fulls)]  # :484
        return exchange_add(self.parts, [p.matvec(x) for p, x in zip(self.parts, xs)])

    def jacobi(self):
        """updatePreconditioner (pcg_solver.py:346-352): 1/diag(K) assembled over the interface."""
        if self.ebe:
            if self.comm:
                ds = [self.comm.exchange_add_full(self.parts[0], self.parts[0].diag_full())]
            else:
                ds = exchange_add_full(self.parts, [p.diag_full() for p in self.parts])
            return [(1.0 / d)[p.eff] for p, d in zip(self.parts, ds)]
        ds = exchange_add(self.parts, [p.diag() for p in self.parts])
        return [1.0 / d for d in ds]


def update_bc(parts, delta=1.0, comm=None):
    """updateBC (pcg_solver.py:226-238) for EbeParts: Fext = F*delta - K (Ud*delta); sets p.b and returns Udi."""
    udis = [np.asarray(p.mp["Ud"], dtype=float) * delta for p in parts]
    if comm:
        fdis = [comm.exchange_add_full(parts[0], parts[0].matvec_full(udis[0]))]
    else:
        fdis = exchange_add_full(parts, [p.matvec_full(u) for p, u in zip(parts, udis)])
    for p, fdi in zip(parts, fdis):
        fext = np.asarray(p.mp["RefLoadVector"], dtype=float) * delta - fdi
        p.b = fext[p.eff]                          # :377
    return udis


# ----------------------------------------------------------------------------------------- PCG
def _mpi_sum_local(vals):
    """MPI_SUM (pcg_solver.py:622-628): allreduce(SUM) - here a sum over the parts in rank order."""
    tot = vals[0]
    for v in vals[1:]:
        tot = tot + v
    return tot


def ref_pcg(parts, minv, tol, maxiter, nglob=None, resvec=None, exist_dp0=True, comm=None, trace=None, maxstag=3):
    """PCG(RefMeshPart), pcg_solver.py:356-598, for all parts in lock-step.

    comm: None = all parts live in this process (lock-step emulation); an oracle/spmd.ShmComm = SPMD mode, `parts`
    holds this process's single part and reductions / interface sums go through shared memory.
    parts: list of CsrPart / EbePart (fields b, x0, w).  minv: list of InvDiagPreCondVector0 per part
    (ignored when exist_dp0 is False, :446-451).  nglob: GlobNDofEff.  Returns a dict with
    X (list per part), Flag, RelRes, Iter and bookkeeping.  If `resvec` is a list, ||r|| per
    iteration is appended (the reference has this commented out, :428-434, :520-525).  If `trace` is a list, one dict
    per control step is appended with the reduced values it consumed (sums before their sqrt): start (bb, r0r0), head
    (i, ninf, rz), pq, norms (pp, xx, rr, stag), verify (rr, stop) and final (rr of the XMin residual, 0 when converged);
    tests/pcg_shadow.py replays them.
    """
    def _tr(step, **kv):
        if trace is not None:
            trace.append(dict(step=step, **kv))

    op = Operator(parts, comm)
    _mpi_sum = (lambda vals: comm.allreduce(_mpi_sum_local(vals))) if comm else _mpi_sum_local  # noqa: F811
    P = len(parts)
    rng = range(P)
    W = [p.w for p in parts]
    if nglob is None:
        nglob = int(round(sum(float(w.sum()) for w in W)))
    Fext = [np.array(p.b, dtype=float) for p in parts]                 # :377
    X = [np.array(p.x0, dtype=float) for p in parts]                   # :378-379
    XMin = [x for x in X]                                              # :380  MP_XMin = MP_X: the SAME array ...
    aliased = True                                                     # ... until the first np.array(MP_X) copy (:557)
    bb = _mpi_sum([np.dot(Fext[k], Fext[k] * W[k]) for k in rng])
    n2b = np.sqrt(bb)                                                  # :381-383
    tolb = tol * n2b                                                   # :384
    if n2b == 0:                                                       # :387-395 (returns the initial guess)
        return dict(X=X, Flag=0, RelRes=0.0, Iter=0, iMin=0, matvecs=op.matvecs, normb=0.0)
    flag, rho, stag, moresteps = 1, 1.0, 0, 0                          # :399-402
    maxstag = maxstag if maxstag > 0 else 3                            # MaxStagSteps = 3 (:403)
    maxmsteps = min([int(nglob / 50), 5, nglob - maxiter])             # :404
    imin, it = 0, 0                                                    # :405-406
    q0 = op.apply(X)                                                   # :411-413
    R = [Fext[k] - q0[k] for k in rng]                                 # :414
    r0r0 = _mpi_sum([np.dot(R[k], R[k] * W[k]) for k in rng])
    normr = np.sqrt(r0r0)                                              # :415-416
    _tr("start", bb=float(bb), r0r0=float(r0r0))
    normrmin = normr                                                   # :417
    normr_act = normr                                                  # :418
    if resvec is not None:
        resvec.append(normr)
    if normr <= tolb:                                                  # :421-426
        return dict(X=X, Flag=0, RelRes=normr / n2b, Iter=0, iMin=0, matvecs=op.matvecs, normb=n2b)
    Pv = [None] * P
    too_small = False
    i = 0
    for i in range(maxiter):                                           # :438
        if exist_dp0:                                                  # :446-451
            Z = [minv[k] * R[k] for k in rng]
            if any(np.any(np.isinf(z)) for z in Z):
                _tr("head", i=i, ninf=1.0)
                flag = 2
                break
        else:
            Z = R
        rho_1 = rho                                                    # :461
        rho = _mpi_sum([np.dot(Z[k], R[k] * W[k]) for k in rng])       # :462-463
        _tr("head", i=i, ninf=0.0, rz=float(rho))
        if rho == 0 or np.isinf(rho):                                  # :467-469
            flag = 4
            break
        if i == 0:                                                     # :472-479
            Pv = [np.array(z) for z in Z]
        else:
            beta = rho / rho_1
            if beta == 0 or np.isinf(beta):
                flag = 4
                break
            Pv = [Z[k] + beta * Pv[k] for k in rng]
        Q = op.apply(Pv)                                               # :482-484
        pq = _mpi_sum([np.dot(Pv[k], Q[k] * W[k]) for k in rng])       # :487-488
        _tr("pq", i=i, pq=float(pq))
        if pq <= 0 or np.isinf(pq):                                    # :492-498
            flag = 4
            break
        alpha = rho / pq
        if np.isinf(alpha):
            flag = 4
            break
        for k in rng:
            R[k] = R[k] - alpha * Q[k]                                 # :501
        sq = _mpi_sum([np.array([np.dot(Pv[k], Pv[k] * W[k]), np.dot(X[k], X[k] * W[k]), np.dot(R[k], R[k] * W[k])])
                       for k in rng])                                  # :504-507
        normp, normx, normr = np.sqrt(sq)
        if normp * abs(alpha) < EPS * normx:                           # :512-513
            stag += 1
        else:
            stag = 0
        _tr("norms", i=i, pp=float(sq[0]), xx=float(sq[1]), rr=float(sq[2]), stag=stag)
        X = [X[k] + alpha * Pv[k] for k in rng]                        # :516 in place in the reference, so an XMin that is
        if aliased:                                                    #      still bound to MP_X follows the update
            XMin = X
        normr_act = normr                                              # :518
        if resvec is not None:
            resvec.append(normr)
        if normr <= tolb or stag >= maxstag or moresteps > 0:          # :527
            fint = op.apply(X)                                         # :528-530
            R = [Fext[k] - fint[k] for k in rng]                       # :531
            rr_act = _mpi_sum([np.dot(R[k], R[k] * W[k]) for k in rng])
            normr_act = np.sqrt(rr_act)                                # :532-533
            _tr("verify", i=i, rr=float(rr_act), stop=True)
            if resvec is not None:
                resvec[-1] = normr_act
            if normr_act <= tolb:                                      # :540-543
                flag = 0
                it = i
                break
            if stag >= maxstag and moresteps == 0:                     # :545
                stag = 0
            moresteps += 1                                             # :546
            if moresteps >= maxmsteps:                                 # :548-552 - the reference RAISES here
                too_small = True                                       #   (Warning is an Exception); the lines
                flag = 3                                               #   after it (Flag=3, Iter=i) are what
                it = i                                                 #   MATLAB does and what we report
                break
            if trace is not None and stag < maxstag:                   # the loop goes on after this verification
                trace[-1]["stop"] = False
        if normr_act < normrmin:                                       # :555-558
            normrmin = normr_act
            XMin = [np.array(x) for x in X]
            aliased = False
            imin = i
        if stag >= maxstag:                                            # :560-562
            flag = 3
            break
    if flag == 0:                                                      # :566-567
        relres = normr_act / n2b
        Xout = X
        _tr("final", rr=0.0)
    else:                                                              # :568-582
        fint = op.apply(XMin)
        Rm = [Fext[k] - fint[k] for k in rng]
        rr_m = _mpi_sum([np.dot(Rm[k], Rm[k] * W[k]) for k in rng])
        normr_m = np.sqrt(rr_m)
        _tr("final", rr=float(rr_m))
        if normr_m < normr_act:
            it = imin
            relres = normr_m / n2b
        else:
            it = i
            relres = normr_act / n2b
        Xout = XMin                                                    # :569 + :598: Un is built from XMin
    it += 1                                                            # :584
    return dict(X=Xout, Flag=flag, RelRes=float(relres), Iter=int(it), iMin=imin, matvecs=op.matvecs,
                normb=float(n2b), too_small_tol=too_small, stag=stag, moresteps=moresteps, aliased=aliased)


# ----------------------------------------------------------------------------------------- test problems
def poisson27(n: int):
    """Config C1 (SURVEY 8(d)): 27-point operator on an n^3 grid, Dirichlet truncation: diagonal 26,
    off-diagonals -1 (SPD).  Returns scipy CSR with sorted indices."""
    idx = np.arange(n ** 3).reshape(n, n, n)  # [z, y, x], x fastest
    rows, cols, vals = [], [], []
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                src = idx[max(0, -dz):n - max(0, dz), max(0, -dy):n - max(0, dy), max(0, -dx):n - max(0, dx)]
                dst = idx[max(0, dz):n - max(0, -dz), max(0, dy):n - max(0, -dy), max(0, dx):n - max(0, -dx)]
                rows.append(src.ravel())
                cols.append(dst.ravel())
                vals.append(np.full(src.size, 26.0 if (dx, dy, dz) == (0, 0, 0) else -1.0))
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n ** 3, n ** 3))
    A.sort_indices()
    return A


def hex_ke(E=1.0, nu=0.3):
    """Q1 hexahedron stiffness (unit edge), written independently of the product's
    hexmesh.hex_element_stiffness: explicit loops over nodes, shape-function gradients from the
    closed form dN_a/dx_c = s_ac * prod_{d != c} (1/2 + s_ad (x_d - 1/2)), s = +-1, on [0,1]^3."""
    lam = E * nu / ((1 + nu) * (1 - 2 * nu))
    mu = E / (2 * (1 + nu))
    C = np.zeros((3, 3, 3, 3))
    for i in range(3):
        for j in range(3):
            for k in range(3):
                for l in range(3):
                    C[i, j, k, l] = lam * (i == j) * (k == l) + mu * ((i == k) * (j == l) + (i == l) * (j == k))
    s = np.array([[1 if (a >> c) & 1 else -1 for c in range(3)] for a in range(8)], dtype=float)
    gp = [0.5 - 0.5 / np.sqrt(3.0), 0.5 + 0.5 / np.sqrt(3.0)]
    Ke = np.zeros((24, 24))
    for x in gp:
        for y in gp:
            for z in gp:
                pt = (x, y, z)
                grad = np.zeros((8, 3))
                for a in range(8):
                    for c in range(3):
                        g = s[a, c]
                        for d in range(3):
                            if d != c:
                                g *= 0.5 + s[a, d] * (pt[d] - 0.5)
                        grad[a, c] = g
                for a in range(8):
                    for b in range(8):
                        for i in range(3):
                            for k in range(3):
                                v = 0.0
                                for j in range(3):
                                    for l in range(3):
                                        v += grad[a, j] * C[i, j, k, l] * grad[b, l]
                                Ke[3 * a + i, 3 * b + k] += v / 8.0
    return Ke


def hex_box_csr(ng, e0, ne, E=1.0, nu=0.3, h=1.0):
    """Sub-assembled K_i[Eff,Eff] of a box of hex elements by plain scipy COO assembly (the oracle for
    csrc/hexgen.cuh).  Same numbering as the product: local nodes x fastest, nodes with global x index
    0 clamped (dropped), dof = 3*freenode + dir."""
    ke = hex_ke(1.0, nu) * (E * h)
    nx, ny, nz = ne
    x_lo = 1 if e0[0] == 0 else 0
    nxf = nx + 1 - x_lo

    def free(lx, ly, lz):
        return (lz * (ny + 1) + ly) * nxf + (lx - x_lo)

    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ex, ey, ez = ex.ravel(), ey.ravel(), ez.ravel()
    dofs = np.empty((ex.size, 24), dtype=np.int64)
    valid = np.empty((ex.size, 24), dtype=bool)
    for l in range(8):
        lx, ly, lz = ex + (l & 1), ey + ((l >> 1) & 1), ez + ((l >> 2) & 1)
        for d in range(3):
            dofs[:, 3 * l + d] = 3 * free(lx, ly, lz) + d
            valid[:, 3 * l + d] = lx >= x_lo
    rows = np.repeat(dofs[:, :, None], 24, axis=2)
    cols = np.repeat(dofs[:, None, :], 24, axis=1)
    ok = valid[:, :, None] & valid[:, None, :]
    vals = np.broadcast_to(ke[None, :, :], rows.shape)
    n = 3 * nxf * (ny + 1) * (nz + 1)
    A = sp.coo_matrix((vals[ok], (rows[ok], cols[ok])), shape=(n, n)).tocsr()
    A.sum_duplicates()
    A.sort_indices()
    return A
