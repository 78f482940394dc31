"""Host restatement of the multigrid preconditioner across ranks (pcgb_mg_create_ranks, multigrid.HexMultigrid with
`blocks`): the oracle of its tests, built on tests/gmg_cases.py.

Ranked levels halve every rank's box (ng, e0, ne) while every rank's ne is even with halves >= 2 and every e0 is even; the
last of them (la) is gathered into its global box, which continues as the one-rank hierarchy.  Vectors of a ranked level are
consistent: every rank's copy of a shared dof holds the full value.  An exchange-add is restated as the sum of every rank's
local vector scattered into the global box, read back at the rank's dofs.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ref_pcg as R
from tests import gmg_cases as G

MAX_GATHERED = 1 << 17
MAX_COARSE = 1536


class Box:
    """One rank's box at one level: global elements ng, first element e0, elements ne, spacing h."""

    def __init__(self, ng, e0, ne, h=1.0):
        self.ng, self.e0, self.ne, self.h = tuple(int(v) for v in ng), tuple(int(v) for v in e0), tuple(int(v) for v in ne), h

    @property
    def x_lo(self):
        return 1 if self.e0[0] == 0 else 0

    @property
    def n(self):
        return 3 * (self.ne[0] + 1 - self.x_lo) * (self.ne[1] + 1) * (self.ne[2] + 1)

    def half(self):
        return Box([v // 2 for v in self.ng], [v // 2 for v in self.e0], [v // 2 for v in self.ne], 2 * self.h)

    def global_dofs(self):
        """Global free-dof index (the global box's numbering, x = 0 clamped) of every local dof."""
        lz, ly, lx = np.meshgrid(np.arange(self.ne[2] + 1), np.arange(self.ne[1] + 1), np.arange(self.x_lo, self.ne[0] + 1), indexing="ij")
        gn = ((lz.ravel() + self.e0[2]) * (self.ng[1] + 1) + ly.ravel() + self.e0[1]) * self.ng[0] + (lx.ravel() + self.e0[0] - 1)
        return (3 * gn[:, None] + np.arange(3)[None, :]).ravel()

    def csr(self):
        return R.hex_box_csr(self.ng, self.e0, self.ne, h=self.h)


def grid_boxes(pgrid, per, h=None):
    """pgrid[0] x pgrid[1] x pgrid[2] boxes of per^3 elements (rank = x fastest), as hexmesh.partition_blocks cuts them."""
    ng = [pgrid[a] * per for a in range(3)]
    h = 1.0 / ng[0] if h is None else h
    return [Box(ng, (px * per, py * per, pz * per), (per, per, per), h)
            for pz in range(pgrid[2]) for py in range(pgrid[1]) for px in range(pgrid[0])]


def nfree(ne):
    return G.nfree(ne)


def coarsen(boxes):
    """(levels, refusal): levels[l] = the boxes of ranked level l, l = 0 .. la; refusal = None or the reason."""
    ng = boxes[0].ng
    cover = np.zeros((ng[2], ng[1], ng[0]), dtype=np.int64)
    for b in boxes:
        if b.ng != ng or any(b.e0[a] < 0 or b.ne[a] <= 0 or b.e0[a] + b.ne[a] > ng[a] for a in range(3)):
            return None, "tile"
        cover[b.e0[2]:b.e0[2] + b.ne[2], b.e0[1]:b.e0[1] + b.ne[1], b.e0[0]:b.e0[0] + b.ne[0]] += 1
    if np.any(cover != 1):
        return None, "tile"
    levels = [list(boxes)]
    while all(v % 2 == 0 and v // 2 >= 2 for b in levels[-1] for v in b.ne) and all(v % 2 == 0 for b in levels[-1] for v in b.e0):
        levels.append([b.half() for b in levels[-1]])
    if len(levels) == 1:
        return None, "coarsen"
    gl = levels[-1][0].ng
    if 3 * nfree(gl) > MAX_GATHERED:
        return None, "gathered"
    if 3 * nfree(G.levels_of(gl)[-1]) > MAX_COARSE:
        return None, "coarse"
    return levels, None


def global_boxes(levels):
    """The global boxes of the whole hierarchy: those of the ranked levels below la, then levels_of the gathered box."""
    return [b[0].ng for b in levels[:-1]] + G.levels_of(levels[-1][0].ng)


def lists(level_boxes, rank):
    """Neighbours, shared local-dof lists (ascending global node, 3 dofs per node) and 0/1 ownership (lowest rank owns)."""
    me = level_boxes[rank]
    gm = me.global_dofs()
    nbr, out = [], []
    w = np.ones(me.n)
    for r, other in enumerate(level_boxes):
        if r == rank:
            continue
        common = np.intersect1d(gm, other.global_dofs())
        if common.size == 0:
            continue
        loc = np.searchsorted(gm, common)     # gm ascends with the local index
        nbr.append(r)
        out.append(loc.astype(np.int64))
        if r < rank:
            w[loc] = 0.0
    return nbr, out, w


def exchange(level_boxes, locals_):
    """The exchange-add of every rank's local vector: the global sum read back at each rank's dofs."""
    n = 3 * nfree(level_boxes[0].ng)
    tot = np.zeros(n)
    for b, v in zip(level_boxes, locals_):
        np.add.at(tot, b.global_dofs(), v)
    return [tot[b.global_dofs()] for b in level_boxes]


def to_local(level_boxes, v):
    return [v[b.global_dofs()] for b in level_boxes]


def prolongation_box(bf: Box):
    """Local P of a rank's box (fine box bf, coarse box bf.half()): trilinear gather in local coordinates."""
    bc = bf.half()
    nxf_f = bf.ne[0] + 1 - bf.x_lo
    nxf_c = bc.ne[0] + 1 - bc.x_lo
    fz, fy, fx = np.meshgrid(np.arange(bf.ne[2] + 1), np.arange(bf.ne[1] + 1), np.arange(bf.x_lo, bf.ne[0] + 1), indexing="ij")
    fz, fy, fx = fz.ravel(), fy.ravel(), fx.ravel()
    rows, cols, vals = [], [], []
    for kz in (0, 1):
        for ky in (0, 1):
            for kx in (0, 1):
                cz, cy, cx = (fz >> 1) + kz, (fy >> 1) + ky, (fx >> 1) + kx
                w = np.ones(fx.size)
                for f, k in ((fz, kz), (fy, ky), (fx, kx)):
                    w *= np.where(f % 2 == 1, 0.5, np.where(k == 0, 1.0, 0.0))
                ok = (w > 0) & (cx >= bc.x_lo)
                cnode = (cz * (bc.ne[1] + 1) + cy) * nxf_c + (cx - bc.x_lo)
                fnode = (fz * (bf.ne[1] + 1) + fy) * nxf_f + (fx - bf.x_lo)
                for d in range(3):
                    rows.append(3 * fnode[ok] + d)
                    cols.append(3 * cnode[ok] + d)
                    vals.append(w[ok])
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(bf.n, bc.n))


def restrict_ranks(levels, l, rf_locals, weighted=True):
    """P^T r across ranks: each rank restricts its owned fine dofs, the coarse level's exchange-add completes the sum."""
    parts = []
    for r, bf in enumerate(levels[l]):
        own = lists(levels[l], r)[2] if weighted else np.ones(bf.n)
        parts.append(prolongation_box(bf).T @ np.where(own != 0, rf_locals[r], 0.0))
    return exchange(levels[l + 1], parts)


def gather(level_boxes, locals_):
    """The gathered level's global vector: every rank writes its owned entries, the rest are 0, then one exchange-add."""
    n = 3 * nfree(level_boxes[0].ng)
    tot = np.zeros(n)
    for r, (b, v) in enumerate(zip(level_boxes, locals_)):
        own = lists(level_boxes, r)[2]
        part = np.zeros(n)
        part[b.global_dofs()] = np.where(own != 0, v, 0.0)
        tot = tot + part
    return tot


def lanczos_ranks(level_boxes, dinv_locals, steps=G.LANCZOS_STEPS):
    """lambda of D^-1 A on a ranked level: consistent vectors, owner-weighted inner products summed over ranks, start
    vector at the global free index."""
    A = [b.csr() for b in level_boxes]
    own = [lists(level_boxes, r)[2] for r in range(len(level_boxes))]

    def dot(a, b):
        return sum(float(np.dot(a[r] * own[r], b[r])) for r in range(len(a)))

    v = [G.start_vector(3 * nfree(level_boxes[0].ng))[b.global_dofs()] for b in level_boxes]
    nv = np.sqrt(dot(v, [x / d for x, d in zip(v, dinv_locals)]))
    v = [x / nv for x in v]
    vp, beta, al, be = [np.zeros_like(x) for x in v], 0.0, [], []
    for it in range(steps):
        y = exchange(level_boxes, [a @ x for a, x in zip(A, v)])
        al.append(dot(v, y))
        if it + 1 == steps:
            break
        w = [d * yy - al[-1] * x - beta * p for d, yy, x, p in zip(dinv_locals, y, v, vp)]
        beta = np.sqrt(dot(w, [x / d for x, d in zip(w, dinv_locals)]))
        be.append(beta)
        vp, v = v, [x / beta for x in w]
    return np.linalg.eigvalsh(np.diag(al) + np.diag(be, 1) + np.diag(be, -1))[-1]


class HostRankMultigrid:
    """The V-cycle across ranks on the host: ranked levels 0 .. la-1 smooth on local operators with exchanges, level la is
    gathered, the global hierarchy below it is gmg_cases.HostMultigrid's.  lambdas: the global hierarchy's estimates."""

    def __init__(self, levels, h, lambdas, degree=2, lo=0.25):
        self.levels, self.la = levels, len(levels) - 1
        gb = global_boxes(levels)
        self.host = G.HostMultigrid(gb[0], h, degree, lo, lambdas=lambdas)
        self.sub = G.HostMultigrid(gb[self.la], h * 2 ** self.la, degree, lo, lambdas=list(lambdas[self.la:]))
        self.A = [[b.csr() for b in lv] for lv in levels[:-1]]
        self.dinv = [[1.0 / d for d in exchange(lv, [a.diagonal() for a in A])] for lv, A in zip(levels[:-1], self.A)]
        self.coef = [G.cheb_coeffs(lam, degree, lo) for lam in lambdas[:self.la]]

    def op(self, l, xs):
        return exchange(self.levels[l], [a @ x for a, x in zip(self.A[l], xs)])

    def smooth(self, l, b, x, zero_start, resid=False):
        inv_theta, c1, c2 = self.coef[l]
        dinv = self.dinv[l]
        r = [v.copy() for v in b] if zero_start else [bb - q for bb, q in zip(b, self.op(l, x))]
        d = [inv_theta * (di * ri) for di, ri in zip(dinv, r)]
        x = [v.copy() for v in d] if zero_start else [xx + dd for xx, dd in zip(x, d)]
        for j in range(len(c1)):
            q = self.op(l, d)
            r = [ri - qi for ri, qi in zip(r, q)]
            d = [c1[j] * dd + c2[j] * (di * ri) for dd, di, ri in zip(d, dinv, r)]
            x = [xx + dd for xx, dd in zip(x, d)]
        if resid:
            q = self.op(l, d)
            r = [ri - qi for ri, qi in zip(r, q)]
        return x, r

    def apply(self, r_locals):
        la = self.la
        b, x = [None] * (la + 1), [None] * (la + 1)
        b[0] = r_locals
        for l in range(la):
            x[l], res = self.smooth(l, b[l], None, True, resid=True)
            b[l + 1] = restrict_ranks(self.levels, l, res)
        xg = self.sub.apply(gather(self.levels[la], b[la]))
        x[la] = to_local(self.levels[la], xg)
        for l in range(la - 1, -1, -1):
            x[l] = [prolongation_box(bf) @ xc + xf for bf, xc, xf in zip(self.levels[l], x[l + 1], x[l])]
            x[l], _ = self.smooth(l, b[l], x[l], False)
        return x[0]
