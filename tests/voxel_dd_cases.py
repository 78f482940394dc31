"""Host restatement of the voxel-model multigrid across ranks (pcgb_mg_create_ranks_field, multigrid.HexMultigrid with
`blocks` and the global E_field): the oracle of its tests, built on tests/voxel_cases.py and tests/gmg_dd_cases.py.

Ranked levels 0 .. la are those of gmg_dd_cases.coarsen.  Each rank builds the Galerkin element matrices of its own boxes
from its slice of the fine field; a coarse element's matrix depends on its eight children only, so each equals the slice
of voxel_cases.level_elements(field) at that element.  Level la's matrices are gathered into the global box of la (every
rank writes its own elements into a zeroed array, then one exchange-add), and they are the matrices of the replicated
hierarchy below it, which continues as voxel_cases.HostFieldMultigrid.  The ranked levels smooth with their sub-assembled
matrices and the exchange-add of gmg_dd_cases.HostRankMultigrid.
"""
from __future__ import annotations

import numpy as np

from tests import gmg_dd_cases as D
from tests import voxel_cases as V


def box_slice(a, box):
    """The part of an (nz, ny, nx, ...) array of a level's global box that lies in `box` (a gmg_dd_cases.Box)."""
    return a[box.e0[2]:box.e0[2] + box.ne[2], box.e0[1]:box.e0[1] + box.ne[1], box.e0[0]:box.e0[0] + box.ne[0]]


def rank_elements(levels, field, h, nu=0.3):
    """[l][r]: element matrices of rank r's box at ranked level l = 0 .. la, built as the rank builds them: Ck Ke on its
    slice of the fine field, then Galerkin products of its own elements only."""
    ke = V.R.hex_ke(1.0, nu)
    out = [[V.fine_elements(box_slice(field, b), h, ke) for b in levels[0]]]
    for _ in levels[1:]:
        out.append([V.galerkin(k) for k in out[-1]])
    return out


def gather_elements(level_boxes, kels):
    """The gathered level's element matrices of its global box: each rank's own written into a zeroed array, then the
    sum over ranks (the exchange-add over the all-to-all element plan; one non-zero term per entry)."""
    ng = level_boxes[0].ng
    tot = np.zeros((ng[2], ng[1], ng[0], 24, 24))
    for b, k in zip(level_boxes, kels):
        part = np.zeros_like(tot)
        box_slice(part, b)[...] = k
        tot = tot + part
    return tot


class HostRankFieldMultigrid(D.HostRankMultigrid):
    """gmg_dd_cases.HostRankMultigrid's V-cycle with the ranked levels' matrices assembled from the rank's element matrices
    and the replicated hierarchy built from the gathered ones.  lambdas: the global hierarchy's estimates (ranked levels
    below la, then the replicated ones), as HexMultigrid.info()["global_lambda"] or HostFieldMultigrid.lam."""

    def __init__(self, levels, field, h, lambdas, degree=2, lo=0.25, nu=0.3):
        self.levels, self.la = levels, len(levels) - 1
        la = self.la
        self.kel = rank_elements(levels, field, h, nu)
        self.gathered = gather_elements(levels[la], self.kel[la])
        sub_kel = [self.gathered]
        gl = levels[la][0].ng
        for _ in V.levels_of(gl)[1:]:
            sub_kel.append(V.galerkin(sub_kel[-1]))
        self.sub = V.HostFieldMultigrid(np.ones((gl[2], gl[1], gl[0])), h * 2 ** la, degree, lo, lambdas=list(lambdas[la:]),
                                        mats=[V.assemble(k, None) for k in sub_kel])
        self.A = [[V.assemble(k, None, b.e0) for k, b in zip(self.kel[l], levels[l])] for l in range(la)]
        self.dinv = [[1.0 / d for d in D.exchange(lv, [a.diagonal() for a in A])] for lv, A in zip(levels[:-1], self.A)]
        self.coef = [V.cheb_coeffs(lam, degree, lo) for lam in lambdas[:la]]
