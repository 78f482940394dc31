"""Effective (homogenised) elastic stiffness of a periodic voxel cell (DESIGN §2.13).

For each of the 6 unit macroscopic strains eps_bar (Voigt 11, 22, 33, 23, 13, 12 with engineering shears) the periodic
fluctuation u~ solves K u~ = -K u_bar, u_bar = eps_bar x, by Jacobi-PCG on the index-free periodic operator; the volume
average of the stress is then column j of C_eff:

    from pcg_mpi_solver_b200.hexmesh import PeriodicCell, inclusion_field
    cell = PeriodicCell((64, 64, 64), h=1.0 / 64, nu=0.2)
    C, infos = effective_stiffness(cell, E_field=inclusion_field((64, 64, 64), E_inclusion=10.0))

Every hot step runs on the device: the operator (k_hexop's periodic variant), the load (k_hexop_load) and the fused
element pass with its fixed-order average (k_fields_average).  The multigrid does not take periodic cells, so the
iteration count grows with the cell size.
"""
from __future__ import annotations

import numpy as np
import torch

from .fields import PeriodicFields
from .hexmesh import PeriodicCell, generate_periodic_operator, hex_element_stiffness
from .solver import SolveInfo, SubdomainOperator

# A load case is skipped (u~ = 0, 0 iterations) when the RMS entry of b is at most SKIP_RMS times the element-load scale
# max Ck * max|Ke| * h * max|eps_bar|.  Each entry of b sums 192 products of at most that size, so in a homogeneous cell,
# where b is zero in exact arithmetic, its rounding noise is below 192 * 2^-53 (about 2e-14) of the scale; a material
# interface gives entries of the order of the scale times the contrast step.  Solving noise to a relative tolerance would
# run to maxiter; skipping it changes C by a relative O(SKIP_RMS).
SKIP_RMS = 1e-10


def effective_stiffness(cell: PeriodicCell, E_field=None, tol: float = 1e-8, maxiter: int = 20000, device="cuda",
                        return_fields: bool = False):
    """(C, infos): C the 6x6 float64 numpy effective stiffness (column j = <sigma> under unit Voigt strain j, Voigt order
    11, 22, 33, 23, 13, 12, engineering shears), returned as computed (not symmetrised: its asymmetry is a measure of the
    solve error); infos one SolveInfo per load case (flag, relres, iters; a skipped case has flag 0 and 0 iterations).
    E_field: one Young's modulus per element, shape (ne[2], ne[1], ne[0]) (hexmesh.inclusion_field); None = cell.E.
    One operator, one Jacobi vector and one SubdomainOperator serve all 6 solves, each from x0 = 0 to `tol` relative
    residual.  return_fields=True adds a third item, {"u": the 6 fluctuations (device tensors), "strain": the 6x6 matrix of
    average strains (column j ~ unit vector j, tensor shears)}."""
    op = generate_periodic_operator(cell, device=device, E_field=E_field)
    sop = SubdomainOperator(op)
    minv = sop.jacobi()
    F = PeriodicFields(cell, device=device, E_field=E_field)
    ck_max = float(op._ck.max().item()) if op._ck is not None else cell.E * cell.h   # the operator's own Ck copy
    ke_max = float(np.abs(hex_element_stiffness(1.0, cell.nu)).max())
    C = np.empty((6, 6))
    S = np.empty((6, 6))
    infos, us = [], []
    for j in range(6):
        strain = np.zeros(6)
        strain[j] = 1.0
        b = op.load(strain)
        scale = ck_max * ke_max * cell.h * float(np.abs(strain).max())
        if float(torch.linalg.vector_norm(b).item()) <= SKIP_RMS * scale * np.sqrt(cell.n):
            x, info = torch.zeros_like(b), SolveInfo(flag=0, iters=0, relres=0.0)
        else:
            x, info = sop.solve(b, minv, tol, maxiter)
        S[:, j], C[:, j] = F.average(x, strain)
        infos.append(info)
        if return_fields:
            us.append(x)
    if return_fields:
        return C, infos, {"u": us, "strain": S}
    return C, infos
