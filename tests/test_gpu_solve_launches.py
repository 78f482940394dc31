"""Kernel launches of one PCG iteration on the CSR, atomic EBE, ordered EBE and multigrid-on-CSR paths, with the trace off and
on and the CUDA graph off and on.  An iteration's count is launches(2m) - launches(m) over m fixed iterations, so the set-up
and the finalisation cancel; the expected count is derived from what each operator's plan exposes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = 4
NE = (8, 8, 8)


def _block(ne=NE, level=0):
    from pcg_mpi_solver_b200.hexmesh import HexBlock
    ne_l = tuple(v >> level for v in ne)
    return HexBlock(ne_l, (0, 0, 0), ne_l, h=2.0 ** level / ne[0])


def _spmv_launches(A, with_dot):
    """The SpMV kernel, the fixup of rows split across tiles, and (with the p.q partials) their stage reduction above 8192."""
    info = A.plan_info()
    partials = info["resident_ctas"] if info["staged"] == 2 else info["ntiles"]
    return 1 + (info["split_rows"] > 0) + (with_dot and partials > 8192)


def _ebe_groups(blk):
    """The box's elements as three pattern groups: the first half as 24-dof patterns, the second half as 25-dof patterns (Ke
    padded with a zero row and column on a clamped dof, so K is unchanged) and an empty 24-dof group."""
    from pcg_mpi_solver_b200.hexmesh import hex_type_group
    from pcg_mpi_solver_b200.partition import TypeGroup
    grp, eff, ndof = hex_type_group(blk)
    clamped = 0                                  # dof x of node (0, 0, 0), on the clamped face x = 0
    assert clamped not in set(eff.tolist())
    ne = grp.ck.size
    h = ne // 2
    ke25 = np.zeros((25, 25))
    ke25[:24, :24] = grp.ke
    groups = [TypeGroup(0, grp.loc_dof[:, :h], grp.sign[:, :h], grp.ck[:h], grp.ke, None),
              TypeGroup(1, np.vstack([grp.loc_dof[:, h:], np.full((1, ne - h), clamped)]), np.zeros((25, ne - h), dtype=bool),
                        grp.ck[h:], ke25, None),
              TypeGroup(2, np.zeros((24, 0), dtype=np.int64), np.zeros((24, 0), dtype=bool), np.zeros(0), grp.ke, None)]
    return groups, eff, ndof


def _ebe_launches(groups, ordered):
    """One launch per 24-dof group with elements (each finds a constant-memory slot: all share the hex Ke), one warp launch
    when another group has elements, and the ordered operator's per-dof sum."""
    t24 = sum(1 for g in groups if g.loc_dof.shape[0] == 24 and g.ck.size > 0)
    warp = any(g.loc_dof.shape[0] != 24 and g.ck.size > 0 for g in groups)
    return t24 + warp + ordered


def _setup(cuda, path):
    """(operator, M for solve, expected launches of one iteration without the trace)"""
    import gc
    from pcg_mpi_solver_b200.ebe import EbeMatrix, EbeMatrixOrdered
    from pcg_mpi_solver_b200.hexmesh import generate_matrix
    from pcg_mpi_solver_b200.multigrid import HexMultigrid
    from pcg_mpi_solver_b200.solver import SubdomainOperator
    gc.collect()                                 # operators of earlier tests give their constant-memory slots back
    blk = _block()
    # every iteration: p-update, p.q reduction, fused update, norms reduction
    fixed = 4
    if path in ("csr", "mg_csr"):
        A = generate_matrix(blk, device=cuda)
        op = SubdomainOperator(A)
        if path == "csr":
            return op, op.jacobi(), fixed + _spmv_launches(A, True)
        mg = HexMultigrid(op, blk)
        info = mg.info()
        # V-cycle: per smoothed level a pre-smoother (first step + degree x (product + step)), restriction, prolongation and
        # a post-smoother (degree x (product + step)); the coarse solve; then k_mg_rz
        vcycle = 1
        for l in range(info["levels"] - 1):
            op_l = _spmv_launches(A if l == 0 else generate_matrix(_block(level=l), device=cuda), False)
            vcycle += 3 + 2 * mg.degree * (op_l + 1)
        return op, mg, fixed + _spmv_launches(A, True) + vcycle + 1
    groups, eff, ndof = _ebe_groups(blk)
    ordered = path == "ebe_ordered"
    E = (EbeMatrixOrdered if ordered else EbeMatrix)(groups, eff, ndof, device=cuda)
    op = SubdomainOperator(E)
    return op, op.jacobi(), fixed + _ebe_launches(groups, ordered) + 1     # + the p.q dot of the matrix-free product


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("path", ["csr", "ebe", "ebe_ordered", "mg_csr"])
def test_launches_per_iteration(cuda, path, trace, use_graph):
    from pcg_mpi_solver_b200.hexmesh import load_vector
    op, Mp, per_iter = _setup(cuda, path)
    b = load_vector(_block(), device=cuda)
    launches = []
    for maxiter in (M, 2 * M):
        _, info = op.solve(b, Mp, 1e-12, maxiter, fixed_iters=True, use_graph=use_graph, check_every=M, trace=trace)
        assert info.loop_iters == maxiter and info.flag == 1, (info.loop_iters, info.flag)
        launches.append(info.launches)
    assert (launches[1] - launches[0]) == M * (per_iter + trace), (launches, per_iter)
