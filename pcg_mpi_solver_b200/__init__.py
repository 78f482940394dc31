"""pcg_mpi_solver_b200 - H100-native PCG hot path of ankitskr/PCG-MPI-solver.

Public surface (mirrors the reference's solver/partition API for this path, SURVEY.md 8(b)):
    solve(A, b, M, tol, maxiter)    Jacobi-PCG with MATLAB-pcg semantics (pcg_solver.py:356-598)
    partition_mesh(model, nparts)   METIS dual partition + subdomain builder
                                    (run_metis.py + partition_mesh.py)
    CsrMatrix, SubdomainOperator, Communicator
    HexFields(block, ...)           strains, stresses, principal values and their nodal averages of a hex box
                                    (updateElemStrain / getNodalPS, pcg_solver.py:601-618, 730-814)
    effective_stiffness(cell, ...)  the 6x6 effective elastic tensor of a periodic voxel cell (homogenize.py)
Everything numerical runs in csrc/libpcgb200.so (hand-written sm_90a CUDA, C ABI in include/pcgb200.h).
"""
from .solver import Communicator, SolveInfo, SubdomainOperator, solve  # noqa: F401
from .csr import CsrMatrix  # noqa: F401
from .fields import HexFields  # noqa: F401
from .homogenize import effective_stiffness  # noqa: F401


def partition_mesh(*args, **kwargs):
    from .partition import partition_mesh as _pm
    return _pm(*args, **kwargs)


__all__ = ["solve", "partition_mesh", "CsrMatrix", "SubdomainOperator", "Communicator", "SolveInfo", "HexFields", "effective_stiffness"]
