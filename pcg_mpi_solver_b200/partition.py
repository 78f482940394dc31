"""partition_mesh(model, nparts): METIS element partition + subdomain builder, as a function.

Replaces the two file-based stages of the reference that manufacture the solver's input
(SURVEY.md 8(b)):  run_metis.py (element -> part ids) and partition_mesh.py (per-part data), and adds
what the CSR hot path needs: the sub-assembled matrix A_i = K_i[Eff,Eff] of every part.

The quantities are the reference's, computed with vectorised numpy instead of per-element Python loops
(the reference's own "TODO: Perform the element loop in Cython", partition_mesh.py:244):
    DofVector / NodeIdVector      unique global dofs / nodes of the part            partition_mesh.py:257-262
    LocDofVector (per element)    positions in DofVector                              :267-286 (getIndices :63-72)
    LocDofEff                     free dofs, ascending                                :350-351
    type groups                   elements grouped by pattern id, ascending           :443-491
    NbrMPIdVector                 parts sharing >= 1 node, ascending part id          :724-741, 817-830
    OvrlpLocalDofVecList          3*localnode + {0,1,2} over the shared nodes in ascending global id  :822-827
    DofWeightVector               1, but 0 on dofs shared with a LOWER part id        :867-887
    Fext / b                      F*delta - K (Ud*delta), interface-summed            pcg_solver.py:226-238
and, new here:
    A                             K_i[Eff,Eff] = sum_e P_e^T (Ck_e S_e Ke_type(e) S_e) P_e   (SURVEY Fact 1)
    ovrlp (Eff numbering)         the overlap lists with clamped dofs dropped and renumbered on the free dofs
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import scipy.sparse as sp

from .metis import run_metis
from .model import MdfModel, load_mdf


def _ranges(offsets: np.ndarray):
    """Flat indices of the concatenated inclusive ranges offsets[:,0]..offsets[:,1] and their lengths."""
    starts = offsets[:, 0].astype(np.int64)
    lens = (offsets[:, 1] - offsets[:, 0] + 1).astype(np.int64)
    cum = np.concatenate([[0], np.cumsum(lens)])
    idx = np.repeat(starts - cum[:-1], lens) + np.arange(cum[-1], dtype=np.int64)
    return idx, lens, cum


@dataclass
class TypeGroup:
    """Elements of one pattern type inside a part (MP_TypeGroup, partition_mesh.py:470-491)."""
    type_id: int
    loc_dof: np.ndarray   # ElemList_LocDofVector  (nd, N_e) int64, local (all-dof) numbering
    sign: np.ndarray      # ElemList_SignVector    (nd, N_e) bool
    ck: np.ndarray        # ElemList_Ck            (N_e,)
    ke: np.ndarray        # ElemStiffMat           (nd, nd)
    elem_ids: np.ndarray  # global element ids


@dataclass
class SubdomainData:
    """What the hot path needs of one mesh part (the RefMeshPart keys of SURVEY.md 8(b))."""
    id: int
    n_parts: int
    dof_vector: np.ndarray      # DofVector    global dof ids of the local dofs (ascending)
    node_ids: np.ndarray        # NodeIdVector
    loc_dof_eff: np.ndarray     # LocDofEff    local indices of the free dofs
    groups: list                # StrucDataList
    nbr: list                   # NbrMPIdVector
    ovrlp_full: list            # OvrlpLocalDofVecList (local all-dof numbering, like the reference)
    ovrlp: list                 # same lists in the free-dof numbering, clamped dofs dropped
    weights_full: np.ndarray    # DofWeightVector
    F: np.ndarray               # RefLoadVector
    Ud: np.ndarray
    n_global_eff: int           # GlobNDofEff
    n_global: int               # GlobNDof
    A: sp.csr_matrix | None = None     # K_i[Eff,Eff]
    b: np.ndarray | None = None        # Fext[LocDofEff]
    udi: np.ndarray | None = None      # Ud * delta
    extra: dict = field(default_factory=dict)

    @property
    def ndof(self) -> int:
        return self.dof_vector.size

    @property
    def n(self) -> int:
        return self.loc_dof_eff.size

    @property
    def weights(self) -> np.ndarray:
        """DofWeightVector_Eff (pcg_solver.py:997)."""
        return self.weights_full[self.loc_dof_eff]

    @property
    def dof_eff_global(self) -> np.ndarray:
        return self.dof_vector[self.loc_dof_eff]

    def to_refmeshpart(self) -> dict:
        """A dict with the reference's key names (partition_mesh.py:1310-1317) for the keys the hot path
        reads - what oracle.ref_pcg.EbePart and a reference-side binding consume."""
        groups = [{"ElemTypeId": g.type_id, "ElemList_LocDofVector": g.loc_dof, "ElemList_LocDofVector_Flat": g.loc_dof.flatten(),
                   "ElemList_SignVector": g.sign, "ElemList_Ck": g.ck, "ElemStiffMat": g.ke, "ElemDiagStiffMat": np.diag(g.ke).copy(),
                   "ElemList_LocNodeIdVector": g.loc_dof[0::3, :] // 3,      # local node ids (3 dofs per node, partition_mesh.py:454)
                   "ElemList_LocElemId": None, "N_Elem": g.ck.size} for g in self.groups]
        flat = np.concatenate([g["ElemList_LocDofVector_Flat"] for g in groups]) if groups else np.zeros(0, dtype=np.int64)
        return {"Id": self.id, "NDOF": self.ndof, "NNode": self.node_ids.size, "DofVector": self.dof_vector, "NodeIdVector": self.node_ids,
                "LocDofEff": self.loc_dof_eff, "SubDomainData": {"StrucDataList": groups, "MixedDataList": {}},
                "Flat_ElemLocDof": flat, "NCountDof": int(flat.size), "NbrMPIdVector": list(self.nbr),
                "OvrlpLocalDofVecList": list(self.ovrlp_full), "DofWeightVector": self.weights_full, "RefLoadVector": self.F, "Ud": self.Ud,
                "GlobData": {"GlobNDofEff": self.n_global_eff, "GlobNDof": self.n_global}}

    def to_operator(self, comm=None, device="cuda", kind: str = "csr"):
        """Upload A and build the halo plan: the `A` argument of solve() for this rank.
        kind="ebe" selects the opt-in matrix-free operator (ebe.py) instead of the assembled CSR matrix, kind="ebe_ordered"
        its bit-reproducible variant with a fixed summation order."""
        from .csr import CsrMatrix
        from .solver import SubdomainOperator
        if kind == "ebe":
            from .ebe import EbeMatrix
            M = EbeMatrix(self.groups, self.loc_dof_eff, self.ndof, device=device)
        elif kind == "ebe_ordered":
            from .ebe import EbeMatrixOrdered
            M = EbeMatrixOrdered(self.groups, self.loc_dof_eff, self.ndof, device=device)
        elif self.A is not None:
            M = CsrMatrix.from_scipy(self.A, device=device)
        else:  # assemble on the device straight from the pattern groups
            rowptr, col, val = assemble_csr_device(self, device)
            M = CsrMatrix(rowptr, col, val, (self.n, self.n))
        return SubdomainOperator(M, comm, self.nbr, self.ovrlp, self.weights, n_global=self.n_global_eff)


def _assemble(groups, ndof: int) -> sp.csr_matrix:
    """K_i on all local dofs: sum_e P_e^T (Ck_e S_e Ke S_e) P_e, duplicates summed (COO -> CSR)."""
    rows, cols, vals = [], [], []
    for g in groups:
        nd, ne = g.loc_dof.shape
        s = np.where(g.sign, -1.0, 1.0)                                    # pcg_solver.py:278,280
        v = (s[:, None, :] * s[None, :, :]) * g.ke[:, :, None] * g.ck[None, None, :]   # (nd, nd, ne)
        rows.append(np.broadcast_to(g.loc_dof[:, None, :], v.shape).ravel().astype(np.int32))
        cols.append(np.broadcast_to(g.loc_dof[None, :, :], v.shape).ravel().astype(np.int32))
        vals.append(v.ravel())
    if not rows:
        return sp.csr_matrix((ndof, ndof))
    K = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(ndof, ndof)).tocsr()
    K.sum_duplicates()
    K.sort_indices()
    return K


def build_subdomains(model: MdfModel, elepart: np.ndarray, nparts: int, assemble=True, delta: float = 1.0):
    """The partition_mesh.py stage for all parts (single process; the reference's MPGSize = N path)."""
    elepart = np.asarray(elepart)
    subs = []
    eff_mask = np.zeros(model.n_dof, dtype=bool)
    eff_mask[model.dof_eff] = True
    for pid in range(nparts):
        elems = np.nonzero(elepart == pid)[0]                              # partition_mesh.py:120
        didx, dlens, dcum = _ranges(model.dof_offset[elems])
        cum_dofs = model.dof_flat[didx].astype(np.int64)
        nidx, _, _ = _ranges(model.node_offset[elems])
        cum_nodes = model.node_flat[nidx].astype(np.int64)
        sidx, _, _ = _ranges(model.sign_offset[elems])
        cum_sign = model.sign_flat[sidx]
        dof_vector = np.unique(cum_dofs)                                   # :261-262
        node_ids = np.unique(cum_nodes)                                    # :257-258
        loc = np.searchsorted(dof_vector, cum_dofs)                        # getIndices on a sorted unique vector
        loc_dof_eff = np.nonzero(eff_mask[dof_vector])[0]                  # :350-351
        groups = []
        etype = model.etype[elems]
        for t in np.unique(etype):                                         # :443-451
            sel = np.nonzero(etype == t)[0]
            nd = int(dlens[sel[0]])
            assert np.all(dlens[sel] == nd), "elements of one pattern type must have the same dof count"
            take = (dcum[sel][None, :] + np.arange(nd)[:, None])           # (nd, N_e) positions in the part's flat list
            groups.append(TypeGroup(int(t), loc[take], cum_sign[take], model.ck[elems[sel]].astype(float),
                                    np.array(model.ke[int(t)], dtype=float), elems[sel]))
        subs.append(SubdomainData(pid, nparts, dof_vector, node_ids, loc_dof_eff, groups, [], [], [], np.ones(dof_vector.size),
                                  model.F[dof_vector].astype(float), model.Ud[dof_vector].astype(float),
                                  model.n_dof_eff, model.n_dof))
    # ---- neighbours, overlap lists, ownership weights (config_Neighbours, :805-887)
    dirs = np.array([[0], [1], [2]])
    for p in subs:
        is_eff = np.zeros(p.ndof, dtype=bool)
        is_eff[p.loc_dof_eff] = True
        eff_pos = np.cumsum(is_eff) - 1
        for q in subs:                                                     # ascending part id, like range(N_TotalMeshPart)
            if q is p:
                continue
            common = np.intersect1d(p.node_ids, q.node_ids, assume_unique=True)  # :822
            if common.size == 0:
                continue
            lnode = np.searchsorted(p.node_ids, common)                    # :825
            dofs = (3 * lnode + dirs).T.ravel()                            # :826
            p.nbr.append(q.id)
            p.ovrlp_full.append(dofs)
            p.ovrlp.append(eff_pos[dofs[is_eff[dofs]]].astype(np.int64))
            if p.id > q.id:                                                # :885-887
                p.weights_full[dofs] = 0.0
    # ---- right-hand side (updateBC, pcg_solver.py:226-238): Fext = F*delta - K (Ud*delta), interface-summed
    fdi_glob = np.zeros(model.n_dof)
    any_ud = bool(np.any(model.Ud != 0))
    for p in subs:
        p.udi = p.Ud * delta
        if any_ud:
            fdi_glob[p.dof_vector] += _ebe_matvec(p.groups, p.udi, p.ndof)  # the sum over parts IS the interface sum
    for p in subs:
        fext = p.F * delta - fdi_glob[p.dof_vector]
        p.b = fext[p.loc_dof_eff]
    # ---- operator
    if assemble in (True, "host"):
        for p in subs:
            K = _assemble(p.groups, p.ndof)
            p.A = K[p.loc_dof_eff][:, p.loc_dof_eff].tocsr()
            p.A.sort_indices()
    return subs


def _ebe_matvec(groups, x_full, ndof):
    """y = K_i x on all local dofs, element by element (only used once, for the Dirichlet term of the RHS)."""
    y = np.zeros(ndof)
    for g in groups:
        s = np.where(g.sign, -1.0, 1.0)
        v = s * (g.ke @ (g.ck * (s * x_full[g.loc_dof])))
        y += np.bincount(g.loc_dof.ravel(), weights=v.ravel(), minlength=ndof)
    return y


def assemble_csr_device(sub: SubdomainData, device="cuda"):
    """K_i[Eff,Eff] assembled ON THE DEVICE from the pattern groups by the library's own kernels (csrc/assemble.cuh through
    pcgb_assemble_symbolic / pcgb_assemble_numeric): incidence lists per dof, per-row sorted distinct columns, per-row
    accumulation in a fixed (group, element) order - no atomics in the arithmetic, bit-reproducible, and no nd^2 * N_e
    COO expansion (a 128^3 METIS part would need ~50 GB that way).  torch only allocates the output arrays.
    Returns (rowptr int32/int64, col int32, val float64) CUDA tensors."""
    import ctypes

    import torch

    from . import _lib
    lib = _lib.load()
    n = sub.n
    eff_map = np.full(sub.ndof, -1, dtype=np.int32)
    eff_map[sub.loc_dof_eff] = np.arange(n, dtype=np.int32)
    keep = []
    cgroups = (_lib.EbeGroup * max(len(sub.groups), 1))()
    for k, g in enumerate(sub.groups):
        nd, ne = g.loc_dof.shape
        d_idx = torch.from_numpy(np.ascontiguousarray(eff_map[g.loc_dof])).to(device)         # (nd, ne) int32, -1 = clamped
        d_ck = torch.from_numpy(np.ascontiguousarray(g.ck, dtype=np.float64)).to(device)
        d_sign = torch.from_numpy(np.ascontiguousarray(g.sign.astype(np.uint8))).to(device) if g.sign.any() else None
        ke = np.ascontiguousarray(g.ke, dtype=np.float64)
        keep += [d_idx, d_ck, d_sign, ke]
        cg = cgroups[k]
        cg.nd, cg.ne = nd, ne
        cg.d_idx, cg.d_ck = d_idx.data_ptr(), d_ck.data_ptr()
        cg.d_sign = d_sign.data_ptr() if d_sign is not None else None
        cg.ke_host = ke.ctypes.data
    with torch.cuda.device(device):
        rowptr = torch.empty(n + 1, dtype=torch.int64, device=device)
        nnz = ctypes.c_int64(0)
        h = ctypes.c_void_p()
        _lib.check(lib.pcgb_assemble_symbolic(n, len(sub.groups), cgroups, _lib.ptr(rowptr), ctypes.byref(nnz), _lib.stream_ptr(), ctypes.byref(h)),
                   "pcgb_assemble_symbolic")
        try:
            col = torch.empty(nnz.value, dtype=torch.int32, device=device)
            val = torch.empty(nnz.value, dtype=torch.float64, device=device)
            _lib.check(lib.pcgb_assemble_numeric(h, _lib.ptr(rowptr), _lib.ptr(col), _lib.ptr(val), _lib.stream_ptr()), "pcgb_assemble_numeric")
            torch.cuda.current_stream().synchronize()
        finally:
            lib.pcgb_assemble_destroy(h)
    del keep
    if nnz.value < 2**31:
        rowptr = rowptr.to(torch.int32)
    return rowptr, col, val


def partition_mesh(model, nparts: int, elepart: np.ndarray | None = None, assemble=True, ncommon: int = 1):
    """run_metis.py + partition_mesh.py as one call.

    model: MdfModel, or a path to `<model>.zip` / an unpacked MDF directory.
    assemble: True/"host" = scipy COO->CSR on the host (small models, CPU tests); False/"device" = leave A
    unset, SubdomainData.to_operator() then assembles on the GPU (88 s -> ~1 s for data/concrete.zip).
    Returns the list of SubdomainData, one per part (part i is solved by rank / GPU i, pcg_solver.py:91).
    """
    if not isinstance(model, MdfModel):
        model = load_mdf(model)
    if elepart is None:
        elepart = run_metis(model.node_flat, model.node_offset, nparts, ncommon=ncommon)
    return build_subdomains(model, elepart, nparts, assemble=assemble)
