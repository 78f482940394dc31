"""Element partitions of small hex models, and the host side of the METIS-partitioned multi-rank tests.

The box cuts of `hexmesh.partition_blocks` only give aligned sub-boxes: whole shared faces, edges and corners, interface
rows on the faces of each local numbering, at most 26 neighbours. The general pipeline, `partition_mesh(model, nparts,
elepart)` -> `build_subdomains` -> `SubdomainData.to_operator`, builds its interface lists from whatever element split it
is given. The cases here are element splits of `hexmesh.hex_mdf_model(ng)` that reach what the box cuts cannot:

- `metis2`, `metis3`, `metis4`: METIS 2-, 3- and 4-way (`run_metis`, ncommon 1, deterministic for a given METIS build) on
  uneven boxes, so that interface rows are scattered through each part's local numbering;
- `random8`: every element of a 6x5x4 box drawn into one of 8 parts. The parts are disconnected, every part neighbours
  every other, and some node sits in all 8 parts, so its dofs appear in 7 lists of every part;
- `hand`: octants of a 9x7x5 box around the node (4, 3, 2). Part 0 (low octant) and part 1 (high x, high y, low z) touch
  along one edge only; part 0 and part 2 (high octant) touch at one node only, a 3-dof list. Part 3 is a single element
  in a corner on the clamped face x = 0, so 3 of the 7 nodes it shares lose their dofs. Part 4 is the rest.

Why no free-dof list is ever empty on a hex model: the clamped dofs are those of the nodes at x = 0, and every element
that holds a node at x = 0 spans x in [0, 1] and holds the node at x = 1 with the same (y, z). Two parts that share a
node at x = 0 therefore share a node at x = 1, which is free. A list loses all its entries only when every shared node
is clamped, which needs meshes like concrete's, where clamped nodes are not a whole face of hexahedra.

Helpers for the workers: the probe vector as a function of the global dof id, gathering a rank's vector onto the global
dofs, and the exact exchange (`oracle.ref_pcg.exchange_add`: y first, then each neighbour's copy in list order) over
shells that carry each part's neighbour table and free-dof lists."""
from __future__ import annotations

import os
from types import SimpleNamespace

import numpy as np

from oracle import ref_pcg as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CONCRETE_ZIP = os.path.join(ROOT, "oracle", "_ref", "concrete.zip")

# name -> (box in elements, number of parts)
CASES = {"metis2": ((12, 10, 7), 2), "metis3": ((12, 10, 7), 3), "metis4": ((9, 7, 5), 4),
         "random8": ((6, 5, 4), 8), "hand": ((9, 7, 5), 5)}
RANDOM_SEED = 2


def element_grid(ng):
    """Element coordinates (ex, ey, ez) in hex_mdf_model's element order (x fastest)."""
    nx, ny, nz = ng
    ez, ey, ex = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return ex.ravel(), ey.ravel(), ez.ravel()


def elepart(name, model=None):
    """The element -> part vector of a case (int64)."""
    ng, nparts = CASES[name]
    if name.startswith("metis"):
        from pcg_mpi_solver_b200.metis import run_metis
        model = model if model is not None else hex_model(name)
        return run_metis(model.node_flat, model.node_offset, nparts)
    if name == "random8":
        return np.random.default_rng(RANDOM_SEED).integers(0, nparts, ng[0] * ng[1] * ng[2]).astype(np.int64)
    if name == "hand":
        ex, ey, ez = element_grid(ng)
        hi_x, hi_y, hi_z = ex >= 4, ey >= 3, ez >= 2
        ep = np.full(ex.size, 4, dtype=np.int64)
        ep[~hi_x & ~hi_y & ~hi_z] = 0
        ep[hi_x & hi_y & ~hi_z] = 1
        ep[hi_x & hi_y & hi_z] = 2
        ep[(ex == 0) & (ey == ng[1] - 1) & (ez == ng[2] - 1)] = 3
        return ep
    raise KeyError(name)


def hex_model(name):
    from pcg_mpi_solver_b200.hexmesh import hex_mdf_model
    return hex_mdf_model(CASES[name][0])


def subdomains(name, assemble=False):
    """(model, elepart, subdomains) of a hex case."""
    from pcg_mpi_solver_b200.partition import build_subdomains
    model = hex_model(name)
    ep = elepart(name, model)
    return model, ep, build_subdomains(model, ep, CASES[name][1], assemble=assemble)


def probe(gdof, concrete=False):
    """A globally consistent vector: a function of the global dof id only. On concrete it is the vector of the reference's
    own calcMPFint probe (tests/golden/concrete_probe.npz)."""
    g = np.asarray(gdof, dtype=np.float64)
    if concrete:
        return np.sin(0.001 * g) + 0.25 * np.cos(0.37 * g)
    return np.sin(0.37 * g) + 0.01 * (np.asarray(gdof) % 7)


def gather(n_dof, gdofs, vecs):
    """Every rank's vector written onto the global dofs (a later rank's copy overwrites an earlier one's)."""
    out = np.zeros(n_dof)
    for g, v in zip(gdofs, vecs):
        out[g] = v
    return out


def shells(tables):
    """Parts for oracle.ref_pcg.exchange_add from (id, nbr, free-dof lists) tables."""
    return [SimpleNamespace(id=int(i), nbr=list(nbr), ovrlp=[np.asarray(v, dtype=np.int64) for v in lists])
            for i, nbr, lists in tables]


def exchange(tables, ys):
    """The exact interface sum of every rank's vector: y first, then each neighbour's copy in list order."""
    return R.exchange_add(shells(tables), [np.array(y, dtype=np.float64) for y in ys])


def abs_product(sub, v):
    """(|K_i[Eff,Eff]| |v|) of one part on its free dofs, from the pattern groups on the host: the scale of each entry of
    the local product, before the interface sum."""
    xf = np.zeros(sub.ndof)
    xf[sub.loc_dof_eff] = np.abs(v)
    y = np.zeros(sub.ndof)
    for g in sub.groups:
        u = np.abs(g.ke) @ (np.abs(g.ck) * xf[g.loc_dof])
        y += np.bincount(g.loc_dof.ravel(), weights=u.ravel(), minlength=sub.ndof)
    return y[sub.loc_dof_eff]


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(a.view(np.uint64) == b.view(np.uint64)))


def holders(subs, n_dof):
    """For every global dof: how many parts hold its node, and the lowest id among them (n_parts if none)."""
    count = np.zeros(n_dof, dtype=np.int64)
    low = np.full(n_dof, len(subs), dtype=np.int64)
    for s in subs:
        count[s.dof_vector] += 1
        low[s.dof_vector] = np.minimum(low[s.dof_vector], s.id)
    return count, low


def table_failures(subs):
    """What the subdomain builder must guarantee of its interface tables, as a list of failures (empty = all hold):
    symmetric neighbour tables; positional pairs (entry t of p's list for q and of q's list for p are the same global dof),
    on the full and on the free lists; 0/1 weights with the owner the lowest id, summing to n_global_eff; and each dof's
    multiplicity (1 + the lists it is in) equal to the number of parts that hold its node."""
    fails = []
    byid = {s.id: s for s in subs}
    n_dof = subs[0].n_global
    count, low = holders(subs, n_dof)
    for p in subs:
        if sorted(p.nbr) != p.nbr or len(set(p.nbr)) != len(p.nbr):
            fails.append(f"part {p.id}: neighbours not ascending and distinct: {p.nbr}")
        for j, q_id in enumerate(p.nbr):
            q = byid[q_id]
            if p.id not in q.nbr:
                fails.append(f"part {p.id} lists {q_id}, which does not list it")
                continue
            k = q.nbr.index(p.id)
            mine, theirs = p.dof_vector[p.ovrlp_full[j]], q.dof_vector[q.ovrlp_full[k]]
            if not np.array_equal(mine, theirs):
                fails.append(f"parts {p.id}/{q_id}: full lists do not pair up")
            mine, theirs = p.dof_eff_global[p.ovrlp[j]], q.dof_eff_global[q.ovrlp[k]]
            if not np.array_equal(mine, theirs):
                fails.append(f"parts {p.id}/{q_id}: free lists do not pair up")
            if len(np.unique(p.ovrlp[j])) != len(p.ovrlp[j]):
                fails.append(f"parts {p.id}/{q_id}: a free list repeats an index")
        mult = np.ones(p.ndof, dtype=np.int64)
        for lst in p.ovrlp_full:
            mult[lst] += 1
        if not np.array_equal(mult, count[p.dof_vector]):
            fails.append(f"part {p.id}: multiplicity differs from the number of parts holding the node")
        w = p.weights_full
        if not np.all((w == 0.0) | (w == 1.0)):
            fails.append(f"part {p.id}: weights are not 0/1")
        if not np.array_equal(w == 1.0, low[p.dof_vector] == p.id):
            fails.append(f"part {p.id}: weight 1 is not exactly on the dofs it is the lowest holder of")
    wsum = sum(float(s.weights.sum()) for s in subs)
    if wsum != subs[0].n_global_eff:
        fails.append(f"free weights sum to {wsum}, not n_global_eff = {subs[0].n_global_eff}")
    return fails


def features(subs):
    """What a partition reaches: the largest multiplicity, the shortest free list, the smallest part in elements,
    whether every part neighbours every other, how many free lists are empty, and the largest neighbour count."""
    count, _ = holders(subs, subs[0].n_global)
    lens = [len(v) for s in subs for v in s.ovrlp]
    return {"max_multiplicity": int(count.max()), "min_free_list": int(min(lens)) if lens else 0,
            "min_elements": int(min(sum(g.ck.size for g in s.groups) for s in subs)),
            "all_neighbours": all(len(s.nbr) == len(subs) - 1 for s in subs),
            "empty_free_lists": sum(1 for n in lens if n == 0), "max_neighbours": max(len(s.nbr) for s in subs)}


def connected_components(ng, ep, part):
    """Face-connected components of one part's elements (a part split into several pieces has more than one)."""
    nx, ny, nz = ng
    cells = set(np.nonzero(np.asarray(ep) == part)[0].tolist())
    seen, comps = set(), 0
    for c in cells:
        if c in seen:
            continue
        comps += 1
        stack = [c]
        seen.add(c)
        while stack:
            e = stack.pop()
            x, y, z = e % nx, (e // nx) % ny, e // (nx * ny)
            for dx, dy, dz in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)):
                a, b, d = x + dx, y + dy, z + dz
                if 0 <= a < nx and 0 <= b < ny and 0 <= d < nz:
                    f = (d * ny + b) * nx + a
                    if f in cells and f not in seen:
                        seen.add(f)
                        stack.append(f)
    return comps
