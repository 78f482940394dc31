"""Synthetic interface plans for the halo exchange-add (pcgb_halo_*, csrc/peer.cuh, csrc/comm.cuh) and its host reference.

A plan for `world` ranks holds, per rank r, the local length n[r], the neighbour ranks nbr[r] in r's list order and one
list of local indices per neighbour.  Lists are positional pairs: entry t of r's list for s and entry t of s's list for r
name the same dof.  Indices are random and distinct within a list; a dof may sit in several lists of one rank (its
multiplicity).  Every rank with two or more neighbours lists them in a non-ascending order (reversed or rotated), so a
kernel that adds in rank order instead of list order is told apart.

The cases reach the edges of the peer kernels: k_halo_pack_peer stores 256 * 4 = 1024 entries per CTA (m = 1023, 1024,
1025, 4097 and 3 * 2^16 + 17), k_halo_unpack_peer adds 256 distinct dofs per CTA (ndof = 255, 256, 257).  Needs no GPU.
"""
import numpy as np

PACK_PER_CTA = 256 * 4
UNPACK_PER_CTA = 256
BIG_M = 3 * 2 ** 16 + 17


def make_plan(world, pairs, pools=None, hubs=(), seed=0, spare=37):
    """pairs: {(r, s): count} with r < s; count 0 keeps the neighbour with an empty list.  pools: {rank: P} draws that
    rank's lists from P dofs (lists cycle through them, so ndof = P when its lists hold at least P entries in all);
    otherwise every entry of the rank is its own dof.  hubs: ranks that put one dof into every non-empty list."""
    rng = np.random.default_rng(seed)
    pools = pools or {}
    cnt = {}
    for (r, s), c in pairs.items():
        assert r < s and (r, s) not in cnt
        cnt[(r, s)] = cnt[(s, r)] = int(c)
    nbr, lists, n = [], [], []
    for r in range(world):
        asc = sorted(s for s in range(world) if (r, s) in cnt)
        order = asc[::-1] if r % 2 == 0 else asc[1:] + asc[:1]   # reversed or rotated: never ascending with >= 2
        lens = [cnt[(r, s)] for s in order]
        m = sum(lens)
        hub = r in hubs
        size = pools.get(r, m - (max(0, sum(1 for c in lens if c) - 1) if hub else 0))
        n_r = size + spare
        pool = rng.permutation(rng.choice(n_r, size, replace=False)) if size else np.zeros(0, np.int64)
        out, pos = [], 0
        body = pool[1:] if hub else pool
        for c in lens:
            if c == 0:
                out.append(np.zeros(0, np.int64))
                continue
            k = c - 1 if hub else c
            assert k <= len(body), "a list longer than its pool would repeat an index"
            take = body[(pos + np.arange(k)) % len(body)] if k else np.zeros(0, np.int64)
            pos += k
            lst = np.concatenate([pool[:1], take]) if hub else take
            out.append(rng.permutation(lst).astype(np.int64))
        nbr.append(order)
        lists.append(out)
        n.append(n_r)
    return {"world": world, "n": n, "nbr": nbr, "lists": lists}


# name -> (world, pairs, pools, hubs); the worker builds every case of its world in one process group
CASES = {
    # m = 1 on both ranks
    "w2_one": (2, {(0, 1): 1}, None, ()),
    # m = 1025 (one entry past the first pack CTA)
    "w2_1025": (2, {(0, 1): 1025}, None, ()),
    # m = 1023, 1024, 1025 on ranks 0, 1, 2: a + b, a + c, b + c; every dof of rank 0 shared with both others once
    "w3_pack_edge": (3, {(0, 1): 511, (0, 2): 512, (1, 2): 513}, None, (0, 1, 2)),
    # ndof = 255, 256, 257 distinct dofs on ranks 0, 1, 2 (the unpack CTA edge), many dofs in both lists
    "w3_unpack_edge": (3, {(0, 1): 200, (0, 2): 200, (1, 2): 100}, {0: 255, 1: 256, 2: 257}, ()),
    # rank 2 has the larger m (200 against 160); a pack that used its own m as the parity stride would still store
    # inside every receive buffer (the larger rank's segment comes first in the smaller ranks' lists)
    "w3_stride": (3, {(0, 1): 60, (0, 2): 100, (1, 2): 100}, None, (0, 1, 2)),
    # rank 0's only list is empty; rank 1 lists rank 0 (empty) and rank 2 (non-empty)
    "w3_empty": (3, {(0, 1): 0, (1, 2): 300}, None, ()),
    # many pack CTAs on rank 0 (m = 3 * 2^16 + 17), 196x its smallest neighbour's m, one dof in all three of its lists
    "w4_big": (4, {(0, 1): 131072, (0, 2): 64553, (0, 3): 1000, (1, 2): 5}, None, (0,)),
    # m = 4097 on rank 0, rank 3 has no neighbours at all (m = 0)
    "w4_mixed": (4, {(0, 1): 4000, (0, 2): 97, (1, 2): 1}, None, (0, 1, 2)),
    # every rank shares one dof with every other rank (multiplicity 3), moderate sizes
    "w4_hub": (4, {(0, 1): 300, (0, 2): 40, (0, 3): 7, (1, 2): 900, (1, 3): 33, (2, 3): 2}, None, (0, 1, 2, 3)),
}


def plan(name):
    world, pairs, pools, hubs = CASES[name]
    return make_plan(world, pairs, pools, hubs, seed=sum(map(ord, name)))


def cases_of(world):
    return [k for k, v in CASES.items() if v[0] == world]


def m_of(p, r):
    return int(sum(len(v) for v in p["lists"][r]))


def ndof_of(p, r):
    return int(len(np.unique(np.concatenate(p["lists"][r])))) if p["lists"][r] else 0


def max_multiplicity(p, r):
    if not p["lists"][r] or m_of(p, r) == 0:
        return 0
    return int(np.unique(np.concatenate(p["lists"][r]), return_counts=True)[1].max())


def expected(y_by_rank, p, ranks=None):
    """pcg_solver.py:303-334 restated: every dof starts from y[dof]; then, for each neighbour in the rank's list order and
    each entry in list order, that neighbour's copy is added as a Python float.  One result per rank of `ranks` (all)."""
    out = []
    for r in range(p["world"]) if ranks is None else ranks:
        y = [float(v) for v in y_by_rank[r]]
        for j, s in enumerate(p["nbr"][r]):
            mine = p["lists"][r][j]
            theirs = p["lists"][s][p["nbr"][s].index(r)]
            for t in range(len(mine)):
                y[int(mine[t])] += float(y_by_rank[s][int(theirs[t])])
        out.append(np.array(y, dtype=np.float64))
    return out


def refusal(p, r, nranks=None):
    """Why pcgb_halo_create refuses rank r's part of the plan (None = it accepts it): a neighbour that is this rank, below 0
    or at or above nranks, a neighbour listed twice, an index out of 0..n-1, or an index twice in one list."""
    nranks = p["world"] if nranks is None else nranks
    seen = set()
    for s in p["nbr"][r]:
        if s < 0 or s >= nranks or s == r:
            return "bad neighbour table"
        if s in seen:
            return "listed twice"
        seen.add(s)
    for lst in p["lists"][r]:
        lst = np.asarray(lst)
        if len(lst) and (lst.min() < 0 or lst.max() >= p["n"][r]):
            return "out of range"
        if len(np.unique(lst)) != len(lst):
            return "appears twice"
    return None


def refused_plans(seed=0):
    """Rank 0's table of a 4-rank plan, broken in each way pcgb_halo_create refuses: name -> (nbr, lists, n)."""
    base = make_plan(4, {(0, 1): 20, (0, 2): 30, (0, 3): 5, (1, 2): 3}, seed=seed)
    nbr, lists, n = list(base["nbr"][0]), [v.copy() for v in base["lists"][0]], base["n"][0]
    out = {}
    out["duplicate_neighbour"] = (nbr + [nbr[0]], lists + [lists[0][:3].copy()], n)
    dup = [v.copy() for v in lists]
    dup[1][4] = dup[1][0]
    out["duplicate_index"] = (nbr, dup, n)
    out["neighbour_self"] = ([0] + nbr[1:], lists, n)
    out["neighbour_negative"] = ([-1] + nbr[1:], lists, n)
    out["neighbour_nranks"] = ([4] + nbr[1:], lists, n)
    hi = [v.copy() for v in lists]
    hi[2][1] = n
    out["index_out_of_range"] = (nbr, hi, n)
    lo = [v.copy() for v in lists]
    lo[0][0] = -1
    out["index_negative"] = (nbr, lo, n)
    return out
