"""Element colouring for a deterministic, atomics-free scatter of the matrix-free operator (SURVEY 8(f1) follow-up).

Two elements get the same colour only if they share no node, so that `y[dof] += v` needs no atomic inside one
colour and the summation order over the colours is fixed (bit-reproducible EBE operator, the counterpart of the
reference's np.bincount at pcg_solver.py:300).  Host-side set-up code (numpy, vectorised Luby-style rounds with
deterministic priorities); not wired into the GPU path yet - round-2 work.
"""
from __future__ import annotations

import numpy as np


def color_elements(elem_nodes: np.ndarray, elem_ptr: np.ndarray | None = None, n_nodes: int | None = None, max_colors: int = 255):
    """Greedy independent-set colouring.

    elem_nodes: (ne, k) array of node ids (fixed k), or a flat array with `elem_ptr` (ne+1 offsets) for ragged lists.
    Returns (colors uint8 [ne], ncolors).  Deterministic: priorities are a fixed hash of the element id.
    """
    if elem_ptr is None:
        elem_nodes = np.asarray(elem_nodes)
        ne, k = elem_nodes.shape
        flat = elem_nodes.ravel().astype(np.int64)
        owner = np.repeat(np.arange(ne, dtype=np.int64), k)
    else:
        flat = np.asarray(elem_nodes, dtype=np.int64)
        elem_ptr = np.asarray(elem_ptr, dtype=np.int64)
        ne = elem_ptr.size - 1
        owner = np.repeat(np.arange(ne, dtype=np.int64), np.diff(elem_ptr))
    n_nodes = int(flat.max()) + 1 if n_nodes is None else n_nodes
    # fixed pseudo-random priorities (splitmix-style hash), ties impossible because the id is mixed in the low bits
    h = (np.arange(ne, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)) * np.uint64(0xBF58476D1CE4E5B9)
    h ^= h >> np.uint64(31)
    prio = ((h >> np.uint64(20)) << np.uint64(24) | np.arange(ne, dtype=np.uint64) & np.uint64(0xFFFFFF)).astype(np.int64) & np.int64(0x7FFFFFFFFFFFFFFF)
    colors = np.full(ne, 255, dtype=np.uint8)
    uncolored = np.ones(ne, dtype=bool)
    c = 0
    while uncolored.any():
        if c >= max_colors:
            raise RuntimeError("color_elements: more than max_colors colours needed")
        # one colour = a maximal independent set of the still uncoloured elements, built in a few Luby rounds
        cand = uncolored.copy()
        blocked_node = np.zeros(n_nodes, dtype=bool)
        while cand.any():
            act = cand[owner]
            node_max = np.full(n_nodes, -1, dtype=np.int64)
            np.maximum.at(node_max, flat[act], prio[owner[act]])
            is_max = np.ones(ne, dtype=bool)
            lose = act & (node_max[flat] != prio[owner])
            is_max[owner[lose]] = False
            win = cand & is_max
            colors[win] = c
            uncolored[win] = False
            blocked_node[flat[win[owner]]] = True
            # elements touching a node of a winner cannot join this colour any more
            touch = np.zeros(ne, dtype=bool)
            touch[owner[blocked_node[flat]]] = True
            cand &= ~touch & ~win
        c += 1
    return colors, c


def color_groups(groups, ndof: int):
    """Colour the elements of all pattern groups together on the node of EVERY local dof (node = dof // 3).  Two elements
    that share a dof share its node, whatever order a pattern lists its dofs in, so no dof is shared inside a colour.
    (For node-major patterns, local dof j = 3 node[j // 3] + j % 3, the node sets and so the colours are those of the
    first dof of every triple.)  Returns (colors per group, ncolors)."""
    flat = np.concatenate([(g.loc_dof // 3).T.ravel() for g in groups]) if groups else np.zeros(0, np.int64)
    counts = np.concatenate([np.full(g.loc_dof.shape[1], g.loc_dof.shape[0], dtype=np.int64) for g in groups]) if groups else np.zeros(0, np.int64)
    ptr = np.concatenate([[0], np.cumsum(counts)])
    colors, ncolors = color_elements(flat, ptr, ndof // 3 + 1)
    split = np.cumsum([g.loc_dof.shape[1] for g in groups])[:-1]
    return np.split(colors, split), ncolors


def color_conflicts(idx_per_group, colors_per_group, n: int) -> int:
    """Number of (colour, free dof) pairs that two different elements of one colour touch; 0 for a valid colouring.
    idx_per_group: (nd, ne) dof indices in the free numbering (-1 = clamped); an element's own repeats do not count."""
    dofs, cols = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for idx, col in zip(idx_per_group, colors_per_group):
        if idx.shape[1] == 0:
            continue
        s = np.sort(idx, axis=0)
        keep = s >= 0
        keep[1:] &= s[1:] != s[:-1]                  # each element's distinct free dofs once
        dofs.append(s[keep].astype(np.int64))
        cols.append(np.broadcast_to(np.asarray(col, dtype=np.int64)[None, :], s.shape)[keep])
    dofs, cols = np.concatenate(dofs), np.concatenate(cols)
    order = np.argsort(cols, kind="stable")
    cuts = np.nonzero(np.diff(cols[order]))[0] + 1
    bad = 0
    for part in np.split(order, cuts):
        if part.size:
            bad += int((np.bincount(dofs[part], minlength=n) > 1).sum())
    return bad


def hex_parity_colors(ex: np.ndarray, ey: np.ndarray, ez: np.ndarray):
    """The optimal 8-colouring of a structured hex mesh: colour = parity of the element coordinates."""
    return ((ex & 1) | ((ey & 1) << 1) | ((ez & 1) << 2)).astype(np.uint8), 8
