"""Polytopal grids by agglomeration: the cells of a fine grid that share a label become one coarse cell.  Used by the
golden tools (``make_dual_golden``, ``make_hybrid_golden``, ``make_golden.case_geometry``) on the reference's grids
and by the tests on ``porepy_b200.Grid``; it imports neither.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps


def _loop(loops):
    """Boundary loop of a patch of consistently oriented face loops: the directed edges that appear in one face only,
    chained from the first face's first such edge."""
    count = {}
    for lp in loops:
        for a, b in zip(lp, np.roll(lp, -1)):
            key = (min(a, b), max(a, b))
            count[key] = count.get(key, 0) + 1
    nxt = {}
    for lp in loops:
        for a, b in zip(lp, np.roll(lp, -1)):
            if count[(min(a, b), max(a, b))] == 1:
                nxt[int(a)] = int(b)
    start = next(int(a) for a, b in zip(loops[0], np.roll(loops[0], -1)) if int(a) in nxt and nxt[int(a)] == int(b))
    out = [start]
    while nxt[out[-1]] != start:
        out.append(nxt[out[-1]])
    assert len(out) == len(nxt), "the merged faces do not form one simple patch"
    return np.array(out)


def agglomerate(g, label, merge=(), grid_cls=None, name="Agglomerate"):
    """The grid whose cell ``k`` is the union of the cells of ``g`` with ``label == k``.  Faces between two cells of one
    group are removed and nodes no face uses any more are dropped; the remaining faces keep their order and their node
    loops.  ``merge``: groups of faces of ``g`` (coplanar, on the boundary of one coarse cell, consistently oriented),
    each replaced by one polygonal face whose nodes are the group's boundary loop, at the position of its first face.
    ``grid_cls(dim, nodes, face_nodes, cell_faces, name)`` builds the result (default: the class named ``Grid`` among
    the bases of ``g``'s class).  The geometry is not computed."""
    label = np.asarray(label)
    nc = int(label.max()) + 1
    assert np.array_equal(np.unique(label), np.arange(nc))
    if grid_cls is None:
        grid_cls = next(c for c in type(g).__mro__ if c.__name__ == "Grid")
    P = sps.csc_matrix((np.ones(g.num_cells), (np.arange(g.num_cells), label)), shape=(g.num_cells, nc))
    cf = (sps.csc_matrix(g.cell_faces, dtype=float) @ P).tocsr()
    cf.eliminate_zeros()
    fn = sps.csc_matrix(g.face_nodes)
    loops = {f: fn.indices[fn.indptr[f]:fn.indptr[f + 1]] for f in range(g.num_faces)}
    drop = set()
    for group in merge:
        group = sorted(int(f) for f in group)
        rows = cf[group]
        assert all(rows[i].nnz == 1 for i in range(len(group))), "merged faces must lie on the domain boundary"
        assert len({(rows[i].indices[0], rows[i].data[0]) for i in range(len(group))}) == 1, \
            "merged faces must belong to one cell with one orientation"
        loops[group[0]] = _loop([loops[f] for f in group])
        drop.update(group[1:])
    keep = [f for f in range(g.num_faces) if cf.indptr[f + 1] > cf.indptr[f] and f not in drop]
    used = np.unique(np.concatenate([loops[f] for f in keep]))
    renum = np.full(g.num_nodes, -1)
    renum[used] = np.arange(used.size)
    lens = np.array([loops[f].size for f in keep])
    face_nodes = sps.csc_matrix((np.ones(lens.sum(), bool), renum[np.concatenate([loops[f] for f in keep])],
                                 np.r_[0, np.cumsum(lens)]), shape=(used.size, len(keep)))
    cell_faces = sps.csc_matrix(cf[keep].astype(float))
    cell_faces.sort_indices()
    return grid_cls(g.dim, np.asarray(g.nodes, float)[:, used], face_nodes, cell_faces, name)


def interleave(counts):
    """A permutation of the coarse cells that deals them out round-robin by their face count, so that consecutive cells
    have different counts wherever the counts allow it: ``new_label = rank[old_label]``."""
    counts = np.asarray(counts)
    groups = [list(np.flatnonzero(counts == n)) for n in np.unique(counts)]
    order = []
    while any(groups):
        for gr in groups:
            if gr:
                order.append(gr.pop(0))
    rank = np.empty(counts.size, int)
    rank[np.array(order)] = np.arange(counts.size)
    return rank
