"""Generate tests/golden/hybrid_*.npz from the unmodified reference: ``HybridDualVEM.matrix_rhs``
(numerics/vem/hybrid.py) on a Cartesian line, a tilted line, an anisotropic 2-D Cartesian grid, sheared triangles, a
tilted plane, perturbed hexahedra, Delaunay tetrahedra and the agglomerated polygons and polyhedra of
``make_dual_golden`` (up to 32 faces per cell, the most one warp condenses).  Every fixture has Dirichlet faces (the
low end of the grid's longest extent) and Neumann faces (the rest of the boundary), nonzero boundary values and a
nonzero source; the line, the tilted plane, the hexahedra and the polyhedra have a heterogeneous aperture.  Each
fixture holds the grid arrays (``make_golden.grid_arrays``), the tensor (``K``), the boundary condition in the
``golden_io`` layout, ``bc_values``, ``source``, ``aperture`` and the reference's ``H`` and ``rhs``.
   python tools/make_hybrid_golden.py"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_dual_golden import make_grid, rotation  # noqa: E402
from make_golden import OUT, grid_arrays, pp, put_matrix  # noqa: E402


def grid(kind, rng):
    if kind == "line":
        g = pp.CartGrid(np.array([7]), 1.5)
        g.compute_geometry()
        return g
    if kind == "line_tilted":
        g = pp.CartGrid(np.array([6]), 2.0)
        g.nodes = rotation(0.4, -0.7, 0.2) @ g.nodes + np.array([[0.3], [-0.1], [0.5]])
        g.compute_geometry()
        return g
    return make_grid(kind, rng)


def permeability(g, rng):
    """Full anisotropic SPD tensor per cell, scaled by 10^(3 u), u uniform in [0, 1)."""
    nc = g.num_cells
    a = rng.standard_normal((3, 3, nc)) * 0.3
    for i in range(3):
        a[i, i] += 1.0
    k = np.einsum("ikc,jkc->ijc", a, a) * 10.0 ** (3.0 * rng.random(nc))
    if g.dim == 1:
        return pp.SecondOrderTensor(kxx=k[0, 0])
    if g.dim == 2:
        return pp.SecondOrderTensor(kxx=k[0, 0], kyy=k[1, 1], kxy=k[0, 1])
    return pp.SecondOrderTensor(kxx=k[0, 0], kyy=k[1, 1], kzz=k[2, 2], kxy=k[0, 1], kxz=k[0, 2], kyz=k[1, 2])


def boundary(g):
    """Dirichlet on the faces nearest the low end of the grid's longest extent, Neumann on the rest."""
    bf = g.get_all_boundary_faces()
    x = g.face_centers[:, bf]
    ax = int(np.argmax(np.ptp(g.nodes, axis=1)))
    lo, hi = x[ax].min(), x[ax].max()
    lab = np.array(["neu"] * bf.size, dtype=object)
    lab[x[ax] < lo + 1e-8 + 0.2 * (hi - lo)] = "dir"
    return pp.BoundaryCondition(g, bf, list(lab))


def case(kind, seed, aperture):
    rng = np.random.default_rng(seed)
    g = grid(kind, rng)
    k = permeability(g, rng)
    bc = boundary(g)
    bc_values = rng.standard_normal(g.num_faces)
    source = rng.standard_normal(g.num_cells)
    a = 0.2 + rng.random(g.num_cells) if aperture else np.ones(g.num_cells)
    params = {"second_order_tensor": k, "bc": bc, "bc_values": bc_values, "source": source, "aperture": a}
    data = pp.initialize_data({}, "flow", params)
    from porepy.numerics.vem import hybrid
    H, rhs = hybrid.HybridDualVEM("flow").matrix_rhs(g, data)
    assert np.any(bc.is_dir) and np.any(bc.is_neu) and np.any(source != 0), kind
    d = grid_arrays(g)
    d.update(kind=np.array("hybrid"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=bc.is_internal, bc_robin_weight=bc.robin_weight, bc_values=bc_values, source=source,
             aperture=a, rhs=rhs)
    put_matrix(d, "H", H)
    name = f"hybrid_{kind}"
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, g.num_cells, "cells")


CASES = [("line", True), ("line_tilted", False), ("cart2d", False), ("tri2d_sheared", False),
         ("plane_tilted", True), ("cart3d_pert", True), ("tet3d_delaunay", False), ("poly2d", False), ("poly3d", True)]

if __name__ == "__main__":
    for i, (kind, aperture) in enumerate(CASES):
        case(kind, 300 + i, aperture)
