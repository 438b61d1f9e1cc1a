"""Generate tests/golden/dual_{mvem,rt0}_*.npz from the unmodified reference: ``pp.MVEM`` / ``pp.RT0`` discretize and
``assemble_matrix_rhs`` on 1-D, 2-D and 3-D grids (Cartesian, sheared triangles, perturbed Cartesian, structured and
Delaunay tetrahedra, a tilted line and a tilted plane in 3-D, and agglomerated polygons and polyhedra of up to 32
faces: ``poly2d``, ``poly3d`` and ``poly_plane_tilted``), with a heterogeneous full anisotropic permeability of
10^6 contrast, Dirichlet, Neumann and Robin faces together, and a vector source.  Each fixture holds the grid arrays
(``make_golden.grid_arrays``), the tensor (``K``), the boundary condition in the ``golden_io`` layout, ``bc_values``,
``vector_source`` and the reference's ``mass``, ``div``, ``vector_proj``, ``A`` and ``b``.  The prefix ``dual_`` keeps
these fixtures out of every other test's set.
   python tools/make_dual_golden.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from agglomerate import agglomerate, interleave  # noqa: E402
from make_golden import OUT, grid_arrays, pp, put_matrix  # noqa: E402


def rotation(a, b, c):
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    rz = np.array([[ca, -sa, 0], [sa, ca, 0], [0, 0, 1]])
    ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    rx = np.array([[1, 0, 0], [0, cc, -sc], [0, sc, cc]])
    return rz @ ry @ rx


# poly2d: the labels of a 12 x 10 CartGrid, top row first.  A: an 8 x 8 block (32 edges); U: a U-shaped cell whose
# centroid lies in its notch N (16 edges); the rest are 1 x 1 to 5 x 1 and 3 x 2 rectangles (4, 6, 8, 10, 12 edges).
POLY2D = ["aabbbcccddee",
          "fffffcccggee",
          "AAAAAAAAgghi",
          "AAAAAAAAjjji",
          "AAAAAAAAkkkk",
          "AAAAAAAAlllm",
          "AAAAAAAAlllm",
          "AAAAAAAAUNUm",
          "AAAAAAAAUNUm",
          "AAAAAAAAUUUm"]


def polytopes(g, label, merge=()):
    """``agglomerate`` with the coarse cells numbered round-robin by face count (the four warps of one block of the
    hybridization kernel then hold cells of different sizes)."""
    counts = np.diff(sps.csc_matrix(agglomerate(g, label, merge).cell_faces).indptr)
    return agglomerate(g, interleave(counts)[label], merge)


def poly2d():
    g = pp.CartGrid([12, 10], [1.2, 1.0])
    g.nodes = np.array([[1.0, 0.35, 0.0], [0.1, 1.0, 0.0], [0.0, 0.0, 1.0]]) @ g.nodes   # edges off the axes
    _, label = np.unique(np.array([list(r) for r in POLY2D[::-1]]).ravel(), return_inverse=True)
    return polytopes(g, label)


def poly3d(rng):
    """A 5 x 4 x 4 TensorGrid of uneven spacing under a global shear (planar faces), agglomerated into 3 x 2 x 2 (32
    faces), 2 x 2 x 2 (24), 2 x 1 x 1 (10) and single cells; on the 3 x 2 x 2 cell at the origin the boundary sub-faces
    of the planes x = 0 and y = 0 are merged into one face of 8 and one of 10 nodes (that cell keeps 24 faces)."""
    g = pp.TensorGrid(*[np.concatenate(([0.0], np.cumsum(0.5 + rng.random(n)))) for n in (5, 4, 4)])
    lab = -np.ones((5, 4, 4), int)
    blocks = [(slice(0, 3), slice(0, 2), slice(0, 2)), (slice(0, 3), slice(2, 4), slice(0, 2)),
              (slice(3, 5), slice(0, 2), slice(0, 2)), (slice(0, 3), slice(0, 2), slice(2, 4)),
              (slice(3, 5), slice(0, 2), slice(2, 4))]
    blocks += [(slice(3, 5), j, k) for j in (2, 3) for k in (0, 1, 2, 3)]
    blocks += [(i, j, k) for i in range(3) for j in (2, 3) for k in (2, 3)]
    for n, b in enumerate(blocks):
        lab[b] = n
    label = lab.ravel(order="F")    # cell i + nx (j + ny k)
    g.compute_geometry()
    cf = sps.csr_matrix(g.cell_faces)
    first = np.flatnonzero(label == 0)
    faces = np.unique(sps.csc_matrix(g.cell_faces)[:, first].indices)
    bnd = faces[np.diff(cf.indptr)[faces] == 1]
    merge = [bnd[np.abs(g.face_centers[0, bnd]) < 1e-12], bnd[np.abs(g.face_centers[1, bnd]) < 1e-12]]
    g.nodes = np.array([[1.0, 0.3, -0.2], [0.1, 1.0, 0.25], [-0.15, 0.2, 1.0]]) @ g.nodes
    return polytopes(g, label, merge)


def make_grid(kind, rng):
    if kind == "cart2d":
        g = pp.CartGrid([5, 4], [1.0, 1.0])
    elif kind == "tri2d_sheared":
        g = pp.StructuredTriangleGrid([4, 3], [1.0, 1.0])
        g.nodes[0] += 0.4 * g.nodes[1]
    elif kind == "cart3d":
        g = pp.CartGrid([3, 3, 2], [1.0, 1.0, 1.0])
    elif kind == "cart3d_pert":
        # uneven spacing on every axis and a global shear: perturbed nodes, planar faces (a warped hexahedron fails
        # the reference's consistency test; tests/test_dual.py checks that refusal)
        x = [np.concatenate(([0.0], np.cumsum(0.5 + rng.random(3)))) for _ in range(3)]
        g = pp.TensorGrid(*x)
        g.nodes = np.array([[1.0, 0.3, -0.2], [0.1, 1.0, 0.25], [-0.15, 0.2, 1.0]]) @ g.nodes
    elif kind == "tet3d":
        g = pp.StructuredTetrahedralGrid([2, 2, 2], [1.0, 1.0, 1.0])
    elif kind == "tet3d_delaunay":
        # random interior points, redrawn until no tetrahedron is a sliver (volume / diameter^3 >= 0.01; a regular
        # tetrahedron has 0.118): on slivers the MVEM projector is so ill-conditioned that two correct evaluations
        # round apart by more than the 1e-12 the fixtures are compared at
        corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [1, 0, 1],
                            [0, 1, 1], [1, 1, 1]], float).T
        while True:
            g = pp.TetrahedralGrid(np.hstack((corners, 0.15 + 0.7 * rng.random((3, 6)))))
            g.compute_geometry()
            cn = (abs(g.face_nodes) @ abs(g.cell_faces)).tocsc()
            diam = np.array([np.ptp(g.nodes[:, cn.indices[cn.indptr[c]:cn.indptr[c + 1]]], axis=1).max()
                             for c in range(g.num_cells)])
            if (g.cell_volumes / diam ** 3).min() >= 0.01:
                return g
    elif kind == "line_tilted":
        g = pp.CartGrid(np.array([6]), 2.0)
        g.nodes = rotation(0.4, -0.7, 0.2) @ g.nodes + np.array([[0.3], [-0.1], [0.5]])
    elif kind == "plane_tilted":
        g = pp.CartGrid([4, 3], [1.0, 0.8])
        g.nodes = rotation(0.3, 0.9, -0.5) @ g.nodes + np.array([[0.2], [0.1], [-0.3]])
    elif kind == "poly2d":
        g = poly2d()
    elif kind == "poly3d":
        g = poly3d(rng)
    elif kind == "poly_plane_tilted":
        g = poly2d()
        g.nodes = rotation(0.3, 0.9, -0.5) @ g.nodes + np.array([[0.2], [0.1], [-0.3]])
    elif kind == "tri_plane_tilted":
        g = pp.StructuredTriangleGrid([3, 3], [1.0, 1.0])
        g.nodes = rotation(-0.6, 0.5, 1.1) @ g.nodes
    else:
        raise ValueError(kind)
    g.compute_geometry()
    return g


def permeability(g, rng):
    """Full anisotropic SPD tensor per cell, scaled by 10^(6 u), u uniform in [0, 1): a 10^6 contrast."""
    nc = g.num_cells
    a = rng.standard_normal((3, 3, nc)) * 0.3
    for i in range(3):
        a[i, i] += 1.0
    k = np.einsum("ikc,jkc->ijc", a, a) * 10.0 ** (6.0 * rng.random(nc))
    if g.dim == 2 and np.ptp(g.nodes[2]) == 0:   # a grid in the xy-plane: the reference's 2-D tensor (kzz = 1)
        return pp.SecondOrderTensor(kxx=k[0, 0], kyy=k[1, 1], kxy=k[0, 1])
    return pp.SecondOrderTensor(kxx=k[0, 0], kyy=k[1, 1], kzz=k[2, 2], kxy=k[0, 1], kxz=k[0, 2], kyz=k[1, 2])


def boundary(g, rng):
    """Dirichlet on the faces nearest the low end of the grid's longest extent, Robin on the high end, Neumann on the
    rest."""
    bf = g.get_all_boundary_faces()
    x = g.face_centers[:, bf]
    ax = int(np.argmax(np.ptp(g.nodes, axis=1)))
    lo, hi = x[ax].min(), x[ax].max()
    lab = np.array(["neu"] * bf.size, dtype=object)
    lab[x[ax] < lo + 1e-8 + 0.2 * (hi - lo)] = "dir"
    lab[x[ax] > hi - 1e-8 - 0.2 * (hi - lo)] = "rob"
    bc = pp.BoundaryCondition(g, bf, list(lab))
    bc.robin_weight = 0.5 + rng.random(g.num_faces)
    return bc


def case(method, kind, seed):
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    k = permeability(g, rng)
    bc = boundary(g, rng)
    bc_values = rng.standard_normal(g.num_faces)
    vsrc = rng.standard_normal(3 * g.num_cells)
    kw = "flow"
    params = {"second_order_tensor": k, "bc": bc, "bc_values": bc_values, "vector_source": vsrc}
    data = {pp.PARAMETERS: {kw: params}, pp.DISCRETIZATION_MATRICES: {kw: {}}}
    discr = {"mvem": pp.MVEM, "rt0": pp.RT0}[method](kw)
    discr.discretize(g, data)
    A, b = discr.assemble_matrix_rhs(g, data)
    mats = data[pp.DISCRETIZATION_MATRICES][kw]
    assert np.any(bc.is_dir) and np.any(bc.is_rob) and (g.dim == 1 or np.any(bc.is_neu)), kind
    d = grid_arrays(g)
    d.update(kind=np.array(method), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=bc.is_internal, bc_robin_weight=bc.robin_weight, bc_values=bc_values, vector_source=vsrc,
             b=b)
    for key in ("mass", "div", "vector_proj"):
        put_matrix(d, key, mats[key])
    put_matrix(d, "A", A)
    name = f"dual_{method}_{kind}"
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, g.num_cells, "cells")


CASES = [("mvem", "cart2d"), ("mvem", "tri2d_sheared"), ("mvem", "cart3d"), ("mvem", "cart3d_pert"),
         ("mvem", "tet3d"), ("mvem", "tet3d_delaunay"), ("mvem", "line_tilted"), ("mvem", "plane_tilted"),
         ("rt0", "tri2d_sheared"), ("rt0", "tet3d"), ("rt0", "tet3d_delaunay"), ("rt0", "line_tilted"),
         ("rt0", "tri_plane_tilted"), ("mvem", "poly2d"), ("mvem", "poly3d"), ("mvem", "poly_plane_tilted")]

if __name__ == "__main__":
    for i, (m, k) in enumerate(CASES):
        case(m, k, 100 + i)
