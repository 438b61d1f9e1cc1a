"""Generate tests/golden/tpsa_*.npz from the unmodified reference's ``pp.Tpsa.discretize`` (run in the build
container, where the reference is importable).

Each fixture holds one grid (``make_golden.grid_arrays``), the shear modulus ``mu`` (seeded, heterogeneous; every case
has a 10^6 contrast between two groups of cells), the boundary condition in the layout ``tests/golden_io.load_case``
reads, the faces of ``get_all_boundary_faces()`` and the 14 matrices the reference wrote.  Cases the reference refuses
or fails on are listed in ``REFUSED`` with the reason and are not written.

    python tools/make_tpsa_golden.py [name-prefix]
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
from make_golden import OUT, grid_arrays, perturb, pp, put_matrix  # noqa: E402

KEYS = ("stress", "stress_rotation", "stress_total_pressure", "rotation_displacement", "rotation_rotation",
        "solid_mass_displacement", "solid_mass_total_pressure", "bound_displacement_cell",
        "bound_displacement_rotation_cell", "bound_displacement_solid_pressure_cell", "bound_stress",
        "bound_rotation_displacement", "bound_mass_displacement", "bound_displacement_face")

# cases the reference refuses or fails on (name -> reason); none at present
REFUSED: dict = {}


def shear_modulus(g, rng):
    """exp(N(0, 0.5)) per cell, times 10^6 on the cells with x < 0.5 (contrast across a plane of faces)."""
    mu = np.exp(0.5 * rng.standard_normal(g.num_cells))
    mu[g.cell_centers[0] < 0.5] *= 1e6
    return mu


def sides(g, bf, tol=1e-10):
    xf = g.face_centers[:, bf]
    lo = [bf[np.abs(xf[i] - g.nodes[i].min()) < tol] for i in range(g.dim)]
    hi = [bf[np.abs(xf[i] - g.nodes[i].max()) < tol] for i in range(g.dim)]
    return lo, hi


def bc_all_dirichlet(g, rng):
    bf = g.get_all_boundary_faces()
    return pp.BoundaryConditionVectorial(g, bf, ["dir"] * bf.size)


def bc_rollers(g, rng):
    """Rollers on every "low" side (Dirichlet in the normal direction, Neumann tangentially), Dirichlet on the first
    "high" side, Neumann elsewhere."""
    bf = g.get_all_boundary_faces()
    lo, hi = sides(g, bf)
    bc = pp.BoundaryConditionVectorial(g)
    for i in range(g.dim):
        bc.is_dir[i, lo[i]] = True
        bc.is_neu[i, lo[i]] = False
    bc.is_dir[:, hi[0]] = True
    bc.is_neu[:, hi[0]] = False
    return bc


def bc_sheared(g, rng):
    """The sheared triangle grid: rollers on both 45-degree sides (Dirichlet in x on the left one, in y on the right
    one; Neumann in the other component), Dirichlet at y = 0, Neumann at y = 1."""
    bf = g.get_all_boundary_faces()
    n = g.face_normals[:, bf]
    diag = np.abs(n[0]) == np.abs(n[1])
    left = bf[diag & (g.face_centers[0, bf] - g.face_centers[1, bf] < 0.5)]
    right = bf[diag & (g.face_centers[0, bf] - g.face_centers[1, bf] > 0.5)]
    bottom = bf[np.abs(g.face_centers[1, bf]) < 1e-10]
    assert left.size and right.size, "no 45-degree boundary faces"
    bc = pp.BoundaryConditionVectorial(g, bottom, ["dir"] * bottom.size)
    bc.is_dir[0, left] = True
    bc.is_neu[0, left] = False
    bc.is_dir[1, right] = True
    bc.is_neu[1, right] = False
    return bc


def bc_robin(g, rng):
    """Dirichlet at x = min, a roller at y = min, diagonal Robin (weights 0.2 .. 5, different per component) at
    z = max (y = max in 2-D), Neumann elsewhere."""
    bc = bc_rollers(g, rng)
    bf = g.get_all_boundary_faces()
    lo, hi = sides(g, bf)
    bc.is_dir[:, hi[0]] = False
    bc.is_neu[:, hi[0]] = True
    top = hi[g.dim - 1]
    top = top[~np.isin(top, lo[0])]
    bc.is_rob[:, top] = True
    bc.is_dir[:, top] = False
    bc.is_neu[:, top] = False
    w = np.zeros((g.dim, g.dim, g.num_faces))
    for i in range(g.dim):
        w[i, i] = np.exp(rng.uniform(np.log(0.2), np.log(5.0), g.num_faces))
    bc.robin_weight = w
    return bc


def grid_of(kind, rng):
    if kind == "cart2d":
        g = pp.CartGrid([6, 5], [1.0, 1.0])
    elif kind == "tri2d_sheared":
        # x -> x + y turns the vertical sides into 45-degree faces (|n_x| == |n_y| exactly): the tie rule of the
        # scalar Dirichlet filter (tpsa.py:1053) is exercised on its rollers
        g = pp.StructuredTriangleGrid([4, 4], [1.0, 1.0])
        g.nodes[0] += g.nodes[1]
    elif kind == "cart3d":
        g = pp.CartGrid([4, 3, 3], [1.0, 1.0, 1.0])
    elif kind == "cart3d_pert":
        g = pp.CartGrid([4, 4, 3], [1.0, 1.0, 1.0])
        perturb(g, rng)
        return g
    elif kind == "tet3d_delaunay":
        pts = rng.random((3, 20))
        corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [1, 0, 1],
                            [0, 1, 1], [1, 1, 1]], float).T
        g = pp.TetrahedralGrid(np.hstack((corners, pts)))
    elif kind == "frac3d":
        # one fracture plane at z = 0.5, split: its faces are tagged fracture_faces and have one cell each
        frac = np.array([[0.25, 0.75, 0.75, 0.25], [0.25, 0.25, 0.75, 0.75], [0.5, 0.5, 0.5, 0.5]])
        mdg = pp.meshing.cart_grid([frac], [4, 4, 4], physdims=[1.0, 1.0, 1.0])
        g = mdg.subdomains(dim=3)[0]
        return g
    else:
        raise ValueError(kind)
    g.compute_geometry()
    return g


def case(name, kind, make_bc, seed, clear_fracture_faces=False):
    rng = np.random.default_rng(seed)
    try:
        g = grid_of(kind, rng)
        mu = shear_modulus(g, rng)
        bc = make_bc(g, rng)
        if clear_fracture_faces:
            # internal boundaries with no condition set go through the interior formulas (tpsa.py:1023)
            ff = np.asarray(g.tags["fracture_faces"], bool)
            bc.is_neu[:, ff] = bc.is_dir[:, ff] = bc.is_rob[:, ff] = False
        C = pp.FourthOrderTensor(mu, np.ones(g.num_cells))
        data = pp.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc})
        pp.Tpsa("mech").discretize(g, data)
    except Exception as e:  # noqa: BLE001 -- recorded, not dropped silently
        REFUSED[name] = f"{type(e).__name__}: {e}"
        print(name, "REFUSED by the reference:", REFUSED[name])
        return
    M = data[pp.DISCRETIZATION_MATRICES]["mech"]
    d = grid_arrays(g)
    bmask = np.zeros(g.num_faces, bool)
    bmask[g.get_all_boundary_faces()] = True
    d.update(kind=np.array("tpsa"), mu=mu, boundary_faces=bmask,
             bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=np.asarray(bc.is_internal, bool), bc_robin_weight=np.asarray(bc.robin_weight, float),
             bc_basis=np.asarray(bc.basis, float))
    for key in KEYS:
        put_matrix(d, key, M[key])
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print(name, "nc", g.num_cells, "nf", g.num_faces, f"{os.path.getsize(path) / 1e3:.0f} kB")


CASES = [
    ("tpsa_cart2d_dir", "cart2d", bc_all_dirichlet, 101, False),
    ("tpsa_tri2d_sheared", "tri2d_sheared", bc_sheared, 102, False),
    ("tpsa_cart3d_rollers", "cart3d", bc_rollers, 103, False),
    ("tpsa_cart3d_robin", "cart3d", bc_robin, 104, False),
    ("tpsa_cart2d_robin", "cart2d", bc_robin, 105, False),
    ("tpsa_cart3d_pert", "cart3d_pert", bc_rollers, 106, False),
    ("tpsa_tet3d_delaunay", "tet3d_delaunay", bc_robin, 107, False),
    ("tpsa_frac3d", "frac3d", bc_rollers, 108, True),
]


def main():
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    for name, kind, make_bc, seed, clear in CASES:
        if name.startswith(only):
            case(name, kind, make_bc, seed, clear)
    if REFUSED:
        print("refused by the reference:", REFUSED)


if __name__ == "__main__":
    main()
