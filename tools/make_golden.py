"""Generate tests/golden/*.npz from the unmodified reference (run in the build container).

Each fixture holds one grid (the arrays of pp.Grid the hot path reads), one set of
parameters (permeability / stiffness / boundary condition / coupling tensors) and
the matrices the reference's ``Mpfa/Mpsa/Biot.discretize`` wrote to
``data[pp.DISCRETIZATION_MATRICES][kw]``.  The GPU box never sees /root/reference;
tests read only these files.

    python tools/make_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_porepy  # noqa: E402

pp = load_porepy()
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def grid_arrays(g) -> dict:
    fn = sps.csc_matrix(g.face_nodes)
    cf = sps.csc_matrix(g.cell_faces)
    cf.sort_indices()
    return dict(
        dim=np.int64(g.dim), name=np.array(str(g.name)), nodes=g.nodes,
        fn_indptr=fn.indptr.astype(np.int32), fn_indices=fn.indices.astype(np.int32),
        cf_indptr=cf.indptr.astype(np.int32), cf_indices=cf.indices.astype(np.int32),
        cf_data=cf.data.astype(np.int8), face_normals=g.face_normals,
        face_centers=g.face_centers, face_areas=g.face_areas,
        cell_centers=g.cell_centers, cell_volumes=g.cell_volumes,
        fracture_faces=np.asarray(g.tags["fracture_faces"], bool),
    )


def put_matrix(d: dict, key: str, m) -> None:
    m = sps.csr_matrix(m)
    m.sum_duplicates()
    d[f"M__{key}__data"] = m.data
    d[f"M__{key}__indices"] = m.indices.astype(np.int32)
    d[f"M__{key}__indptr"] = m.indptr.astype(np.int32)
    d[f"M__{key}__shape"] = np.array(m.shape, dtype=np.int64)


def perturb(g, rng, amp=0.2):
    g.compute_geometry()
    h = np.min(g.cell_volumes) ** (1.0 / g.dim)
    bn = np.zeros(g.num_nodes, bool)
    bf = g.get_all_boundary_faces()
    fn = sps.csc_matrix(g.face_nodes)
    for f in bf:
        bn[fn.indices[fn.indptr[f]:fn.indptr[f + 1]]] = True
    pert = amp * h * (0.5 - rng.random((g.dim, g.num_nodes)))
    pert[:, bn] = 0
    g.nodes[:g.dim] += pert
    g.compute_geometry()


def make_grid(kind, rng):
    if kind == "cart3d":
        g = pp.CartGrid([4, 3, 3], [1.0, 1.0, 1.0])
    elif kind == "cart3d_pert":
        g = pp.CartGrid([4, 4, 3], [1.0, 1.0, 1.0])
        perturb(g, rng)
        return g
    elif kind == "tet3d":
        g = pp.StructuredTetrahedralGrid([2, 2, 2], [1.0, 1.0, 1.0])
    elif kind in ("tet3d_delaunay", "tet3d_delaunay_small"):
        # the small mesh keeps the MPSA fixture (nearly dense 3 x 3 blocks) under 1 MB
        pts = rng.random((3, 22 if kind == "tet3d_delaunay" else 12))
        corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [1, 0, 1],
                            [0, 1, 1], [1, 1, 1]], float).T
        g = pp.TetrahedralGrid(np.hstack((corners, pts)))
    elif kind == "cart2d":
        g = pp.CartGrid([5, 4], [1.0, 1.0])
    elif kind == "tri2d":
        g = pp.StructuredTriangleGrid([3, 3], [1.0, 1.0])
    else:
        raise ValueError(kind)
    g.compute_geometry()
    return g


def scalar_bc(g, rng, robin):
    bf = g.get_all_boundary_faces()
    xf = g.face_centers[:, bf]
    labels = np.array(["neu"] * bf.size, dtype=object)
    labels[xf[0] < 1e-10] = "dir"
    labels[xf[0] > 1 - 1e-10] = "dir"
    if robin:
        labels[(xf[1] < 1e-10) & (xf[0] > 1e-10) & (xf[0] < 1 - 1e-10)] = "rob"
    bc = pp.BoundaryCondition(g, bf, list(labels))
    if robin:
        bc.robin_weight = 0.5 + rng.random(g.num_faces)
    return bc


def vector_bc(g, rng, robin):
    bf = g.get_all_boundary_faces()
    xf = g.face_centers[:, bf]
    bc = pp.BoundaryConditionVectorial(g)
    d0 = bf[xf[0] < 1e-10]
    bc.is_dir[:, d0] = True
    bc.is_neu[:, d0] = False
    r0 = bf[(xf[1] < 1e-10) & (xf[0] > 1e-10)]  # roller: Dirichlet in y only
    bc.is_dir[1, r0] = True
    bc.is_neu[1, r0] = False
    if robin:
        t0 = bf[(xf[1] > 1 - 1e-10) & (xf[0] > 1e-10)]
        bc.is_rob[:, t0] = True
        bc.is_neu[:, t0] = False
        bc.robin_weight = bc.robin_weight * (0.5 + rng.random(g.num_faces))
    return bc


def case_mpfa(name, kind, robin, seed, contrast=False):
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc = g.num_cells
    if contrast:  # heterogeneous isotropic kappa = 1e+-6 (test_mpfa.py:140-251 pattern)
        kk = np.where(rng.random(nc) < 0.5, 1e-6, 1e6)
        k = pp.SecondOrderTensor(kk)
    else:
        k = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                                 0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
    bc = scalar_bc(g, rng, robin)
    data = pp.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc,
                                            "mpfa_inverter": "python"})
    discr = pp.Mpfa("flow")
    discr.discretize(g, data)
    M = data[pp.DISCRETIZATION_MATRICES]["flow"]
    d = grid_arrays(g)
    d.update(kind=np.array("mpfa"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu,
             bc_is_rob=bc.is_rob, bc_is_internal=bc.is_internal,
             bc_robin_weight=np.asarray(bc.robin_weight, float),
             eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
    for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face",
                "vector_source", "bound_pressure_vector_source"):
        put_matrix(d, key, M[key])
    # a solved problem: A p = b with unit Dirichlet data on x=0 (fv_elliptic.py:67-112)
    bv = np.zeros(g.num_faces)
    bf = g.get_all_boundary_faces()
    bv[bf[g.face_centers[0, bf] < 1e-10]] = 1.0
    data[pp.PARAMETERS]["flow"]["bc_values"] = bv
    A, b = discr.assemble_matrix_rhs(g, data)
    d["bc_values"] = bv
    d["solution"] = sps.linalg.spsolve(sps.csc_matrix(A), b)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "nf", g.num_faces)


def tilt_rotation(rng):
    """A generic rotation (proper orthogonal matrix) from a seeded QR factorization."""
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1
    return q


def case_mpfa_embedded(name, kind, seed, tilt):
    """2-D grid embedded in 3-D (a fracture plane): the reference rotates it into its own plane
    (mpfa.py:733-754) and maps the vector source back to the ambient space (mpfa.py:423-466)."""
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc = g.num_cells
    bc = scalar_bc(g, rng, robin=True)   # labels from the untilted face centres
    if tilt:
        Q = tilt_rotation(rng)
        g.nodes = Q @ g.nodes + np.array([[0.3], [-0.2], [0.7]])
        g.compute_geometry()
    k = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                             0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
    data = pp.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc, "mpfa_inverter": "python",
                                            "ambient_dimension": 3})
    discr = pp.Mpfa("flow")
    discr.discretize(g, data)
    M = data[pp.DISCRETIZATION_MATRICES]["flow"]
    d = grid_arrays(g)
    d.update(kind=np.array("mpfa"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu,
             bc_is_rob=bc.is_rob, bc_is_internal=bc.is_internal,
             bc_robin_weight=np.asarray(bc.robin_weight, float), ambient_dimension=np.int64(3),
             eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
    for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face",
                "vector_source", "bound_pressure_vector_source"):
        put_matrix(d, key, M[key])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "nf", g.num_faces, "vector_source", M["vector_source"].shape)


def case_next_rows(name, kind, seed):
    """TPFA and first-order upwinding (SURVEY 8(f) rank 3) on the same grid / tensors / boundary
    conditions: fixtures for oracle/next_rows_oracle.py."""
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc, nf = g.num_cells, g.num_faces
    k = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                             0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
    bc = scalar_bc(g, rng, robin=False)
    data = pp.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc})
    pp.Tpfa("flow").discretize(g, data)
    M = data[pp.DISCRETIZATION_MATRICES]["flow"]
    d = grid_arrays(g)
    d.update(kind=np.array("next"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu,
             bc_is_rob=bc.is_rob, bc_is_internal=bc.is_internal,
             bc_robin_weight=np.asarray(bc.robin_weight, float), eta=np.float64(0.0))
    for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face",
                "vector_source", "bound_pressure_vector_source"):
        put_matrix(d, "tpfa_" + key, M[key])
    q = rng.standard_normal(nf)
    q[rng.random(nf) < 0.1] = 0.0                       # exact zeros take the "positive" branch
    up = pp.Upwind("transport")
    dat = pp.initialize_data({}, "transport", {"bc": bc, up._flux_array_key: q})
    up.discretize(g, dat)
    U = dat[pp.DISCRETIZATION_MATRICES]["transport"]
    d["darcy_flux"] = q
    put_matrix(d, "upwind", U[up.upwind_matrix_key])
    put_matrix(d, "bound_transport_dir", U[up.bound_transport_dir_matrix_key])
    put_matrix(d, "bound_transport_neu", U[up.bound_transport_neu_matrix_key])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "nf", nf)


def case_partial_update(name, kind, seed, mech=False):
    """The reference's in-place update (``Mpfa / Mpsa.update_discretization`` -> ``partial_update_discretization``,
    _fvutils.py:1090-1257) after the parameters of two cells changed: fixture holds the old and the new
    tensors, the modified cells and the matrices the reference ends up with."""
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc = g.num_cells
    cells = np.sort(rng.choice(nc, size=2, replace=False))
    d = grid_arrays(g)
    if mech:
        C = pp.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))
        bc = vector_bc(g, rng, False)
        kw, discr = "mech", pp.Mpsa("mech")
        data = pp.initialize_data({}, kw, {"fourth_order_tensor": C, "bc": bc, "inverter": "python"})
        discr.discretize(g, data)
        C2 = C.copy()
        C2.values[:, :, cells] *= 3.0
        C2.mu[cells] *= 3.0
        C2.lmbda[cells] *= 3.0
        data[pp.PARAMETERS][kw]["fourth_order_tensor"] = C2
        d.update(kind=np.array("partial_mpsa"), C=C.values, C2=C2.values)
    else:
        k = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                                 0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
        bc = scalar_bc(g, rng, False)
        kw, discr = "flow", pp.Mpfa("flow")
        data = pp.initialize_data({}, kw, {"second_order_tensor": k, "bc": bc, "mpfa_inverter": "python"})
        discr.discretize(g, data)
        k2 = k.copy()
        k2.values[:, :, cells] *= 7.0
        data[pp.PARAMETERS][kw]["second_order_tensor"] = k2
        d.update(kind=np.array("partial_mpfa"), K=k.values, K2=k2.values)
    data["update_discretization"] = {"modified_cells": cells}
    discr.update_discretization(g, data)
    d.update(bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob, bc_is_internal=bc.is_internal,
             bc_robin_weight=np.asarray(bc.robin_weight, float), modified_cells=cells,
             eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
    for key, m in data[pp.DISCRETIZATION_MATRICES][kw].items():
        put_matrix(d, key, m)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "modified", cells)


def case_line(name, seed):
    """A 1-D grid on a tilted line in 3-D (an intersection line of fractures): ``pp.Mpfa`` (which delegates to
    TPFA, mpfa.py:690-712) with 3 ambient components, ``pp.Mpsa`` (mpsa.py:666-697) and upwinding."""
    rng = np.random.default_rng(seed)
    g = pp.CartGrid([6], [1.0])
    g.nodes[0, 1:-1] += 0.05 * (0.5 - rng.random(5))
    x = g.nodes[0].copy()
    g.nodes = np.vstack((0.6 * x, 0.3 * x + 0.1, 0.74 * x - 0.2))
    g.compute_geometry()
    nc, nf = g.num_cells, g.num_faces
    k = pp.SecondOrderTensor(1 + rng.random(nc))
    bc = pp.BoundaryCondition(g, np.array([0]), "dir")
    data = pp.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc, "ambient_dimension": 3})
    pp.Mpfa("flow").discretize(g, data)
    d = grid_arrays(g)
    d.update(kind=np.array("line"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=bc.is_internal, bc_robin_weight=np.asarray(bc.robin_weight, float), eta=np.float64(0.0))
    for key, m in data[pp.DISCRETIZATION_MATRICES]["flow"].items():
        put_matrix(d, "tpfa_" + key, m)
    mu, lam = 1 + rng.random(nc), rng.random(nc)
    md = pp.initialize_data({}, "mech", {"fourth_order_tensor": pp.FourthOrderTensor(mu, lam),
                                         "bc": pp.BoundaryConditionVectorial(g)})
    pp.Mpsa("mech").discretize(g, md)
    d["mu"], d["lmbda"] = mu, lam
    for key, m in md[pp.DISCRETIZATION_MATRICES]["mech"].items():
        put_matrix(d, "mpsa_" + key, m)
    q = rng.standard_normal(nf)
    up = pp.Upwind("transport")
    dat = pp.initialize_data({}, "transport", {"bc": bc, up._flux_array_key: q})
    up.discretize(g, dat)
    U = dat[pp.DISCRETIZATION_MATRICES]["transport"]
    d["darcy_flux"] = q
    put_matrix(d, "upwind", U[up.upwind_matrix_key])
    put_matrix(d, "bound_transport_dir", U[up.bound_transport_dir_matrix_key])
    put_matrix(d, "bound_transport_neu", U[up.bound_transport_neu_matrix_key])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "nf", nf)


def case_geometry(name, kind, seed, amp=0.3):
    """``Grid.compute_geometry`` (grids/grid.py:362-778) of a 3-D grid whose nodes -- ALL of them, so the
    faces of the hexahedra are warped -- were displaced: topology with the face-node loops in the
    reference's own order, nodes, and the five geometry arrays the reference computes.  ``poly3d``: the agglomerated
    polyhedra of ``make_dual_golden`` (up to 32 faces, faces of 4, 8 and 10 nodes), displaced like the rest."""
    rng = np.random.default_rng(seed)
    if kind == "poly3d":
        from make_dual_golden import poly3d
        g = poly3d(rng)
    elif kind == "cart3d":
        g = pp.CartGrid([5, 4, 3], [1.0, 0.8, 0.6])
    elif kind == "tet3d":
        g = pp.StructuredTetrahedralGrid([3, 2, 2], [1.0, 1.0, 1.0])
    else:
        pts = rng.random((3, 30))
        corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [0, 0, 1], [1, 0, 1],
                            [0, 1, 1], [1, 1, 1]], float).T
        g = pp.TetrahedralGrid(np.hstack((corners, pts)))
    g.compute_geometry()
    if kind != "delaunay":
        h = np.min(g.cell_volumes) ** (1.0 / 3)
        g.nodes += amp * h * (0.5 - rng.random(g.nodes.shape))
        g.compute_geometry()
    fn = g.face_nodes                      # NOT re-created / sorted: the loop order is part of the input
    cf = sps.csc_matrix(g.cell_faces)
    cf.sort_indices()
    d = dict(dim=np.int64(3), name=np.array(str(g.name)), nodes=g.nodes,
             fn_indptr=fn.indptr.astype(np.int32), fn_indices=fn.indices.astype(np.int32),
             cf_indptr=cf.indptr.astype(np.int32), cf_indices=cf.indices.astype(np.int32),
             cf_data=cf.data.astype(np.int8), face_normals=g.face_normals, face_centers=g.face_centers,
             face_areas=g.face_areas, cell_centers=g.cell_centers, cell_volumes=g.cell_volumes,
             fracture_faces=np.asarray(g.tags["fracture_faces"], bool), kind=np.array("geometry"))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, g.num_cells, "cells")


def case_diff_tpfa(name, kind, seed):
    """``DifferentiableTpfa`` (numerics/fv/tpfa.py:281-760): its helper matrices on one grid, and the AD evaluation
    of the face transmissibilities the reference builds from them (constitutive_laws.py:1544-1583) with the
    permeability as the independent AD variable: value, Jacobian dT_f/dk_c and the half-face values."""
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc = g.num_cells
    d = grid_arrays(g)
    d["kind"] = np.array("diff_tpfa")
    d["tip_faces"] = np.asarray(g.tags["tip_faces"], bool)
    d["domain_boundary_faces"] = np.asarray(g.tags["domain_boundary_faces"], bool)
    # a full SPD tensor per cell, 9 values per cell, cell-major (the layout of the reference's k_c vector)
    q = rng.standard_normal((nc, 3, 3))
    kt = np.einsum("cij,ckj->cik", q, q) + 0.5 * np.eye(3)
    k_val = kt.reshape(-1)
    d["k_c"] = k_val
    dt = pp.numerics.fv.tpfa.DifferentiableTpfa()
    sds = [g]
    n, d_vec, dist = dt.half_face_geometry_matrices(sds)
    put_matrix(d, "n", n)
    put_matrix(d, "d_vec", d_vec)
    d["dist"] = dist
    put_matrix(d, "hf_to_f_signed", dt.half_face_map(sds, to_entity="faces", with_sign=True))
    put_matrix(d, "c_to_hf", dt.half_face_map(sds, to_entity="half_faces", from_entity="cells"))
    put_matrix(d, "c3_to_hf3", dt.half_face_map(sds, from_entity="cells", to_entity="half_faces", dimensions=(3, 3)))
    put_matrix(d, "hf3_to_f", dt.half_face_map(sds, from_entity="half_faces", to_entity="faces", dimensions=(1, 3), with_sign=True))
    put_matrix(d, "face_pairing", dt.face_pairing_from_cell_array(sds))
    put_matrix(d, "nd_to_3d_cells_2", dt.nd_to_3d(sds, 2))
    put_matrix(d, "nd_to_3d_faces_3", dt.nd_to_3d(sds, 3, "faces"))
    d["boundary_sign"] = np.asarray(dt.boundary_sign(sds)._values, float)
    d["internal_boundary_filter"] = np.asarray(dt.internal_boundary_filter(sds)._values, float)
    d["tip_filter"] = np.asarray(dt.tip_filter(sds)._values, float)
    # the AD chain of constitutive_laws.py:1559-1581 on AdArrays
    d_n_by_dist = sps.diags(1 / dist) * d_vec @ n
    k = pp.ad.AdArray(k_val, sps.identity(9 * nc, format="csr"))
    hf_to_f = dt.half_face_map(sds, to_entity="faces", with_sign=True)
    t_hf_inv = 1.0 / (sps.csr_matrix(d_n_by_dist) @ k)
    T = 1.0 / (sps.csr_matrix(hf_to_f) @ t_hf_inv)
    d["t_hf"] = 1.0 / t_hf_inv.val
    d["T_f"] = T.val
    put_matrix(d, "dT_dk", T.jac)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, nc, "cells")


def case_mdg(prefix, seed):
    """A mixed-dimensional fracture network (BASELINE configs[1] / [4] in miniature): a 6 x 6 x 6 Cartesian matrix cut by
    three grid-aligned fractures (``pp.meshing.cart_grid``) -> one 3-D grid with split faces / nodes along the
    fractures, three 2-D fracture planes, six 1-D intersection lines and one 0-D point.  One fixture per subdomain:
    the flux discretization (``pp.Mpfa`` with ``ambient_dimension = 3``; TPFA on the lines, mpfa.py:690-712) with
    the fracture / tip faces as internal Neumann boundaries; the 3-D grid also gets ``pp.Mpsa``."""
    rng = np.random.default_rng(seed)
    f1 = np.array([[2, 2, 2, 2], [1, 5, 5, 1], [1, 1, 5, 5]], float)
    f2 = np.array([[1, 5, 5, 1], [3, 3, 3, 3], [1, 1, 5, 5]], float)
    f3 = np.array([[1, 5, 5, 1], [1, 1, 5, 5], [2, 2, 2, 2]], float)
    mdg = pp.meshing.cart_grid([f1, f2, f3], nx=np.array([6, 6, 6]), physdims=np.array([6.0, 6.0, 6.0]))
    mdg.compute_geometry()
    for i, g in enumerate(mdg.subdomains()):
        if g.dim == 0:
            continue
        nc = g.num_cells
        k = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                                 0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
        bf = g.get_boundary_faces()                       # domain boundary only; fracture / tip faces stay Neumann
        x = g.face_centers[0, bf]
        bc = pp.BoundaryCondition(g, bf[(x < 1e-10) | (x > 6 - 1e-10)], "dir")
        data = pp.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc, "mpfa_inverter": "python",
                                                "ambient_dimension": 3})
        pp.Mpfa("flow").discretize(g, data)
        M = data[pp.DISCRETIZATION_MATRICES]["flow"]
        d = grid_arrays(g)
        d.update(kind=np.array("mpfa"), K=k.values, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
                 bc_is_internal=bc.is_internal, bc_robin_weight=np.asarray(bc.robin_weight, float),
                 ambient_dimension=np.int64(3), tip_faces=np.asarray(g.tags["tip_faces"], bool),
                 domain_boundary_faces=np.asarray(g.tags["domain_boundary_faces"], bool),
                 eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
        for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face", "vector_source",
                    "bound_pressure_vector_source"):
            put_matrix(d, key, M[key])
        name = f"{prefix}_flow_sd{i:02d}_dim{g.dim}"
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
        print(name, "nc", nc, "nf", g.num_faces, "fracture faces", int(g.tags["fracture_faces"].sum()))
        if g.dim == 3:
            C = pp.FourthOrderTensor(np.exp(0.4 * rng.standard_normal(nc)), np.exp(0.4 * rng.standard_normal(nc)))
            vbc = pp.BoundaryConditionVectorial(g, bf[g.face_centers[2, bf] < 1e-10], "dir")
            dm = pp.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": vbc, "mpsa_inverter": "python"})
            pp.Mpsa("mech").discretize(g, dm)
            Mm = dm[pp.DISCRETIZATION_MATRICES]["mech"]
            e = grid_arrays(g)
            e.update(kind=np.array("mpsa"), C=C.values, bc_is_dir=vbc.is_dir, bc_is_neu=vbc.is_neu, bc_is_rob=vbc.is_rob,
                     bc_is_internal=vbc.is_internal, bc_robin_weight=np.asarray(vbc.robin_weight, float),
                     eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
            for key in ("stress", "bound_stress", "bound_displacement_cell", "bound_displacement_face"):
                put_matrix(e, key, Mm[key])
            name = f"{prefix}_mech_sd{i:02d}_dim3"
            np.savez_compressed(os.path.join(OUT, name + ".npz"), **e)
            print(name, "nc", nc)


def case_mpsa(name, kind, robin, seed, biot=False, basis=False):
    rng = np.random.default_rng(seed)
    g = make_grid(kind, rng)
    nc = g.num_cells
    mu = np.exp(0.5 * rng.standard_normal(nc))
    lam = np.exp(0.5 * rng.standard_normal(nc))
    C = pp.FourthOrderTensor(mu, lam)
    bc = vector_bc(g, rng, robin)
    if basis:  # boundary conditions in a rotated frame, a different rotation on every face
        nd = g.dim
        B = np.zeros((nd, nd, g.num_faces))
        for f in range(g.num_faces):
            q, r = np.linalg.qr(rng.standard_normal((nd, nd)))
            B[:, :, f] = q * np.sign(np.diag(r))
        bc.basis = B
    params = {"fourth_order_tensor": C, "bc": bc, "inverter": "python"}
    d = grid_arrays(g)
    if biot:
        at = pp.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                                  0.2 * rng.random(nc), 0.2 * rng.random(nc), 0.2 * rng.random(nc))
        params["scalar_vector_mappings"] = {"flow": at, "temp": 0.5}
        d["alpha__flow"] = at.values
        d["alpha__temp"] = np.float64(0.5)
    data = pp.initialize_data({}, "mech", params)
    discr = pp.Biot("mech") if biot else pp.Mpsa("mech")
    discr.discretize(g, data)
    M = data[pp.DISCRETIZATION_MATRICES]["mech"]
    d.update(kind=np.array("biot" if biot else "mpsa"), C=C.values, mu=mu, lmbda=lam,
             bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=bc.is_internal, bc_robin_weight=np.asarray(bc.robin_weight, float),
             bc_basis=np.asarray(bc.basis, float), eta=np.float64(pp.numerics.fv._fvutils.determine_eta(g)))
    for key in ("stress", "bound_stress", "bound_displacement_cell", "bound_displacement_face"):
        put_matrix(d, key, M[key])
    if biot:
        for key in ("displacement_divergence", "boundary_displacement_divergence",
                    "scalar_gradient", "mpsa_consistency", "bound_displacement_pressure"):
            for ak in ("flow", "temp"):
                put_matrix(d, f"{key}:{ak}", M[key][ak])
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "nc", nc, "nf", g.num_faces)


def main():
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1] if len(sys.argv) > 1 else ""   # optional fixture-name prefix
    cases = [
        (case_mpfa, ("mpfa_cart3d", "cart3d", False, 1), {}),
        (case_mpfa, ("mpfa_cart3d_robin", "cart3d", True, 2), {}),
        (case_mpfa, ("mpfa_cart3d_pert", "cart3d_pert", False, 3), {}),
        (case_mpfa, ("mpfa_cart3d_contrast", "cart3d", False, 4), {"contrast": True}),
        (case_mpfa, ("mpfa_tet3d_robin", "tet3d", True, 5), {}),
        (case_mpfa, ("mpfa_tet3d_delaunay", "tet3d_delaunay", False, 6), {}),
        (case_mpfa, ("mpfa_cart2d", "cart2d", True, 7), {}),
        (case_mpfa, ("mpfa_tri2d", "tri2d", False, 8), {}),
        (case_mpsa, ("mpsa_cart3d", "cart3d", False, 11), {}),
        (case_mpsa, ("mpsa_cart3d_robin", "cart3d", True, 12), {}),
        (case_mpsa, ("mpsa_cart3d_pert", "cart3d_pert", False, 13), {}),
        (case_mpsa, ("mpsa_tet3d", "tet3d", False, 14), {}),
        (case_mpsa, ("mpsa_tet3d_delaunay", "tet3d_delaunay_small", False, 15), {}),
        (case_mpsa, ("mpsa_cart2d_robin", "cart2d", True, 16), {}),
        (case_mpsa, ("mpsa_tri2d", "tri2d", False, 17), {}),
        (case_mpsa, ("biot_cart3d", "cart3d", False, 21), {"biot": True}),
        (case_mpsa, ("biot_tet3d_robin", "tet3d", True, 22), {"biot": True}),
        (case_mpsa, ("biot_cart2d", "cart2d", False, 23), {"biot": True}),
        # fracture planes: 2-D grids embedded in 3-D (prefix keeps them out of the "mpfa_*" sweeps)
        (case_mpfa_embedded, ("embedded_tri2d_tilted", "tri2d", 31, True), {}),
        (case_mpfa_embedded, ("embedded_cart2d_tilted", "cart2d", 32, True), {}),
        (case_mpfa_embedded, ("embedded_cart2d_xy", "cart2d", 33, False), {}),
        # vectorial boundary conditions in rotated bases (prefix keeps them out of the mpsa_/biot_ sweeps)
        (case_mpsa, ("rotbasis_mpsa_cart3d", "cart3d", True, 51), {"basis": True}),
        (case_mpsa, ("rotbasis_biot_tet3d", "tet3d", True, 52), {"biot": True, "basis": True}),
        (case_mpsa, ("rotbasis_mpsa_cart2d", "cart2d", True, 53), {"basis": True}),
        # next scope row (TPFA, upwinding): fixtures for oracle/next_rows_oracle.py
        (case_next_rows, ("next_cart3d", "cart3d_pert", 41), {}),
        (case_next_rows, ("next_tet3d", "tet3d", 42), {}),
        (case_next_rows, ("next_tri2d", "tri2d", 43), {}),
        # mixed-dimensional fracture network, one fixture per subdomain (prefix "mdgnet")
        (case_mdg, ("mdgnet", 91), {}),
        # DifferentiableTpfa (prefix "difftpfa")
        (case_diff_tpfa, ("difftpfa_cart3d", "cart3d_pert", 81), {}),
        (case_diff_tpfa, ("difftpfa_tet3d", "tet3d_delaunay", 82), {}),
        (case_diff_tpfa, ("difftpfa_tri2d", "tri2d", 83), {}),
        # Grid.compute_geometry (prefix "geom")
        (case_geometry, ("geom_cart3d_warped", "cart3d", 71), {}),
        (case_geometry, ("geom_tet3d_perturbed", "tet3d", 72), {}),
        (case_geometry, ("geom_tet3d_delaunay", "delaunay", 73), {}),
        # displaced by 0.1 h: at 0.3 h the reference finds negative sub-tetrahedra in these cells
        (case_geometry, ("geom_poly3d", "poly3d", 74), {"amp": 0.1}),
        # a 1-D intersection line (prefix "line")
        (case_line, ("line1d_tilted", 44), {}),
        # the reference's in-place partial update (prefix "partial")
        (case_partial_update, ("partial_mpfa_cart3d", "cart3d_pert", 61), {}),
        (case_partial_update, ("partial_mpfa_tet3d", "tet3d", 62), {}),
        (case_partial_update, ("partial_mpsa_cart3d", "cart3d_pert", 63), {"mech": True}),
        (case_partial_update, ("partial_mpsa_tet3d", "tet3d", 64), {"mech": True}),
    ]
    for fn, args, kw in cases:
        if args[0].startswith(only):
            fn(*args, **kw)


if __name__ == "__main__":
    main()
