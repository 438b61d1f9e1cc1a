"""The local-solver classes the dispatcher (build_classes, porepy_b200/csrc/api.cu) produces, reached end to end
through a whole discretization and compared with the oracle at the 1e-10 bar of test_gpu_parity.py.  The class of
each node is read back with DevicePlan.class_counts: {(solver configuration, A in global memory): nodes}.

On structured tetrahedra an interior MPSA node has 36 sub-faces (n = 108) and 24 sub-cells, so its row width is
W = (108 + 72 + 24 * n_alpha) | 1: 181 (MPSA, cfg 4, or cfg 7 with POREB200_CFG4=reg), 253 with 3 coupling
tensors (cfg 5 at the top of its width range) and 277 with 4 (cfg 6; 108 x 277 doubles do not fit shared memory)."""
import numpy as np
import pytest

import porepy_b200 as pb
from cases import flatten, load_case, max_rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-10

REACHED = {"mpfa": {}, "mpsa": {}}   # (cfg, a_global) -> nodes, over the cases of this module


def _record(g, kind):
    counts = pb.DevicePlan.for_grid(g).class_counts(kind)
    for key, v in counts.items():
        REACHED[kind][key] = REACHED[kind].get(key, 0) + v
    print(f"\n{kind} classes {sorted(counts.items())}")
    return counts


def _fresh(g):
    if hasattr(g, "_b200_plan"):
        del g._b200_plan
    return g


def _mixed_vector_bc(g):
    bf = g.get_all_boundary_faces()
    bc = pb.BoundaryConditionVectorial(g)
    bot = bf[g.face_centers[2, bf] < 1e-10]
    bc.is_dir[:, bot] = True
    bc.is_neu[:, bot] = False
    return bc


def _aniso(nc, rng):
    return pb.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                                0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))


def _biot(g, n_alpha, seed):
    from oracle import fv_oracle as fo
    rng = np.random.default_rng(seed)
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))
    bc = _mixed_vector_bc(g)
    maps = {f"a{q}": (_aniso(nc, rng) if q % 2 == 0 else 0.5 + 0.1 * q) for q in range(n_alpha)}
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc, "scalar_vector_mappings": maps})
    pb.Biot("mech").discretize(g, data)
    ref = flatten(fo.mpsa(g, C.values, bc, pb.determine_eta(g),
                          alpha={k: (v.values if hasattr(v, "values") else v) for k, v in maps.items()}))
    err, key = max_rel_err(ref, data[pb.DISCRETIZATION_MATRICES]["mech"])
    assert err < TOL, (key, err)
    return _record(g, "mpsa")


def test_biot_three_coupling_tensors_tet_reaches_cfg5_top_width():
    counts = _biot(_fresh(pb.structured_tet_grid([3, 3, 3])), 3, 21)
    assert counts.get((5, True), 0) + counts.get((5, False), 0) > 0, counts


def test_biot_four_coupling_tensors_tet_reaches_cfg6_global():
    counts = _biot(_fresh(pb.structured_tet_grid([3, 3, 3])), 4, 22)
    assert counts.get((6, True), 0) > 0, counts


def test_five_coupling_tensors_raise():
    g = pb.structured_tet_grid([2, 2, 2])
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.ones(nc), np.ones(nc))
    bc = _mixed_vector_bc(g)
    maps = {f"a{q}": 0.5 + 0.1 * q for q in range(5)}
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc, "scalar_vector_mappings": maps})
    with pytest.raises(NotImplementedError, match="at most 4 coupling tensors"):
        pb.Biot("mech").discretize(g, data)


def test_mpsa_tet_register_solver_cfg7(monkeypatch):
    from oracle import fv_oracle as fo
    monkeypatch.setenv("POREB200_CFG4", "reg")
    g = pb.structured_tet_grid([3, 3, 3])     # a fresh grid: classes are built once per plan and n_alpha
    rng = np.random.default_rng(23)
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))
    bc = _mixed_vector_bc(g)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc})
    pb.Mpsa("mech").discretize(g, data)
    ref = fo.mpsa(g, C.values, bc, pb.determine_eta(g))
    err, key = max_rel_err(ref, data[pb.DISCRETIZATION_MATRICES]["mech"])
    assert err < TOL, (key, err)
    counts = _record(g, "mpsa")
    assert counts.get((7, False), 0) > 0 and (4, False) not in counts, counts


def test_mpsa_delaunay_fixture():
    from oracle import fv_oracle as fo
    c = load_case("mpsa_tet3d_delaunay")
    g = _fresh(c.g)
    C = pb.FourthOrderTensor.from_values(c.raw["C"])
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": c.bc, "mpsa_eta": c.eta})
    pb.Mpsa("mech").discretize(g, data)
    ref = fo.mpsa(g, C.values, c.bc, c.eta)
    err, key = max_rel_err(ref, data[pb.DISCRETIZATION_MATRICES]["mech"])
    assert err < TOL, (key, err)
    _record(g, "mpsa")


def test_mpfa_and_mpsa_small_meshes():
    """MPFA on hexahedra and tetrahedra, MPSA / Biot on hexahedra: the smaller configurations."""
    from oracle import fv_oracle as fo
    rng = np.random.default_rng(24)
    for g in (pb.cart_grid_3d([4, 4, 3], perturb=0.2, seed=4), pb.structured_tet_grid([3, 3, 2])):
        k = _aniso(g.num_cells, rng)
        bf = g.get_all_boundary_faces()
        bc = pb.BoundaryCondition(g, bf, list(np.where(g.face_centers[0, bf] < 1e-10, "dir", "neu")))
        data = pb.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc})
        pb.Mpfa("flow").discretize(g, data)
        err, key = max_rel_err(fo.mpfa(g, k.values, bc, pb.determine_eta(g)), data[pb.DISCRETIZATION_MATRICES]["flow"])
        assert err < TOL, (key, err)
        _record(g, "mpfa")
    g = _fresh(pb.cart_grid_3d([4, 4, 3], perturb=0.2, seed=6))
    _biot(g, 1, 25)
    g = _fresh(pb.cart_grid_3d([4, 4, 3], perturb=0.2, seed=7))
    from oracle import fv_oracle as fo  # noqa: F811
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))
    bc = _mixed_vector_bc(g)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc})
    pb.Mpsa("mech").discretize(g, data)
    err, key = max_rel_err(fo.mpsa(g, C.values, bc, pb.determine_eta(g)), data[pb.DISCRETIZATION_MATRICES]["mech"])
    assert err < TOL, (key, err)
    _record(g, "mpsa")


# Classes the size rules produce on the meshes above.  Not reached: cfg 5 with A in shared memory (on structured
# tetrahedra the MPSA rest of a cfg-5 node pushes A to global memory), and cfg 6 with A in shared memory.  That needs an MPSA
# node with n = 3 * nsf > 112 (nsf >= 38 sub-faces) whose A, solver scratch and the rest fit 227 KB, e.g. nsf = 38,
# nsc = 26 on tetrahedra: 114 x 193 doubles of A plus ~4.9k of the rest, ~27k of 29k doubles.  Such nodes occur on
# unstructured tetrahedral meshes, but not on the structured meshes here or the 70-cell Delaunay fixture.
EXPECTED = {(0, False), (1, False), (2, False), (3, False), (4, False), (5, True), (6, True), (7, False)}


def test_every_class_is_reached():
    got = set(REACHED["mpfa"]) | set(REACHED["mpsa"])
    print(f"\nreached: mpfa {sorted(REACHED['mpfa'].items())}  mpsa {sorted(REACHED['mpsa'].items())}")
    assert EXPECTED <= got, sorted(EXPECTED - got)
