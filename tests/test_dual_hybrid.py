"""Hybridization of the mixed schemes (csrc/dual_hybrid.cuh): ``pb.HybridDualVEM`` (reference numerics/vem/hybrid.py)
against the ``hybrid_*`` golden fixtures of the unmodified reference (tools/make_hybrid_golden.py), and
``MVEM.solve`` / ``RT0.solve`` against a direct solve of the saddle-point system, on the host build of the lane
routines (tests/emu_dual_hybrid.py, with a direct solve of the face system) and on the GPU (fused Jacobi BiCGStab)."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200 import fv
import dual_mp
from emu_dual_hybrid import EmuHybridDualGrid
from golden_io import case_names, load_case, rel_err

HYBRID = case_names("hybrid_")
DUAL = case_names("dual_")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class CachedEmuDualGrid(EmuHybridDualGrid):
    """The host build kept on the grid as ``fv.DualGrid.for_grid`` keeps the device handle, so that ``solve`` finds
    the discretization it belongs to."""

    @classmethod
    def for_grid(cls, sd):
        dg = getattr(sd, "_b200_dual", None)
        if not isinstance(dg, cls) or dg.fingerprint != fv.DevicePlan._fingerprint(sd, sd.cell_faces, sd.face_nodes):
            dg = cls(sd)
            sd._b200_dual = dg
        return dg


@pytest.fixture
def host_build(monkeypatch):
    monkeypatch.setattr(fv, "DualGrid", CachedEmuDualGrid)


def direct(H, rhs):
    """Stand-in for the face system's Krylov solve on the host build: a direct solve of the ``HostCsr`` (or of the
    scipy matrix ``HybridDualVEM.matrix_rhs`` returns)."""
    return spla.spsolve(sps.csc_matrix(H.to_scipy() if hasattr(H, "to_scipy") else H), rhs)


def _hybrid_data(c):
    params = {"second_order_tensor": pb.SecondOrderTensor.from_values(c.raw["K"]), "bc": c.bc,
              "bc_values": c.raw["bc_values"], "source": c.raw["source"], "aperture": c.raw["aperture"]}
    return pb.initialize_data({}, "flow", params)


def _dual_data(c):
    params = {"second_order_tensor": pb.SecondOrderTensor.from_values(c.raw["K"]), "bc": c.bc,
              "bc_values": c.raw["bc_values"], "vector_source": c.raw["vector_source"]}
    return pb.initialize_data({}, "flow", params)


def _discr(c):
    return {"mvem": pb.MVEM, "rt0": pb.RT0}[c.kind]("flow")


def _check_hybrid(c, H, rhs, tol):
    assert rel_err(c.mats["H"], H) <= tol, (c.name, rel_err(c.mats["H"], H))
    ref = c.raw["rhs"]
    assert np.abs(rhs - ref).max() <= tol * np.abs(ref).max(), c.name
    keep = ~np.asarray(c.bc.is_dir, bool)   # symmetric apart from the Dirichlet rows
    Hk = sps.csr_matrix(H)[keep][:, keep]
    assert abs(Hk - Hk.T).max() <= 1e-12 * abs(Hk).max(), c.name


def test_fixtures_cover_the_cases():
    assert {f"hybrid_{k}" for k in ("line", "line_tilted", "cart2d", "tri2d_sheared", "plane_tilted", "cart3d_pert",
                                    "tet3d_delaunay", "poly2d", "poly3d")} <= set(HYBRID)
    apertures = 0
    for name in HYBRID:
        c = load_case(name)
        assert c.bc.is_dir.any() and c.bc.is_neu.any() and np.abs(c.raw["source"]).max() > 0
        apertures += bool(np.any(c.raw["aperture"] != 1))
    assert apertures >= 2


@pytest.mark.parametrize("name", HYBRID)
def test_hybrid_goldens_on_the_host_build(name, host_build):
    c = load_case(name)
    d = pb.HybridDualVEM("flow")
    H, rhs = d.matrix_rhs(c.g, _hybrid_data(c))
    _check_hybrid(c, H, rhs, 1e-12)
    assert d.ndof(c.g) == c.g.num_faces


def test_point_grid_gets_the_identity():
    from porepy_b200.grid import Grid
    g = Grid(0, np.zeros((3, 1)), sps.csc_matrix((0, 0)), sps.csc_matrix((0, 1)), name="PointGrid")
    H, rhs = pb.HybridDualVEM("flow").matrix_rhs(g, pb.initialize_data({}, "flow", {}))
    assert H.shape == (0, 0) and np.array_equal(rhs, np.zeros(1))


def _assembled(d, g, data):
    """assemble_matrix_rhs, then the discretization again: the host build assembles with the host formulas, which
    download the stored matrices (the device assembly downloads nothing, and the values repeat bit for bit)."""
    A, b = d.assemble_matrix_rhs(g, data)
    d.discretize(g, data)
    return A, b


def _seeded_b(c, d, data, seed=5):
    """The right-hand side of assemble_matrix_rhs with a seeded source added to the cell rows."""
    A, b = _assembled(d, c.g, data)
    b = b.copy()
    b[c.g.num_faces:] += np.random.default_rng(seed).standard_normal(c.g.num_cells)
    return A, b


def _check_solve(c, linear_solver, tol):
    data = _dual_data(c)
    d = _discr(c)
    d.discretize(c.g, data)
    A, b = _seeded_b(c, d, data)
    up = d.solve(c.g, data, b, linear_solver=linear_solver)
    ref = spla.spsolve(sps.csc_matrix(A.device_csr.to_scipy() if getattr(A, "device_csr", None) else A), b)
    assert np.abs(up - ref).max() <= tol * np.abs(ref).max(), (c.name, np.abs(up - ref).max() / np.abs(ref).max())
    return d


@pytest.mark.parametrize("name", DUAL)
def test_solve_matches_the_saddle_point_on_the_host_build(name, host_build):
    _check_solve(load_case(name), direct, 1e-9)


def tutorial_sum_p(linear_solver=None):
    """flux_discretizations.ipynb cells 33-37 through ``solve``: sum(p) of the MVEM tutorial."""
    g = pb.cart_grid_2d([20, 20], [1, 1])
    b_faces = g.tags["domain_boundary_faces"].nonzero()[0]
    bc = pb.BoundaryCondition(g, b_faces, ["dir"] * b_faces.size)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(g.num_cells)),
                                           "source": g.cell_volumes, "bc": bc, "bc_values": np.zeros(g.num_faces)})
    d = pb.MVEM("flow")
    d.discretize(g, data)
    _, b = _assembled(d, g, data)
    b = b + np.concatenate((np.zeros(g.num_faces), -g.cell_volumes))
    up = d.solve(g, data, b, linear_solver=linear_solver)
    return np.sum(d.extract_pressure(g, up, data)), d


def test_tutorial_through_solve_on_the_host_build(host_build):
    s, _ = tutorial_sum_p(direct)
    assert np.isclose(s, 14.348068220560325, rtol=1e-12, atol=0)


def linear_pressure_problem(g, method):
    """K = I, Dirichlet data from p(x) = a . x + p0 on the whole boundary: both schemes reproduce p at the cell
    centres and the flux u = -grad p . n area exactly."""
    a, p0 = np.array([0.7, -1.3, 0.4])[:g.dim], 0.25
    rot = fv.dual_frame(g)
    a3 = rot[:g.dim].T @ a       # the gradient in the ambient space, tangential to the grid
    bf = g.get_all_boundary_faces()
    bc = pb.BoundaryCondition(g, bf, ["dir"] * bf.size)
    bcv = np.zeros(g.num_faces)
    bcv[bf] = a3 @ g.face_centers[:, bf] + p0
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(g.num_cells)),
                                           "bc": bc, "bc_values": bcv})
    d = {"mvem": pb.MVEM, "rt0": pb.RT0}[method]("flow")
    d.discretize(g, data)
    _, b = _assembled(d, g, data)
    return d, data, b, a3 @ g.cell_centers + p0, -(a3 @ g.face_normals)


def check_linear_pressure(g, method, linear_solver, accuracy, **kw):
    d, data, b, p_ref, u_ref = linear_pressure_problem(g, method)
    up = d.solve(g, data, b, linear_solver=linear_solver, **kw)
    u, p = up[:g.num_faces], up[g.num_faces:]
    assert np.abs(p - p_ref).max() <= accuracy * np.abs(p_ref).max(), (method, np.abs(p - p_ref).max())
    assert np.abs(u - u_ref).max() <= accuracy * np.abs(u_ref).max(), (method, np.abs(u - u_ref).max())
    return d


@pytest.mark.parametrize("name", ["dual_mvem_cart3d_pert", "dual_mvem_tri2d_sheared", "dual_rt0_tet3d_delaunay",
                                  "dual_rt0_tri2d_sheared", "dual_mvem_line_tilted", "dual_mvem_plane_tilted",
                                  "dual_mvem_poly2d", "dual_mvem_poly3d", "dual_mvem_poly_plane_tilted"])
def test_linear_pressure_is_exact_on_the_host_build(name, host_build):
    c = load_case(name)
    check_linear_pressure(c.g, c.kind, direct, 1e-10)


def _up_pair(c, linear_solver):
    """The hybrid solution through compute_up and the MVEM saddle point of the same problem (the class docstring's
    mapping): aperture 1, a tensor the frame leaves unchanged (isotropic per cell), Dirichlet and Neumann faces."""
    g = c.g
    kxx = 10.0 ** np.random.default_rng(3).random(g.num_cells)
    K = pb.SecondOrderTensor(kxx)
    bc = pb.BoundaryCondition(g, np.flatnonzero(c.bc.is_dir | c.bc.is_neu),
                              ["dir" if x else "neu" for x in c.bc.is_dir[c.bc.is_dir | c.bc.is_neu]])
    bcv, f = c.raw["bc_values"], c.raw["source"]
    hyb = pb.initialize_data({}, "flow", {"second_order_tensor": K, "bc": bc, "bc_values": bcv, "source": f,
                                          "aperture": np.ones(g.num_cells)})
    h = pb.HybridDualVEM("flow")
    H, rhs = h.matrix_rhs(g, hyb)
    u_h, p_h = h.compute_up(g, linear_solver(H, rhs), hyb)
    cf = sps.csc_matrix(g.cell_faces)
    faces, first = np.unique(cf.indices, return_index=True)
    sign = np.zeros(g.num_faces)
    sign[faces] = cf.data[first]
    mv_bcv = np.where(bc.is_neu, sign * bcv * g.face_areas, bcv)
    mv = pb.initialize_data({}, "flow", {"second_order_tensor": K, "bc": bc, "bc_values": mv_bcv})
    d = pb.MVEM("flow")
    d.discretize(g, mv)
    A, b = d.assemble_matrix_rhs(g, mv)
    b = b + np.concatenate((np.zeros(g.num_faces), -f))
    A = A.device_csr.to_scipy() if getattr(A, "device_csr", None) else A
    up = spla.spsolve(sps.csc_matrix(A), b)
    return u_h, p_h, up[:g.num_faces], up[g.num_faces:]


@pytest.mark.parametrize("name", ["hybrid_cart2d", "hybrid_tri2d_sheared", "hybrid_cart3d_pert",
                                  "hybrid_tet3d_delaunay", "hybrid_line", "hybrid_poly2d", "hybrid_poly3d"])
def test_compute_up_matches_the_mvem_saddle_point_on_the_host_build(name, host_build):
    u_h, p_h, u, p = _up_pair(load_case(name), direct)
    assert np.abs(p_h - p).max() <= 1e-10 * np.abs(p).max()
    assert np.abs(u_h - u).max() <= 1e-10 * np.abs(u).max()


def test_refusals(host_build):
    c = load_case("dual_mvem_cart3d")
    g = c.g
    d = pb.MVEM("flow")
    # no Dirichlet and no Robin face: singular
    bf = g.get_all_boundary_faces()
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(g.num_cells)),
                                           "bc": pb.BoundaryCondition(g, bf, ["neu"] * bf.size),
                                           "bc_values": np.zeros(g.num_faces)})
    d.discretize(g, data)
    _, b = _assembled(d, g, data)
    with pytest.raises(ValueError, match="no Dirichlet and no Robin"):
        d.solve(g, data, b, linear_solver=direct)
    # the stored matrices downloaded: no device-resident discretization
    data = _dual_data(c)
    d.discretize(g, data)
    _, b = d.assemble_matrix_rhs(g, data)
    data[pb.DISCRETIZATION_MATRICES]["flow"]["mass"].data
    with pytest.raises(ValueError, match="device-resident"):
        d.solve(g, data, b, linear_solver=direct)
    # RT0 on non-simplices is refused by its discretize, so no solve can follow
    with pytest.raises(ValueError, match="RT0 needs simplices"):
        pb.RT0("flow").discretize(g, _dual_data(c))
    # a cell with 33 faces (a polygon): one warp condenses at most 32
    from porepy_b200.grid import Grid
    t = 2 * np.pi * np.arange(33) / 33
    nodes = np.vstack((np.cos(t), np.sin(t), np.zeros(33)))
    fn = sps.csc_matrix((np.ones(66, bool), (np.r_[np.arange(33), (np.arange(33) + 1) % 33], np.r_[np.arange(33),
                                                                                               np.arange(33)])),
                        shape=(33, 33))
    g33 = Grid(2, nodes, fn, sps.csc_matrix(np.ones((33, 1))), name="polygon")
    x0, x1 = nodes, np.roll(nodes, -1, axis=1)
    g33.face_centers, g33.face_areas = (x0 + x1) / 2, np.linalg.norm(x1 - x0, axis=0)
    g33.face_normals = np.vstack(((x1 - x0)[1], -(x1 - x0)[0], np.zeros(33)))
    g33.cell_centers, g33.cell_volumes = np.zeros((3, 1)), np.array([16.5 * np.sin(t[1])])
    h = pb.HybridDualVEM("flow")
    hd = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(1)), "bc": None,
                                         "bc_values": np.zeros(33), "source": np.zeros(1), "aperture": np.ones(1)})
    assert np.diff(sps.csc_matrix(g33.cell_faces).indptr).max() > 32
    with pytest.raises(NotImplementedError, match="32"):
        h.matrix_rhs(g33, hd)


def test_reference_unit_tests_on_the_plugin_class():
    """The reference's own test_hybrid_vem.py with HybridDualVEM rebound to the plugin class (host build without a
    GPU): all pass, after passing on the stock class; matrix_rhs runs on the porepy_b200 path, none is handed over."""
    if not os.path.isdir("/root/reference/tests/numerics/vem"):
        pytest.skip("reference tree not present")
    tool = [os.sys.executable, os.path.join(ROOT, "tools", "run_reference_tests.py"), "numerics/vem/test_hybrid_vem.py"]
    stock = subprocess.run(tool + ["--stock"], capture_output=True, text=True, timeout=1200).stdout
    assert re.search(r"\b\d+ passed\b", stock) and " failed" not in stock, stock[-3000:]
    out = subprocess.run(tool, capture_output=True, text=True, timeout=1200).stdout
    n = re.search(r"\b(\d+) passed\b", out)
    assert n and " failed" not in out and n.group(1) == re.search(r"\b(\d+) passed\b", stock).group(1), out[-3000:]
    calls = re.search(r"HybridDualVEM\.matrix_rhs on the porepy_b200 path: (\d+)", out)
    assert calls and int(calls.group(1)) > 0, out[-3000:]
    assert "HybridDualVEM.matrix_rhs on the reference path" not in out, out[-3000:]
    assert "handed to the reference" not in out, out[-3000:]


def test_hybrid_kernels_do_not_spill():
    """Every instantiation of the hybridization kernels: no stack frame, no spills."""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(ROOT, "porepy_b200", "csrc", "dual.cu"), "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    blocks = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", out, re.S)
    names = [b[0] for b in blocks if "hybrid" in b[0]]
    assert sum("hybrid_cell_kernel" in n for n in names) == 6 and any("hybrid_bc_kernel" in n for n in names), out
    for name, stack, st, ld in blocks:
        if "hybrid" in name:
            assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", HYBRID)
def test_hybrid_goldens_on_the_gpu(name):
    c = load_case(name)
    d = pb.HybridDualVEM("flow")
    H, rhs = d.matrix_rhs(c.g, _hybrid_data(c))
    _check_hybrid(c, H, rhs, 1e-12)
    H2, rhs2 = d.matrix_rhs(c.g, _hybrid_data(c))
    assert np.array_equal(H.data, H2.data) and np.array_equal(rhs, rhs2)
    emu = EmuHybridDualGrid(c.g)
    geo, codes, values = d._inputs(c.g, _hybrid_data(c))
    He, rhse, _, _ = emu.hybrid_system(0, geo, codes, np.zeros(c.g.num_faces), c.g.face_areas, values)
    He = He.to_scipy()
    # entry by entry, each at the scale of its own cells (tests/dual_mp.py): kappa(A_c) max |E_c| for H, and for the
    # right-hand side and the recovery what the errors of E, z and S bring in
    R = dual_mp.HybridReference(c.g, geo, codes, values)
    assert dual_mp.worst(H.toarray(), He.toarray(), R.Hs)[0] <= dual_mp.HYBRID_TOL
    assert dual_mp.worst(rhs, rhse, R.rs)[0] <= dual_mp.HYBRID_TOL
    lam = spla.spsolve(sps.csc_matrix(H), rhs)
    u, p = d.compute_up(c.g, lam, _hybrid_data(c))
    upe, _ = emu.hybrid_recover(0, geo, codes, values, lam)
    _, ups = R.recover(lam)
    assert dual_mp.worst(np.concatenate((u, p)), upe, ups)[0] <= dual_mp.HYBRID_TOL


# Jacobi BiCGStab does not converge on the face system of dual_rt0_tet3d (a 2 x 2 x 2 tetrahedral grid with a 10^6
# permeability contrast): it stops at 5,000 iterations with a face residual of 51.  On dual_rt0_tet3d_delaunay it reaches
# the 1e-14 of the test in about two runs of three only: the dot products of the recurrence are summed with atomics, so
# the iterations differ from run to run, and the others stop at 5,000 iterations near 1e-9 or break down.  Measured on
# an H100 with bit-identical face systems, Jacobi diagonals and right-hand sides in every run.  Both face systems are
# right: a direct solve of them reproduces the saddle point (test_solve_matches_the_saddle_point_on_the_host_build).
GPU_SOLVE = [n for n in DUAL if n not in ("dual_rt0_tet3d", "dual_rt0_tet3d_delaunay")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SOLVE)
def test_solve_matches_the_saddle_point_on_the_gpu(name):
    from porepy_b200.sparse import LazyCsr
    c = load_case(name)
    data = _dual_data(c)
    d = _discr(c)
    d.discretize(c.g, data)
    A, b = _seeded_b(c, d, data)
    before = dict(LazyCsr.downloads)
    # the fixtures' 10^6 permeability contrast makes the face system ill-conditioned: a residual of 1e-10 leaves
    # errors near 1e-7, so the face system is solved to 1e-14 here
    up = d.solve(c.g, data, b, tol=1e-14)
    assert LazyCsr.downloads == before
    assert d.last_solve["converged"], d.last_solve
    ref = spla.spsolve(sps.csc_matrix(A.device_csr.to_scipy()), b)
    assert np.abs(up - ref).max() <= 1e-9 * np.abs(ref).max(), (name, np.abs(up - ref).max() / np.abs(ref).max())


@pytest.mark.gpu
def test_tutorial_through_solve_on_the_gpu():
    s, d = tutorial_sum_p()
    assert np.isclose(s, 14.348068220560325, rtol=1e-9, atol=0), s


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["mvem_tet", "rt0_tet", "mvem_cart"])
def test_bench_size(which):
    """998,250 tetrahedra (MVEM, RT0) and 100^3 hexahedra (MVEM): the solve converges, the true residual of the
    saddle-point system is at most 1e-8 |b|, and the linear pressure is reproduced to 1e-7."""
    import torch
    from porepy_b200.grid import cart_grid_3d, structured_tet_grid
    g = cart_grid_3d([100, 100, 100]) if which == "mvem_cart" else structured_tet_grid([55, 55, 55])
    method = which.split("_")[0]
    d, data, b, p_ref, u_ref = linear_pressure_problem(g, method)
    b = b.copy()
    b[g.num_faces:] += np.random.default_rng(9).standard_normal(g.num_cells) * g.cell_volumes
    A, _ = _assembled(d, g, data)
    up = d.solve(g, data, b, tol=1e-10)
    info = d.last_solve
    assert info["converged"], info
    r = b - (A.device_csr @ torch.as_tensor(up, device="cuda")).cpu().numpy()
    rel = np.linalg.norm(r) / np.linalg.norm(b)
    print(which, info, "true relative residual", rel)
    assert rel <= 1e-8, (which, rel, info)
    check_linear_pressure(g, method, None, 1e-7, tol=1e-10)
