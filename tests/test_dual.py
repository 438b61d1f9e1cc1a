"""Mixed (dual) discretizations of Darcy flow, ``pb.MVEM`` and ``pb.RT0`` (reference numerics/vem/mvem.py,
numerics/fem/rt0.py, numerics/vem/dual_elliptic.py): the per-(cell, face) routines of csrc/dual_cell.cuh on the host
build (tests/emu_dual.py) and on the GPU, against the ``dual_*`` golden fixtures of the unmodified reference
(tools/make_dual_golden.py), the MVEM part of the tutorial ``flux_discretizations.ipynb``, the refusals and the
compiler's register report."""
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
from emu_dual import EmuDualGrid
from golden_io import case_names, load_case, rel_err

CASES = case_names("dual_")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _data(c):
    params = {"second_order_tensor": pb.SecondOrderTensor.from_values(c.raw["K"]), "bc": c.bc,
              "bc_values": c.raw["bc_values"], "vector_source": c.raw["vector_source"]}
    return pb.initialize_data({}, "flow", params)


def _discr(c):
    return {"mvem": pb.MVEM, "rt0": pb.RT0}[c.kind]("flow")


def _check_case(c, data, A, b, tol):
    mats = data[pb.DISCRETIZATION_MATRICES]["flow"]
    for key in ("mass", "div", "vector_proj"):
        err = rel_err(c.mats[key], mats[key])
        assert err < tol, (c.name, key, err)
    err = rel_err(c.mats["A"], A)
    assert err < tol, (c.name, "A", err)
    ref_b = c.raw["b"]
    assert np.abs(b - ref_b).max() <= tol * np.abs(ref_b).max(), (c.name, "b")


@pytest.fixture
def host_build(monkeypatch):
    monkeypatch.setattr(fv, "DualGrid", EmuDualGrid)


def test_fixtures_cover_the_cases():
    names = set(CASES)
    for m, k in [("mvem", "cart2d"), ("mvem", "tri2d_sheared"), ("rt0", "tri2d_sheared"), ("mvem", "cart3d"),
                 ("mvem", "cart3d_pert"), ("mvem", "tet3d"), ("rt0", "tet3d"), ("mvem", "tet3d_delaunay"),
                 ("rt0", "tet3d_delaunay"), ("mvem", "line_tilted"), ("rt0", "line_tilted"), ("mvem", "plane_tilted"),
                 ("rt0", "tri_plane_tilted"), ("mvem", "poly2d"), ("mvem", "poly3d"),
                 ("mvem", "poly_plane_tilted")]:
        assert f"dual_{m}_{k}" in names
    for name in CASES:
        c = load_case(name)
        assert c.bc.is_dir.any() and c.bc.is_rob.any() and (c.g.dim == 1 or c.bc.is_neu.any())
        K = c.raw["K"]
        assert np.abs(K[0, 1]).max() > 0 and K[0, 0].max() / K[0, 0].min() > 1e4


@pytest.mark.parametrize("name", CASES)
def test_goldens_on_the_host_build(name, host_build):
    c = load_case(name)
    data = _data(c)
    d = _discr(c)
    d.discretize(c.g, data)
    A, b = d.assemble_matrix_rhs(c.g, data)
    _check_case(c, data, A, b, 1e-12)
    assert d.ndof(c.g) == c.g.num_cells + c.g.num_faces


def tutorial_problem():
    g = pb.cart_grid_2d([20, 20], [1, 1])
    perm = pb.SecondOrderTensor(np.ones(g.num_cells))
    b_faces = g.tags["domain_boundary_faces"].nonzero()[0]
    bc = pb.BoundaryCondition(g, b_faces, ["dir"] * b_faces.size)
    parameters = {"second_order_tensor": perm, "source": g.cell_volumes, "bc": bc,
                  "bc_values": np.zeros(g.num_faces)}
    return g, pb.initialize_data({}, "flow", parameters)


def tutorial_numbers():
    """flux_discretizations.ipynb cells 33-37: MVEM, the source as DualScalarSource writes it (-source in the cell
    rows), a direct solve, and the tutorial's three assertions."""
    g, data = tutorial_problem()
    d = pb.MVEM("flow")
    d.discretize(g, data)
    A, b_flow = d.assemble_matrix_rhs(g, data)
    b_rhs = np.concatenate((np.zeros(g.num_faces), -data[pb.PARAMETERS]["flow"]["source"]))
    up = spla.spsolve(sps.csc_matrix(A), b_flow + b_rhs)
    u, p = d.extract_flux(g, up, data), d.extract_pressure(g, up, data)
    P0u = d.project_flux(g, u, data)
    assert np.isclose(np.sum(p), 14.348068220560325)
    assert np.isclose(np.sum(u), 0)
    assert np.isclose(np.sum(P0u), 0)
    return up


def test_tutorial_on_the_host_build(host_build):
    tutorial_numbers()


def test_point_grid_gets_the_reference_matrices():
    from porepy_b200.grid import Grid
    g = Grid(0, np.zeros((3, 1)), sps.csc_matrix((0, 0)), sps.csc_matrix((0, 1)), name="PointGrid")
    data = pb.initialize_data({}, "flow", {})
    for cls in (pb.MVEM, pb.RT0):
        cls("flow").discretize(g, data)
        m = data[pb.DISCRETIZATION_MATRICES]["flow"]
        assert m["mass"].shape == (0, 0) and m["div"].shape == (0, 1) and m["vector_proj"].shape == (3, 0)


def test_refusals(host_build):
    c = load_case("dual_mvem_cart3d")
    with pytest.raises(ValueError, match="RT0 needs simplices"):
        pb.RT0("flow").discretize(c.g, _data(c))
    data = _data(c)
    data["is_tangential"] = True   # read by the reference on 1-D and 2-D grids only
    pb.MVEM("flow").discretize(c.g, data)
    c2 = load_case("dual_mvem_cart2d")
    data = _data(c2)
    data["is_tangential"] = True
    with pytest.raises(NotImplementedError):
        pb.MVEM("flow").discretize(c2.g, data)
    g = load_case("dual_mvem_cart3d").g
    g.periodic_face_map = np.zeros((2, 0), int)
    with pytest.raises(NotImplementedError):
        pb.MVEM("flow").discretize(g, _data(c))
    # face centres that do not close the cell's moments, as on a warped hexahedron: the reference's consistency test
    # allclose(G, F D) fails, and the error names the first failing cell
    g = load_case("dual_mvem_cart3d").g
    f = int(np.flatnonzero(np.diff(sps.csr_matrix(g.cell_faces).indptr) == 2)[0])
    cells = sps.csr_matrix(g.cell_faces)[f].indices
    g.face_centers[:, f] += 0.1
    with pytest.raises(AssertionError, match=f"cell {cells.min()}"):
        pb.MVEM("flow").discretize(g, _data(c))


def test_reference_unit_tests_on_the_plugin_classes():
    """The reference's own MVEM / RT0 tests with pp.MVEM / pp.RT0 rebound to the plugin classes (host build of the
    routines without a GPU): all pass, every discretize runs on the porepy_b200 path, none is handed over."""
    if not os.path.isdir("/root/reference/tests/numerics/vem"):
        pytest.skip("reference tree not present")
    out = subprocess.run([os.sys.executable, os.path.join(ROOT, "tools", "run_reference_tests.py"),
                          "numerics/vem/test_dual_vem.py", "numerics/vem/test_rt0.py"],
                         capture_output=True, text=True, timeout=1200).stdout
    assert re.search(r"\b51 passed\b", out) and " failed" not in out, out[-3000:]
    counts = {k: int(v) for k, v in re.findall(r"\[porepy_b200\] (\w+)\.discretize on the porepy_b200 path: (\d+)", out)}
    assert counts.get("MVEM", 0) > 0 and counts.get("RT0", 0) > 0, out[-3000:]
    assert "reference path: " not in out and "handed to the reference" not in out, out[-3000:]


def test_dual_kernels_do_not_spill():
    """Every instantiation of dual_kernel and the pattern kernel: no stack frame, no spills."""
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(ROOT, "porepy_b200", "csrc", "dual.cu"), "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    blocks = re.findall(r"Compiling entry function '(\w+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                        r"(\d+) bytes spill loads", out, re.S)
    names = [b[0] for b in blocks if "dual_kernel" in b[0]]
    assert len(names) == 6, out
    for name, stack, st, ld in blocks:
        if "dual" not in name and "pattern_kernel" not in name:
            continue   # cub's scan kernels
        assert (stack, st, ld) == ("0", "0", "0"), (name, stack, st, ld)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_goldens_on_the_gpu(name):
    c = load_case(name)
    data = _data(c)
    d = _discr(c)
    d.discretize(c.g, data)
    A, b = d.assemble_matrix_rhs(c.g, data)
    _check_case(c, data, A, b, 1e-12)
    # the device against the host build of the same routines, and bit-identical repeats
    emu = EmuDualGrid(c.g)
    geo_rot = fv.dual_frame(c.g)
    geo = [geo_rot @ np.asarray(a, float) for a in (c.g.nodes, c.g.face_normals, c.g.face_centers,
                                                    c.g.cell_centers)] + [c.g.cell_volumes]
    perm = fv.rotate_second_order(c.raw["K"], geo_rot)
    dg = fv.DualGrid.for_grid(c.g)
    assert all(np.array_equal(x, y) for x, y in zip(dg.mass_pattern(), emu.mass_pattern()))
    bad1, _ = dg.discretize(d._method, geo, perm, geo_rot)
    m1, p1 = dg.download()
    bad2, _ = dg.discretize(d._method, geo, perm, geo_rot)
    m2, p2 = dg.download()
    bade, _ = emu.discretize(d._method, geo, perm, geo_rot)
    me, pe = emu.download()
    assert bad1 == bad2 == bade == -1
    assert np.array_equal(m1, m2) and np.array_equal(p1, p2)
    # entry by entry, each at the scale of its own cells (tests/dual_mp.py): the cells of permeability 10^6 count
    ip, ix = emu.mass_pattern()
    _, Ms, _, Ps = dual_mp.mass_reference(c.g, d._method, geo, perm, geo_rot)
    rows = np.repeat(np.arange(c.g.num_faces), np.diff(ip))
    assert dual_mp.worst(m1, me, Ms[rows, ix])[0] <= dual_mp.MASS_TOL
    assert dual_mp.worst(p1, pe, Ps)[0] <= dual_mp.PROJ_TOL


@pytest.mark.gpu
def test_tutorial_on_the_gpu():
    up = tutorial_numbers()
    assert np.array_equal(up, tutorial_numbers())


def _constant_velocity(g, d):
    """project_flux(face_normals^T v) returns v in every cell (exact for both schemes on planar faces)."""
    rng = np.random.default_rng(7)
    v = rng.standard_normal(3)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(g.num_cells))})
    d.discretize(g, data)
    P0u = d.project_flux(g, g.face_normals.T @ v, data)
    assert np.abs(P0u - v[:, None]).max() <= 1e-12 * np.abs(v).max()
    return data


def _sample_rows(g, d, data, cls_ref):
    """Mass rows whose cells all lie in a seeded sample of 2,000 cells equal the sum of the reference's static
    massHdiv over those cells."""
    pytest.importorskip("scipy")
    import sys
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    try:
        from ref_loader import load_porepy
        pp = load_porepy()
    except Exception:
        pytest.skip("reference not present")
    rng = np.random.default_rng(11)
    cells = np.sort(rng.choice(g.num_cells, 2000, replace=False))
    cf = sps.csc_matrix(g.cell_faces)
    cf.sort_indices()
    mass = data[pb.DISCRETIZATION_MATRICES]["flow"]["mass"].tocsr()
    ref = {}
    K = np.eye(3)
    for c in cells:
        fl = cf.indices[cf.indptr[c]:cf.indptr[c + 1]]
        sg = cf.data[cf.indptr[c]:cf.indptr[c + 1]]
        if cls_ref == "mvem":
            nodes = np.unique(sps.csc_matrix(g.face_nodes)[:, fl].indices)
            x = g.nodes[:, nodes]
            diam = np.sqrt(((x[:, :, None] - x[:, None, :]) ** 2).sum(0)).max()
            A = pp.MVEM.massHdiv(K, K, g.cell_centers[:, c], g.cell_volumes[c], g.face_centers[:, fl],
                                 g.face_normals[:, fl], sg, diam, diam ** (2 - g.dim))[0]
        else:
            fn = sps.csc_matrix(g.face_nodes)
            fnodes = [fn.indices[fn.indptr[f]:fn.indptr[f + 1]] for f in fl]
            alln = np.unique(np.concatenate(fnodes))
            opp = [np.setdiff1d(alln, f)[0] for f in fnodes]
            d3 = g.dim
            size = d3 * (d3 + 1)
            HB = np.zeros((size, size))
            for it in range(0, size, d3):
                HB += np.diagflat(np.ones(size - it), it)
            HB += HB.T
            HB /= d3 * d3 * (d3 + 1) * (d3 + 2)
            A = pp.RT0.massHdiv(K, g.cell_volumes[c], g.nodes[:, opp], sg, d3, HB)
        for i, fi in enumerate(fl):
            for j, fj in enumerate(fl):
                ref[(fi, fj)] = ref.get((fi, fj), 0.0) + A[i, j]
    face_cells = abs(cf).tocsr()
    in_sample = np.zeros(g.num_cells, bool)
    in_sample[cells] = True
    checked = 0
    for f in np.unique(cf.indices[np.concatenate([np.arange(cf.indptr[c], cf.indptr[c + 1]) for c in cells])]):
        if not in_sample[face_cells.indices[face_cells.indptr[f]:face_cells.indptr[f + 1]]].all():
            continue
        row = mass.getrow(f)
        for j, v in zip(row.indices, row.data):
            assert abs(v - ref[(f, j)]) <= 1e-12 * max(abs(v), abs(ref[(f, f)])), (f, j)
        checked += 1
    assert checked > 50   # 63 rows on the tetrahedra (mostly boundary faces), more on the Cartesian grid


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["mvem_tet", "rt0_tet", "mvem_cart"])
def test_bench_size(which):
    from porepy_b200.grid import structured_tet_grid, cart_grid_3d
    g = cart_grid_3d([100, 100, 100]) if which == "mvem_cart" else structured_tet_grid([55, 55, 55])
    d = pb.RT0("flow") if which.startswith("rt0") else pb.MVEM("flow")
    data = _constant_velocity(g, d)
    _sample_rows(g, d, data, which.split("_")[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_assembly_matches_the_host_formulas(name):
    """While the discretization is device resident, assemble_matrix_rhs builds the saddle-point system on the GPU
    without downloading anything; it equals the host formulas applied to the same matrices."""
    from porepy_b200.sparse import LazyCsr
    c = load_case(name)
    data = _data(c)
    d = _discr(c)
    d.discretize(c.g, data)
    before = dict(LazyCsr.downloads)
    A, b = d.assemble_matrix_rhs(c.g, data)
    assert getattr(A, "device_csr", None) is not None
    assert LazyCsr.downloads == before
    A2, b2 = d.assemble_matrix_rhs(c.g, data)   # same values: bit-identical
    assert np.array_equal(b, b2) and np.array_equal(A.device_csr.to_scipy().data, A2.device_csr.to_scipy().data)
    M = d.assemble_matrix(c.g, data)   # touches the stored matrices: the host formulas from here on
    M, norm = d.assemble_neumann_robin(c.g, data, M, bc_weight=True)
    rhs = d.assemble_rhs(c.g, data, norm)
    assert rel_err(M, A) <= 1e-14
    assert np.abs(rhs - b).max() <= 1e-14 * np.abs(rhs).max()
    A3, _ = d.assemble_matrix_rhs(c.g, data)
    assert getattr(A3, "device_csr", None) is None
