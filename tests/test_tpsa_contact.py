"""TPSA elasticity with fractures in frictional contact (``porepy_b200.TpsaFracturedMomentumBalance``,
``pb_tpsa_contact_system`` / ``pb_tpsa_contact_rows``, csrc/tpsa_system.cuh) against the unmodified reference's
``pp.MomentumBalance`` + ``TpsaMomentumBalanceMixin``: Jacobian and -R at the zero state and at the stored iterate, the
residual histories and converged states of the sliding, sticking, open and mixed loads in 3-D and 2-D (fixtures of
tools/make_tpsa_contact_golden.py), live stock models with two fractures through the bridge, the refusals, the grouped
block-Jacobi GMRES on every fixture Jacobian.  The checks shared with the other TPSA systems are those of
tpsa_checks.py.
CPU: host build of tpsa_system.cuh + the scipy stand-in for the device sparse algebra."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200.contact import FractureContact
from porepy_b200.tpsa_contact import TpsaFracturedMomentumBalance
from golden_io import case_names
from tpsa_checks import (ZERO, check_bridge_linearization, check_linearizations, compare_with_host_build, csr, direct,
                         host, to_model, to_solver, use_host_build)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsacontact_")
CONSTANTS = ("numerical_constant", "characteristic_traction", "friction_coefficient", "dilation_angle", "reference_gap",
             "open_state_tolerance")


def _problem(name, fractures=None):
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False))
    g = pb.Grid.from_arrays({k[len("matrix__"):]: v for k, v in d.items() if k.startswith("matrix__")})
    nf = g.num_faces
    bc = SimpleNamespace(is_dir=d["bc_is_dir"], is_neu=d["bc_is_neu"], is_rob=d["bc_is_rob"],
                         is_internal=d["bc_is_internal"], robin_weight=d["bc_robin_weight"], basis=d["bc_basis"],
                         bc_type="vectorial", num_faces=nf)
    data = pb.initialize_data({}, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(d["mu"], d["lmbda"]),
                                                "bc": bc})
    if fractures is None:
        fractures = [FractureContact(csr(d, "mortar_to_primary_avg"), csr(d, "primary_to_mortar_int"),
                                     csr(d, "mortar_to_secondary_avg"), csr(d, "secondary_to_mortar_int"),
                                     d["mortar_sign"], d["mortar_volumes"], csr(d, "local_coordinates"))]
    prob = TpsaFracturedMomentumBalance(g, data, d["bc_values"], fractures, {k: float(d[k]) for k in CONSTANTS},
                                        body_force=d["body_force"], angular_source=d["angular_source"],
                                        mass_source=d["mass_source"])
    prob.column_map, prob.row_map = d["column_map"], d["row_map"]
    return prob, d


def _linearizations(prob, d):
    # the stored iterate of the sticking case is converged: -R is compared on the scale of -R(0)
    return check_linearizations(prob, d, [("zero", d["previous"], d["previous"], "J0", "rhs0"),
                                          ("iterate", d["iterate"], d["previous"], "iterate_jacobian", "iterate_rhs")],
                                1e-12, ZERO)


def check_time_step(prob, d, tol, linear_solver):
    """The first residual from the previous state, the converged state, and the history restarted from the reference's
    stored iterate for the two steps it pins: after that the tangential jump is zero up to round-off and sign(u_t),
    the Jacobian of |u_t|, is decided by round-off on either side (as test_models_2d explains), so later steps of the
    two semismooth loops may take different, equally converging paths."""
    prev, ref = to_solver(prob, d["previous"]), d["residual_norms"]
    x, hist = prob.time_step(prev, linear_solver, tol=1e-14)       # to round-off, as the stored state
    assert abs(hist[0]["residual"] - ref[0]) <= tol * ref[0]
    assert np.linalg.norm(to_model(prob, x) - d["solution"]) <= tol * np.linalg.norm(d["solution"]), hist
    _, hist = prob.time_step(prev, linear_solver, x0=to_solver(prob, d["iterate"]), tol=1e-11)
    mine = np.array([h["residual"] for h in hist])
    n = min(len(mine), len(ref) - 1, 2)
    assert np.abs(mine[:n] - ref[1:1 + n]).max() <= tol * ref[0], (mine, ref)


@pytest.fixture()
def host_build(monkeypatch):
    use_host_build(monkeypatch)


def test_fixtures_present():
    assert len(CASES) == 6
    assert {int(_problem(n)[1]["dim"]) for n in CASES} == {2, 3}


@pytest.mark.parametrize("name", CASES)
def test_host_build_matches_reference(name, host_build):
    prob, d = _problem(name)
    _linearizations(prob, d)
    check_time_step(prob, d, 1e-10, direct)


@pytest.mark.parametrize("name", CASES)
def test_gmres_with_groups_converges_on_fixture_jacobians(name, host_build):
    """scipy GMRES with the grouped block-Jacobi of ``preconditioner_groups()`` on J0 and the iterate's Jacobian, with
    the restart and iteration budget of the default solver of ``time_step`` (GMRES(30), 1,000 iterations)."""
    prob, d = _problem(name)
    groups = prob.preconditioner_groups()
    rows, cols, ptr = np.asarray(groups.rows), np.asarray(groups.cols), np.asarray(groups.ptr)
    for x in (d["previous"], d["iterate"]):
        J, rhs = prob.linearize(to_solver(prob, x), to_solver(prob, d["previous"]))
        A, b = J.to_scipy().tocsr(), host(rhs)
        inv = [np.linalg.inv(A[rows[ptr[q]:ptr[q + 1]]][:, cols[ptr[q]:ptr[q + 1]]].toarray())
               for q in range(len(ptr) - 1)]

        def apply(v, inv=inv):
            out = np.zeros_like(v)
            for q, Bi in enumerate(inv):
                out[cols[ptr[q]:ptr[q + 1]]] = Bi @ v[rows[ptr[q]:ptr[q + 1]]]
            return out
        M = spla.LinearOperator(A.shape, matvec=apply)
        y, info = spla.gmres(A, b, M=M, rtol=1e-10, restart=30, maxiter=1000 // 30)
        assert info == 0 and np.linalg.norm(A @ y - b) <= 1e-9 * np.linalg.norm(b)


def _refusals():
    prob, d = _problem(CASES[0])
    fc = prob.fractures[0]
    # a mortar cell on two faces (non-matching mortar grid)
    m2p = csr(d, "mortar_to_primary_avg").tolil()
    f0, f1 = np.flatnonzero(csr(d, "mortar_to_primary_avg")[:, 0].toarray().ravel())[0], 0
    m2p[f1, 0] = 0.5
    bad = FractureContact(m2p.tocsr(), csr(d, "primary_to_mortar_int"), csr(d, "mortar_to_secondary_avg"),
                          csr(d, "secondary_to_mortar_int"), d["mortar_sign"], d["mortar_volumes"],
                          csr(d, "local_coordinates"))
    with pytest.raises(ValueError, match="matching mortar grids"):
        _problem(CASES[0], [bad])[0].discretize()
    # two mortar cells on one face
    p2m = csr(d, "primary_to_mortar_int").tolil()
    m2p = csr(d, "mortar_to_primary_avg").tolil()
    g0 = int(np.flatnonzero(m2p[:, 0].toarray().ravel())[0])
    g1 = int(np.flatnonzero(m2p[:, 1].toarray().ravel())[0])
    m2p[g1, 1], m2p[g0, 1], p2m[1, g1], p2m[1, g0] = 0.0, 1.0, 0.0, 1.0
    bad = FractureContact(m2p.tocsr(), p2m.tocsr(), csr(d, "mortar_to_secondary_avg"),
                          csr(d, "secondary_to_mortar_int"), d["mortar_sign"], d["mortar_volumes"],
                          csr(d, "local_coordinates"))
    with pytest.raises(ValueError, match="more than one mortar cell"):
        _problem(CASES[0], [bad])[0].discretize()
    assert f0 >= 0 and fc.num_mortar == 2 * fc.num_cells
    with pytest.raises(ValueError, match="no dof maps"):
        TpsaFracturedMomentumBalance(prob.sd, prob.data, d["bc_values"], prob.fractures,
                                     {k: float(d[k]) for k in CONSTANTS}).to_model_order(sps.eye(prob.num_dofs))
    with pytest.raises(ValueError, match="bc_values must have"):
        TpsaFracturedMomentumBalance(prob.sd, prob.data, d["bc_values"][:-1], prob.fractures,
                                     {k: float(d[k]) for k in CONSTANTS})
    prob.sd.periodic_face_map = np.zeros((2, 1), int)
    try:
        with pytest.raises(NotImplementedError, match="periodic"):
            prob.discretize()
    finally:
        del prob.sd.periodic_face_map


def test_refusals_host(host_build):
    _refusals()
    from porepy_b200 import model_bridge
    fake = SimpleNamespace(equation_system=SimpleNamespace(equations={"mass_balance_equation": None}))
    with pytest.raises(NotImplementedError, match="fractured TPSA poromechanics"):
        model_bridge.tpsa_fractured_momentum_from_model(fake)
    m3, m2, m1 = SimpleNamespace(dim=3), SimpleNamespace(dim=2), SimpleNamespace(dim=1)
    fake = SimpleNamespace(equation_system=SimpleNamespace(equations={}), mdg=SimpleNamespace(
        dim_max=lambda: 3, subdomains=lambda dim=None: [s for s in (m3, m2, m1) if dim is None or s.dim == dim]))
    with pytest.raises(NotImplementedError, match="intersections"):
        model_bridge.tpsa_fractured_momentum_from_model(fake)


def test_too_many_face_neighbours_host(host_build):
    """A cell with 32 face neighbours (a fan of 32 triangles around one centre cell) is refused."""
    from emu_tpsa import EmuTpsaFaceGrid
    n = 32
    # one centre cell with n faces, each shared with one outer cell; every outer cell also has two boundary faces
    rows, cols, vals = [], [], []
    for f in range(n):
        rows += [f, f]
        cols += [0, 1 + f]
        vals += [1, -1]
    nf = n + 2 * n
    for c in range(n):
        for q in range(2):
            rows.append(n + 2 * c + q)
            cols.append(1 + c)
            vals.append(1)
    cf = sps.csc_matrix((vals, (rows, cols)), shape=(nf, n + 1))
    ang = 2 * np.pi * np.arange(nf) / nf
    g = SimpleNamespace(num_cells=n + 1, num_faces=nf, cell_faces=cf,
                        face_normals=np.vstack([np.cos(ang), np.sin(ang), np.zeros(nf)]),
                        face_centers=np.vstack([np.cos(ang), np.sin(ang), np.zeros(nf)]),
                        cell_centers=np.zeros((3, n + 1)))
    fg = EmuTpsaFaceGrid(g)
    codes = np.zeros((nf, 2), np.uint8)
    flags = np.zeros(nf, np.uint8)
    flags[n:] = 1
    mortars = {k: np.zeros(0) for k in ("face", "cell", "m2p", "p2m", "sign", "volume")}
    with pytest.raises(ValueError, match="too many face neighbours"):
        fg.tpsa_contact_system(2, np.ones(n + 1), np.ones(n + 1), np.ones(n + 1), codes, None, flags, np.ones(nf),
                               mortars, np.zeros(0), 1.0)


# ---- live stock models with two fractures through the bridge -------------------------------------------------------


def _stock_model(pp, nd):
    import make_contact_golden as gc
    from make_mdflow_golden import rect

    class Geometry:
        set_domain, grid_type, stiffness_tensor = gc.Model.set_domain, gc.Model.grid_type, gc.Model.stiffness_tensor
        bc_type_mechanics = gc.Model.bc_type_mechanics

        def meshing_arguments(self):
            return {"cell_size": 0.25}

        def set_fractures(self):
            self._fractures = [pp.PlaneFracture(rect(0, 0.25, 0.25, 0.75)), pp.PlaneFracture(rect(0, 0.75, 0.0, 0.5))]

        def bc_values_displacement(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros((self.nd, bg.num_cells))
            v[0, s.east] = 0.02 * (bg.cell_centers[self.nd - 1, s.east] - 0.4)
            v[1, s.east] = 0.01
            return v.ravel("F")

    class Geometry2d(Geometry):
        set_domain = gc.Model2d.set_domain

        def set_geometry(self):
            self.set_domain()
            self.mdg = pp.meshing.cart_grid([np.array([[0.25, 0.25], [0.25, 0.75]]),
                                             np.array([[0.75, 0.75], [0.5, 1.0]])], [8, 8], physdims=[1, 1])
            self.nd = self.mdg.dim_max()
            pp.set_local_coordinate_projections(self.mdg)
            self.set_well_network()

    base = Geometry if nd == 3 else Geometry2d
    M = type("Stock", (base, pp.models.momentum_balance.TpsaMomentumBalanceMixin, pp.MomentumBalance), {})
    solid = pp.SolidConstants(lame_lambda=2.0, shear_modulus=1.5, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1)
    m = M({"times_to_export": [], "material_constants": {"solid": solid}})
    m.prepare_simulation()
    rng = np.random.default_rng(nd)
    x = 1e-3 * rng.standard_normal(m.equation_system.num_dofs())
    m.equation_system.set_variable_values(x, iterate_index=0)
    m.equation_system.set_variable_values(0.5 * x, time_step_index=0)
    return m


def _check_bridge(nd, solve=False):
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    es = m.equation_system
    prob, cols, rows = plugin(pp).tpsa_fractured_momentum_from_model(m)
    assert len(prob.fractures) == 2 and prob.num_dofs == es.num_dofs()
    check_bridge_linearization(m, prob, cols, rows)
    with pytest.raises(NotImplementedError, match="fractures are not supported"):
        plugin(pp).tpsa_momentum_from_model(m)
    if solve:                                        # the device problem reaches the reference's own state
        xp = es.get_variable_values(time_step_index=0)
        es.set_variable_values(xp, iterate_index=0)
        m.before_nonlinear_loop()
        for _ in range(30):                          # the reference's own semismooth Newton loop
            m.before_nonlinear_iteration()
            m.assemble_linear_system()
            if np.linalg.norm(m.linear_system[1]) < 1e-11:
                break
            m.after_nonlinear_iteration(m.solve_linear_system())
        xr = es.get_variable_values(iterate_index=0)
        xd, hist = prob.time_step(xp[cols], direct, tol=1e-11)
        assert hist[-1]["residual"] <= 1e-10 * hist[0]["residual"], hist
        assert np.linalg.norm(host(xd) - xr[cols]) <= 1e-8 * np.linalg.norm(xr), hist


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("nd", [2, 3])
def test_bridge_host_build(nd, host_build):
    _check_bridge(nd)


# ---- GPU ----------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_reference_and_host_build(name):
    prob, d = _problem(name)
    dev = _linearizations(prob, d)
    dev2 = _linearizations(prob, d)                              # a second assembly: bit-identical
    for (A, b), (A2, b2) in zip(dev, dev2):
        assert np.array_equal(A.indptr, A2.indptr) and np.array_equal(A.indices, A2.indices)
        assert np.array_equal(A.data, A2.data) and np.array_equal(b, b2)
    check_time_step(prob, d, 1e-10, direct)
    compare_with_host_build(lambda: _linearizations(*_problem(name)), dev, same_pattern=True)


@pytest.mark.gpu
def test_gpu_leaves_tpsa_system_pattern_alone():
    """pb_tpsa_contact_system on a handle leaves a later pb_tpsa_system matrix bit-identical."""
    prob, d = _problem(CASES[0])
    sd = prob.sd
    el = pb.TpsaElasticity(sd, prob.data, "mechanics", d["bc_values"])
    el.discretize()
    A0 = el.A.to_scipy()
    fg = el._fg
    prob._fg = fg
    prob.discretize()                               # the contact system on the same handle
    el.discretize()
    A1 = el.A.to_scipy()
    assert np.array_equal(A0.indptr, A1.indptr) and np.array_equal(A0.indices, A1.indices)
    assert np.array_equal(A0.data, A1.data)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_time_step_with_device_gmres(name, monkeypatch):
    """The Newton loop with the default device GMRES reaches the stored converged state; no matrix leaves the device.
    The stored states are converged to round-off (tools/make_tpsa_contact_golden.py), so a Newton path other than the
    reference's still meets them to 1e-10."""
    from porepy_b200.sparse import DeviceCsr
    prob, d = _problem(name)
    prob.discretize()

    def refuse(self):
        raise AssertionError("to_scipy inside the Newton loop")
    monkeypatch.setattr(DeviceCsr, "to_scipy", refuse)
    x, hist = prob.time_step(to_solver(prob, d["previous"]), tol=1e-14)
    monkeypatch.undo()
    assert np.linalg.norm(to_model(prob, x) - d["solution"]) <= 1e-10 * np.linalg.norm(d["solution"]), hist


@pytest.mark.gpu
def test_gpu_refusals():
    import torch
    _refusals()
    prob, d = _problem(CASES[0])
    prob.discretize()
    fg, nk = prob._fg, prob.fractures[0].num_cells
    b = torch.zeros(prob.num_dofs, dtype=torch.float64, device="cuda")
    r = torch.zeros(3 * nk, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="contact Jacobian must be"):
        fg.tpsa_contact_rows(prob.A, pb.DeviceCsr(sps.csr_matrix((3 * nk, 3 * nk))), r, b)
    with pytest.raises(ValueError, match="not the TPSA contact system"):
        fg.tpsa_contact_rows(pb.DeviceCsr(sps.eye(prob.num_dofs, format="csr")),
                             pb.DeviceCsr(sps.csr_matrix((3 * nk, 9 * nk))), r, b)


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("nd", [2, 3])
def test_gpu_bridge(nd):
    _check_bridge(nd, solve=True)
