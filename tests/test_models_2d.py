"""The device model classes in 2-D: ``Poromechanics``, ``Thermoporomechanics``, ``FracturedMomentumBalance``,
``FracturedPoromechanics`` and ``FracturedThermoporomechanics`` on a 2-D matrix (cut by a line fracture where there is
contact) against the unmodified reference -- Jacobian and residual at a stored iterate, the residual history of the Newton
loop and the converged state (tests/golden/*_2d*.npz: tools/make_poromech_golden.py, make_thm_golden.py and
make_contact_golden.py); the group sizes of the block-Jacobi preconditioner in 2-D; live stock models through the bridges
of ``model_bridge`` (where the reference is importable); the refusals of intersecting line fractures and of a 1-D matrix.
CPU: host build of the node / face routines + the scipy stand-in for the device sparse algebra.  GPU: the same checks on
the device, and a time step of every contact fixture with the device GMRES and no matrix leaving the device."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
import test_poromech_model
import test_thm_model
from golden_io import GOLDEN_DIR
from porepy_b200 import krylov
from porepy_b200.contact import FractureContact, FracturedMomentumBalance
from porepy_b200.fractured_poromech import FractureCoupling, FracturedPoromechanics
from porepy_b200.fractured_thm import FracturedThermoporomechanics
from porepy_b200.grid import Grid
from porepy_b200.poromech import Poromechanics
from porepy_b200.thermoporomech import Thermoporomechanics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CONTACT = ["contact_2d", "contact_2d_mixed"]
CONTACT_FLOW = ["contact_poromech_2d", "contact_thm_2d"]
BULK = ["poromech_model_2d", "thm_model_2d"]
FIXTURES = BULK + CONTACT + CONTACT_FLOW
CONTACT_CONSTANTS = ("numerical_constant", "characteristic_traction", "friction_coefficient", "dilation_angle",
                     "reference_gap", "open_state_tolerance")


# ---------------------------------------------------------------- fixtures -> problems


def _load(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))


def _csr(d, key):
    return sps.csr_matrix((d[key + "__data"], d[key + "__indices"], d[key + "__indptr"]), shape=tuple(d[key + "__shape"]))


def _grid(d, prefix=""):
    g = Grid.from_arrays({k[len(prefix):]: v for k, v in d.items() if k.startswith(prefix)})
    for tag in ("domain_boundary_faces", "tip_faces"):
        if prefix + tag in d:
            g.tags[tag] = np.asarray(d[prefix + tag], bool)
    return g


def _scalar_bc(d, prefix, nf, internal=None):
    internal = np.zeros(nf, bool) if internal is None else internal
    return SimpleNamespace(is_dir=d[prefix + "is_dir"], is_neu=d[prefix + "is_neu"],
                           is_rob=d.get(prefix + "is_rob", np.zeros(nf, bool)),
                           is_internal=d.get(prefix + "is_internal", internal), robin_weight=np.ones(nf),
                           bc_type="scalar", num_faces=nf)


def _vector_bc(d, g):
    nd, nf = int(g.dim), g.num_faces
    assert np.shape(d["mech_is_dir"]) == (nd, nf)
    return SimpleNamespace(is_dir=d["mech_is_dir"], is_neu=d["mech_is_neu"], is_rob=d["mech_is_rob"],
                           is_internal=d["mech_is_internal"], robin_weight=np.zeros((nd, nd, nf)), bc_type="vectorial",
                           num_faces=nf)


def _projections(d):
    return {k: _csr(d, k) for k in ("mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg",
                                    "secondary_to_mortar_int", "mortar_to_primary_int", "primary_to_mortar_avg",
                                    "mortar_to_secondary_int", "secondary_to_mortar_avg")}


def _thermal_constants(d):
    fluid = dict(compressibility=d["compressibility"], density=d["density"], viscosity=d["viscosity"],
                 thermal_expansion=d["fluid_thermal_expansion"], heat_capacity=d["fluid_heat_capacity"],
                 conductivity=d["fluid_conductivity"], reference_pressure=d["reference_pressure"],
                 reference_temperature=d["reference_temperature"])
    solid = dict(reference_porosity=d["reference_porosity"], n_inv=d["n_inv"], biot_coefficient=d["biot_coefficient"],
                 thermal_expansion=d["solid_thermal_expansion"], heat_capacity=d["solid_heat_capacity"],
                 conductivity=d["solid_conductivity"], density=d["solid_density"])
    return fluid, solid


def load_problem(name):
    """(problem, fixture) of one 2-D fixture."""
    d = _load(name)
    if name == "poromech_model_2d":
        g = _grid(d)
        nf = g.num_faces
        data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(d["K"]),
                                               "bc": _scalar_bc(d, "flow_", nf)})
        pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor.from_values(d["C"]),
                                               "bc": _vector_bc(d, g),
                                               "scalar_vector_mappings": {"flow": float(d["biot_coefficient"])}})
        fluid = {k: float(d[k]) for k in ("compressibility", "density", "viscosity", "reference_pressure")}
        solid = {"reference_porosity": float(d["reference_porosity"]), "n_inv": float(d["n_inv"])}
        return Poromechanics(g, data, fluid, solid, d["flow_bc_values"], d["mech_bc_values"], _scalar_bc(d, "ff_", nf),
                             d["ff_values"]), d
    if name == "thm_model_2d":
        g = _grid(d)
        nf = g.num_faces
        data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(d["K"]),
                                               "bc": _scalar_bc(d, "flow_", nf)})
        pb.initialize_data(data, "fourier", {"bc": _scalar_bc(d, "fourier_", nf)})
        pb.initialize_data(data, "mechanics", {
            "fourth_order_tensor": pb.FourthOrderTensor.from_values(d["C"]), "bc": _vector_bc(d, g),
            "scalar_vector_mappings": {"flow": pb.SecondOrderTensor.from_values(d["alpha_flow"]),
                                       "thermal": pb.SecondOrderTensor.from_values(d["alpha_thermal"])}})
        fluid, solid = _thermal_constants(d)
        bc = dict(flow=d["flow_bc_values"], fourier=d["fourier_bc_values"], mechanics=d["mech_bc_values"],
                  fluid_flux=d["ff_values"], enthalpy_flux=d["ef_values"], fluid_flux_type=_scalar_bc(d, "ff_", nf),
                  enthalpy_flux_type=_scalar_bc(d, "ef_", nf))
        return Thermoporomechanics(g, data, fluid, solid, bc), d
    contact = {k: float(d[k]) for k in CONTACT_CONSTANTS}
    if name in CONTACT:
        g = _grid(d, "matrix__")
        data = pb.initialize_data({}, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor.from_values(d["C"]),
                                                    "bc": _vector_bc(d, g)})
        frac = FractureContact(_csr(d, "mortar_to_primary_avg"), _csr(d, "primary_to_mortar_int"),
                               _csr(d, "mortar_to_secondary_avg"), _csr(d, "secondary_to_mortar_int"), d["mortar_sign"],
                               d["mortar_volumes"], _csr(d, "local_coordinates"))
        return FracturedMomentumBalance(g, data, d["mech_bc_values"], [frac], contact), d
    g, gf = _grid(d, "matrix__"), _grid(d, "fracture__")
    nd, nf, nff = int(g.dim), g.num_faces, gf.num_faces
    internal = np.asarray(g.tags["fracture_faces"], bool)
    thermal = name == "contact_thm_2d"
    kf = d["fracture__flow_K"] if thermal else d["fracture__K"]
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(
        d["matrix__flow_K"] if thermal else d["matrix__K"]), "bc": _scalar_bc(d, "matrix__flow_", nf)})
    fdata = pb.initialize_data({}, "flow", {"bc": _scalar_bc(d, "fracture__flow_", nff), "ambient_dimension": nd})
    mappings = {"flow": float(d["biot_coefficient"])}
    if thermal:
        pb.initialize_data(data, "fourier", {"bc": _scalar_bc(d, "matrix__fourier_", nf)})
        pb.initialize_data(fdata, "fourier", {"bc": _scalar_bc(d, "fracture__fourier_", nff), "ambient_dimension": nd})
        mappings = {"flow": pb.SecondOrderTensor.from_values(d["alpha_flow"]),
                    "thermal": pb.SecondOrderTensor.from_values(d["alpha_thermal"])}
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor.from_values(d["C"]),
                                           "bc": _vector_bc(d, g), "scalar_vector_mappings": mappings})
    # the fixture stores the fracture tensor of the initial state: tangential permeability x residual aperture
    frac = FractureCoupling(gf, fdata, _projections(d), d["mortar_sign"], d["mortar_volumes"], _csr(d, "local_coordinates"),
                            d["normal_permeability"], kf / float(d["residual_aperture"]))
    bc = dict(flow=d["flow_bc_values"], mechanics=d["mech_bc_values"], fluid_flux=d["ff_values"],
              fluid_flux_type=_scalar_bc(d, "ff_", nf, internal))
    if not thermal:
        fluid = {k: float(d[k]) for k in ("compressibility", "density", "viscosity", "reference_pressure")}
        solid = {k: float(d[k]) for k in ("reference_porosity", "n_inv", "residual_aperture")}
        return FracturedPoromechanics(g, data, [frac], fluid, solid, contact, bc), d
    fluid, solid = _thermal_constants(d)
    solid["residual_aperture"] = d["residual_aperture"]
    bc.update(fourier=d["fourier_bc_values"], enthalpy_flux=d["ef_values"], enthalpy_flux_type=_scalar_bc(d, "ef_", nf, internal))
    return FracturedThermoporomechanics(g, data, [frac], fluid, solid, contact, bc, [d["normal_thermal_conductivity"]]), d


# ---------------------------------------------------------------- checks shared by the host and device legs


def _orders(prob, d):
    cm = d["column_map"]
    rm = d["row_map"] if "row_map" in d else np.arange(prob.num_dofs)
    assert np.array_equal(np.sort(cm), np.arange(prob.num_dofs)) and np.array_equal(np.sort(rm), np.arange(prob.num_dofs))
    return cm, rm


def _linearizer(prob, d):
    cm = d["column_map"]
    if isinstance(prob, FracturedMomentumBalance):
        return lambda x: prob.linearize(x, d["previous"][cm])
    return lambda x: prob.linearize(x, d["previous"][cm], float(d["dt"]))


def _time_step(prob, d, x_prev, solver):
    if isinstance(prob, FracturedMomentumBalance):
        return prob.time_step(x_prev, solver, tol=1e-11)
    return prob.time_step(x_prev, float(d["dt"]), solver, tol=1e-11)


def check_contact_state(prob, d, x, name):
    """Open cells carry no traction, closed ones a compressive normal traction on (sliding) or inside (sticking) the
    friction cone; the load cases are sliding everywhere, and two open cells next to two sliding ones."""
    nd = prob.nd
    t = prob.unknown_layout.parts(x)["contact_traction"][0].reshape(-1, nd)
    tt, tn = np.abs(t[:, 0]), t[:, nd - 1]                       # a line fracture: one tangential component
    mu = float(d["friction_coefficient"])
    is_open = np.abs(tn) < 1e-12
    assert np.all(np.abs(t[is_open]) < 1e-12) and np.all(tn[~is_open] < 0)
    assert np.allclose(tt[~is_open], mu * np.abs(tn[~is_open]), rtol=1e-8), (name, t)     # sliding
    assert is_open.sum() == {"contact_2d": 0, "contact_2d_mixed": 2}.get(name, 0), (name, t)


def check(prob, d, to_host, make_tensor, name):
    """J and -R at the stored iterate(s) within 1e-10, the Newton history, the converged state (direct solves)."""
    if name == "poromech_model_2d":
        return test_poromech_model.check(prob, d, to_host, linear_solver=lambda J, r: make_tensor(
            spla.spsolve(J.to_scipy().tocsc(), to_host(r))))
    if name == "thm_model_2d":
        return test_thm_model.check(prob, d, to_host, linear_solver=lambda J, r: make_tensor(
            spla.spsolve(J.to_scipy().tocsc(), to_host(r))))
    cm, rm = _orders(prob, d)
    for state, jac, rhs_key in ((d["previous"], "initial_jacobian", "initial_rhs"), (d["iterate"], "iterate_jacobian", "iterate_rhs")):
        if jac + "__data" not in d:
            continue
        J, rhs = prob.linearize(state[cm], d["previous"][cm]) if name in CONTACT else \
            prob.linearize(state[cm], d["previous"][cm], float(d["dt"]))
        Jref, bref = _csr(d, jac)[rm][:, cm], d[rhs_key][rm]
        assert abs(J.to_scipy() - Jref).max() <= 1e-10 * abs(Jref).max(), jac
        assert np.abs(to_host(rhs) - bref).max() <= 1e-10 * max(np.abs(bref).max(), 1e-3 * abs(Jref).max()), rhs_key

    def direct(Jd, r):
        return make_tensor(spla.spsolve(Jd.to_scipy().tocsc(), to_host(r)))
    x, hist = _time_step(prob, d, d["previous"][cm], direct)
    check_history_and_state(prob, d, to_host(x), hist, name, direct)


def check_history_and_state(prob, d, x, hist, name, solver):
    """The time step from the previous state converges to the stored state, through the reference's first iterate.
    After that the paths may part: the first step leaves the tangential jump of the sticking start at zero, up to
    round-off, and the reference's norm of a one-component tangential vector is ``pp.ad.functions.abs``, whose
    Jacobian is sign(u_t) -- 0 at an exact zero, +-1 at +-1e-17.  So the rest of the history is compared on the
    reference's own path: the Newton loop restarted from its stored iterate, where J and -R agree to 1e-10."""
    from porepy_b200 import ad
    from porepy_b200.newton import newton_loop
    cm = d["column_map"]
    ref = d["residual_norms"]
    assert hist[-1]["residual"] <= 1e-10 * hist[0]["residual"] and len(hist) <= len(ref) + 1, hist
    for mine, theirs in zip(hist[:2], ref[:2]):
        assert abs(mine["residual"] - theirs) <= 0.05 * theirs, (hist, ref)
    assert np.linalg.norm(x - d["solution"][cm]) <= 1e-8 * np.linalg.norm(d["solution"])
    check_contact_state(prob, d, x, name)
    k = int(np.argmin(np.abs(ref - np.linalg.norm(d["iterate_rhs"]))))          # the stored iterate's place in the loop
    _, replay = newton_loop(_linearizer(prob, d), ad.device_vector(d["iterate"][cm]), solver, 1e-11 * ref[0] / ref[k],
                            len(ref) - k)
    assert len(replay) == len(ref) - k, ([h["residual"] for h in replay], ref[k:])
    for mine, theirs in zip(replay, ref[k:]):
        if theirs > 1e-9 * ref[0]:
            assert abs(mine["residual"] - theirs) <= 0.05 * theirs, ([h["residual"] for h in replay], ref[k:])


@pytest.fixture()
def host_build(monkeypatch):
    from emu_binding import EmuBackedFaceGrid, EmuBackedPlan, emu_interface_upwind_masks
    from porepy_b200 import fv
    import emu_sparse
    monkeypatch.setattr(fv, "DevicePlan", EmuBackedPlan)
    monkeypatch.setattr(fv, "FaceGrid", EmuBackedFaceGrid)
    monkeypatch.setattr(fv, "interface_upwind_masks", emu_interface_upwind_masks)
    emu_sparse.install(monkeypatch)


def _host_tensor(a):
    import torch
    return torch.as_tensor(np.asarray(a, float))


def _cuda(a):
    import torch
    return torch.as_tensor(np.asarray(a, float), device="cuda")


# ---------------------------------------------------------------- CPU


def test_fixtures_are_two_dimensional():
    for name in FIXTURES:
        d = _load(name)
        prefix = "" if name in BULK else "matrix__"
        assert int(d[prefix + "dim"]) == 2, name
        if name not in BULK:
            nfc = d["fracture__cell_volumes"].size
            assert int(d["fracture__dim"]) == 1 and _csr(d, "local_coordinates").shape == (2 * nfc, 2 * nfc)
            assert d["matrix__cell_volumes"].size == 64 and nfc == 4, name      # 8 x 8 cells, a line of four


@pytest.mark.parametrize("name", FIXTURES)
def test_model_2d_host_build(name, host_build):
    prob, d = load_problem(name)
    assert prob.nd == 2
    prob.discretize()
    check(prob, d, lambda t: t.numpy(), _host_tensor, name)


@pytest.mark.parametrize("name", CONTACT + CONTACT_FLOW)
def test_preconditioner_groups_2d(name):
    """nd (+1, +2) rows per matrix cell; 3 nd (+3, +8) per fracture cell with its two mortar cells: the groups partition
    the unknowns and the equations, and every block of the stored Jacobians is well conditioned."""
    prob, d = load_problem(name)
    groups = prob.preconditioner_groups()
    assert groups.n == prob.num_dofs
    assert np.array_equal(np.sort(groups.rows), np.arange(prob.num_dofs))
    assert np.array_equal(np.sort(groups.cols), np.arange(prob.num_dofs))
    nc, nfc = prob.nc, prob.fractures[0].num_cells
    expect = {FracturedMomentumBalance: (2, 6), FracturedPoromechanics: (3, 9), FracturedThermoporomechanics: (4, 14)}
    matrix, fracture = expect[type(prob)]
    assert groups.sizes.tolist() == [matrix] * nc + [fracture] * nfc
    cm, rm = _orders(prob, d)
    for key in ("initial_jacobian", "iterate_jacobian"):
        if key + "__data" not in d:
            continue
        J = _csr(d, key)[rm][:, cm].tocsr()
        for g in range(groups.num_groups):
            r, c = groups.rows[groups.ptr[g]:groups.ptr[g + 1]], groups.cols[groups.ptr[g]:groups.ptr[g + 1]]
            assert np.linalg.cond(J[r][:, c].toarray()) < 1e4, (key, g)


def test_contact_operators_2d(monkeypatch):
    """A line fracture: the local frame is (tangent, normal) per cell, ``sel_n`` takes component 1, ``sel_t`` component 0
    and ``s2t`` is the identity."""
    import emu_sparse
    from porepy_b200.contact import contact_operators
    emu_sparse.install(monkeypatch)
    prob, d = load_problem("contact_2d")
    fc = prob.fractures[0]
    assert fc.nd == 2 and fc.m2s.shape == (2 * fc.num_cells, 2 * fc.num_mortar)
    q = contact_operators(fc.rotation, fc.m2s, fc.sign, fc.s2m, fc.volumes, 1.0, 2)
    n = fc.num_cells
    assert q["nd"] == 2
    assert (q["sel_n"].to_scipy() != sps.csr_matrix((np.ones(n), (np.arange(n), 2 * np.arange(n) + 1)), shape=(n, 2 * n))).nnz == 0
    assert (q["sel_t"].to_scipy() != sps.csr_matrix((np.ones(n), (np.arange(n), 2 * np.arange(n))), shape=(n, 2 * n))).nnz == 0
    assert (q["s2t"].to_scipy() != sps.identity(n, format="csr")).nnz == 0


def test_refusals_of_the_classes():
    g1 = SimpleNamespace(dim=1, num_cells=3, num_faces=4)
    for make in (lambda: Poromechanics(g1, {}, {"compressibility": 0, "density": 1, "viscosity": 1},
                                       {"reference_porosity": 0.1, "n_inv": 0}, None, None, None, None),
                 lambda: Thermoporomechanics(g1, {}, {}, {}, {}),
                 lambda: FracturedMomentumBalance(g1, {}, np.zeros(4), [], {})):
        with pytest.raises(NotImplementedError, match="2-D or 3-D .* not a 1-D"):
            make()
    # a fracture with 3-D local coordinates in a 2-D matrix
    prob2, d2 = load_problem("contact_2d")
    d3 = _load("contact_model")
    frac3 = FractureContact(_csr(d3, "mortar_to_primary_avg"), _csr(d3, "primary_to_mortar_int"),
                            _csr(d3, "mortar_to_secondary_avg"), _csr(d3, "secondary_to_mortar_int"), d3["mortar_sign"],
                            d3["mortar_volumes"], _csr(d3, "local_coordinates"))
    assert frac3.nd == 3
    with pytest.raises(ValueError, match="3-D local coordinates in a 2-D matrix"):
        FracturedMomentumBalance(prob2.sd, prob2.data, d2["mech_bc_values"], [frac3], {})
    with pytest.raises(ValueError, match="frame per cell"):
        FractureContact(sps.csr_matrix((2, 2)), sps.csr_matrix((2, 2)), sps.csr_matrix((1, 2)), sps.csr_matrix((2, 1)),
                        [1, -1], [1, 1], sps.identity(4))


class _FakeMdg:
    """The parts of a ``pp.MixedDimensionalGrid`` the bridges read before they refuse."""

    def __init__(self, dims):
        self.grids = [SimpleNamespace(dim=d) for d in dims]

    def subdomains(self, dim=None):
        return [g for g in self.grids if dim is None or g.dim == dim]

    def dim_max(self):
        return max(g.dim for g in self.grids)


def test_bridge_refusals():
    from porepy_b200 import model_bridge as mb
    crossing = SimpleNamespace(mdg=_FakeMdg([2, 1, 1, 0]))          # two crossing lines and their intersection point
    for build in (mb.fractured_momentum_from_model, mb.fractured_poromechanics_from_model,
                  mb.fractured_thermoporomechanics_from_model):
        with pytest.raises(NotImplementedError, match="0-D subdomains .* in a 2-D matrix"):
            build(crossing)
    line = SimpleNamespace(mdg=_FakeMdg([1]))
    for build in (mb.fractured_momentum_from_model, mb.fractured_poromechanics_from_model,
                  mb.fractured_thermoporomechanics_from_model):
        with pytest.raises(NotImplementedError, match="a 1-D matrix"):
            build(line)
    for build in (mb.poromechanics_from_model, mb.thermoporomechanics_from_model):
        with pytest.raises(NotImplementedError, match="2-D or 3-D subdomain, the model's is 1-D"):
            build(line)
        with pytest.raises(NotImplementedError, match="one subdomain without fractures .* dimensions \\[2, 1\\]"):
            build(SimpleNamespace(mdg=_FakeMdg([2, 1])))
    with pytest.raises(NotImplementedError, match="1-D subdomains .* in a 3-D matrix"):
        mb.fractured_momentum_from_model(SimpleNamespace(mdg=_FakeMdg([3, 2, 2, 1])))


# ---------------------------------------------------------------- live stock models (reference present)


needs_reference = pytest.mark.skipif(not reference_available(), reason="reference tree not present")


def _live_models(pp):
    """(model, bridge, dt) of the five 2-D stock models: ``pp.Poromechanics`` / ``pp.Thermoporomechanics`` on the default
    geometry (the unit square, 2 x 2 cells) with loads, and ``pp.MomentumBalance`` / ``pp.Poromechanics`` /
    ``pp.Thermoporomechanics`` on an 8 x 8 square cut by two line fractures that do not intersect, the second one
    reaching the domain boundary."""
    import make_contact_golden as gc
    import make_poromech_golden as gp
    from porepy_b200.porepy_plugin import plugin
    b = plugin(pp)

    class Loads:
        permeability = gc.permeability
        stiffness_tensor = gc.Model.stiffness_tensor

        def bc_type_darcy_flux(self, sd):
            s = self.domain_boundary_sides(sd)
            return pp.BoundaryCondition(sd, s.south + s.north, "dir")
        bc_type_fluid_flux = bc_type_fourier_flux = bc_type_enthalpy_flux = bc_type_darcy_flux

        def bc_values_pressure(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros(bg.num_cells)
            v[s.south] = 0.02 * (1 + bg.cell_centers[0, s.south])
            return v

        def bc_values_temperature(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros(bg.num_cells)
            v[s.south] = 0.3 + 0.1 * bg.cell_centers[0, s.south]
            return v

    class Bulk(Loads):
        bc_type_mechanics = gp.Model2d.bc_type_mechanics
        bc_values_stress = gp.Model2d.bc_values_stress
        bc_values_displacement = gp.Model2d.bc_values_displacement

    class TwoLines(Loads):
        bc_type_mechanics = gc.Model.bc_type_mechanics
        set_domain = gc.Model2d.set_domain

        def set_geometry(self):
            self.set_domain()
            lines = [np.array([[0.25, 0.25], [0.25, 0.75]]), np.array([[0.75, 0.75], [0.0, 0.5]])]
            self.mdg = pp.meshing.cart_grid(lines, [8, 8], physdims=[1, 1])
            self.nd = self.mdg.dim_max()
            pp.set_local_coordinate_projections(self.mdg)
            self.set_well_network()

        def bc_values_displacement(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros((2, bg.num_cells))
            v[0, s.east] = 0.02 * (bg.cell_centers[1, s.east] - 0.4)       # part of each fracture closes, part opens
            v[1, s.east] = 0.01
            return v.ravel("F")
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7, thermal_expansion=0.03,
                              specific_heat_capacity=2.0, thermal_conductivity=0.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0,
                              normal_permeability=2.0, residual_aperture=0.05, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1, thermal_expansion=0.02, specific_heat_capacity=1.5,
                              thermal_conductivity=1.1, density=2.5)
    params = {"times_to_export": [], "material_constants": {"fluid": fluid, "solid": solid}}
    for mixin, ref_cls, build, dt in ((Bulk, pp.Poromechanics, b.poromechanics_from_model, 0.25),
                                      (Bulk, pp.Thermoporomechanics, b.thermoporomechanics_from_model, 0.25),
                                      (TwoLines, pp.MomentumBalance, b.fractured_momentum_from_model, None),
                                      (TwoLines, pp.Poromechanics, b.fractured_poromechanics_from_model, 0.25),
                                      (TwoLines, pp.Thermoporomechanics, b.fractured_thermoporomechanics_from_model, 0.25)):
        model = type("Live2d", (mixin, ref_cls), {})(dict(params, time_manager=pp.TimeManager([0, 1.0], dt or 1.0,
                                                                                             constant_dt=True)))
        model.prepare_simulation()
        model.time_manager.increase_time()
        model.time_manager.increase_time_index()
        model.before_nonlinear_loop()
        yield model, build, dt


def _bridged(model, build):
    """(problem, column_map, row_map) of a bridge; the bridges without row maps keep the model's equation order."""
    out = build(model)
    if not isinstance(out, tuple):
        return out, np.arange(out.num_dofs), np.arange(out.num_dofs)
    return out[0], out[1], out[2] if len(out) > 2 else np.arange(out[0].num_dofs)


def _linearize(prob, x, x_prev, dt):
    return prob.linearize(x, x_prev) if dt is None else prob.linearize(x, x_prev, dt)


def _check_live(model, build, dt, to_host, n_before=3):
    """The bridged problem linearizes to the model's own J and -R at the model's iterate ``n_before``."""
    es = model.equation_system
    for _ in range(n_before):
        model.before_nonlinear_iteration()
        model.assemble_linear_system()
        model.after_nonlinear_iteration(model.solve_linear_system())
    model.before_nonlinear_iteration()
    model.assemble_linear_system()
    A, rhs = model.linear_system
    x_prev, x_it = es.get_variable_values(time_step_index=0), es.get_variable_values(iterate_index=0)
    prob, cm, rm = _bridged(model, build)
    assert prob.nd == 2 and (not hasattr(prob, "fractures") or len(prob.fractures) == 2)
    prob.discretize()
    J, r = _linearize(prob, x_it[cm], x_prev[cm], dt)
    Aref = A.tocsr()[rm][:, cm]
    assert abs(J.to_scipy() - Aref).max() <= 1e-10 * abs(Aref).max(), type(model).__mro__[2]
    assert np.abs(to_host(r) - rhs[rm]).max() <= 1e-10 * max(np.abs(rhs).max(), 1e-3 * abs(A).max())
    return prob, cm


@needs_reference
def test_live_2d_models_through_the_bridges(host_build):
    pp = load_porepy()
    seen = set()
    for model, build, dt in _live_models(pp):
        _check_live(model, build, dt, lambda t: t.numpy())
        seen.add(build.__name__)
        if build.__name__.startswith("fractured"):
            fracs = model.mdg.subdomains(dim=1)
            assert len(fracs) == 2 and any(np.any(f.tags["domain_boundary_faces"]) for f in fracs)
    assert len(seen) == 5


@needs_reference
def test_live_crossing_lines_are_refused():
    """Two crossing line fractures: the 0-D intersection point is refused by every contact bridge."""
    pp = load_porepy()
    from porepy_b200 import model_bridge as mb
    mdg = pp.meshing.cart_grid([np.array([[0.5, 0.5], [0.25, 0.75]]), np.array([[0.25, 0.75], [0.5, 0.5]])], [8, 8],
                               physdims=[1, 1])
    assert sorted({g.dim for g in mdg.subdomains()}) == [0, 1, 2]
    for build in (mb.fractured_momentum_from_model, mb.fractured_poromechanics_from_model,
                  mb.fractured_thermoporomechanics_from_model):
        with pytest.raises(NotImplementedError, match="0-D subdomains .* in a 2-D matrix"):
            build(SimpleNamespace(mdg=mdg))


# ---------------------------------------------------------------- GPU


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_model_2d_gpu(name):
    prob, d = load_problem(name)
    prob.discretize()
    check(prob, d, lambda t: t.cpu().numpy(), _cuda, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CONTACT + CONTACT_FLOW)
def test_time_step_2d_with_device_gmres_gpu(name, monkeypatch):
    """A time step of every 2-D contact fixture with ``krylov.gmres_solver(prob.preconditioner_groups())``: no matrix
    leaves the device, and the loop reaches the reference's converged state."""
    from porepy_b200.sparse import DeviceCsr
    prob, d = load_problem(name)
    prob.discretize()
    solver = krylov.gmres_solver(prob.preconditioner_groups())

    def refuse(self):
        raise AssertionError("a matrix left the device")
    monkeypatch.setattr(DeviceCsr, "to_scipy", refuse)
    x, hist = _time_step(prob, d, d["previous"][d["column_map"]], solver)
    xh = x.cpu().numpy()
    check_history_and_state(prob, d, xh, hist, name, solver)
    monkeypatch.undo()
    assert solver.last_info["converged"] and solver.last_info["cuda_graph"]


@pytest.mark.gpu
def test_live_2d_models_reach_the_reference_state_gpu():
    """Where the reference is present: the five live 2-D models through the bridges linearize to the model's J and -R on
    the device, then take a time step with the device GMRES (contact) or BiCGStab (no fractures) and reach the state of
    the reference's own Newton loop."""
    if not reference_available():
        pytest.skip("oracle/_ref not present")
    pp = load_porepy()
    for model, build, dt in _live_models(pp):
        es = model.equation_system
        x_prev = es.get_variable_values(time_step_index=0)
        prob, cm = _check_live(model, build, dt, lambda t: t.cpu().numpy(), n_before=1)
        norms = []
        for _ in range(30):                                        # the reference's loop to convergence
            model.before_nonlinear_iteration()
            model.assemble_linear_system()
            norms.append(np.linalg.norm(model.linear_system[1]))
            if norms[-1] < 1e-12 * norms[0] or norms[-1] < 1e-15:
                break
            model.after_nonlinear_iteration(model.solve_linear_system())
        x_ref = es.get_variable_values(iterate_index=0)[cm]
        if hasattr(prob, "preconditioner_groups"):
            solver = krylov.gmres_solver(prob.preconditioner_groups())
            x, hist = prob.time_step(x_prev[cm], solver, tol=1e-11) if dt is None else \
                prob.time_step(x_prev[cm], dt, solver, tol=1e-11)
        else:
            x, hist = prob.time_step(x_prev[cm], dt, tol=1e-11)
        assert hist[-1]["residual"] <= 1e-10 * hist[0]["residual"], hist
        assert np.linalg.norm(x.cpu().numpy() - x_ref) <= 1e-8 * max(np.linalg.norm(x_ref), 1e-12), type(prob)
