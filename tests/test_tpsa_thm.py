"""TPSA thermo-poromechanics (``porepy_b200.TpsaThermoporomechanics``, ``pb_tpsa_thm_system`` /
``pb_tpsa_thm_balance_rows``, csrc/tpsa_system.cuh with two scalar balances) against the unmodified reference's
``pp.Thermoporomechanics`` + ``TpsaPoromechanicsMixin``: the couplings the fixtures carry, Jacobian and -R at the zero
state and at an intermediate Newton iterate of two time steps, the residual histories and converged states (fixtures of
tools/make_tpsa_thm_golden.py), a live stock model through the bridge, the refusals and the bench-size mesh.  The checks
themselves are those of tpsa_checks.py.
CPU: host build of tpsa_system.cuh + the scipy stand-in for the device sparse algebra."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200.tpsa_thermoporomech import TpsaThermoporomechanics
from golden_io import case_names, load_case
from tpsa_checks import (OWN, check_bridge_linearization, check_full_size_linearization, check_linearizations,
                         check_single_grid_refusals, check_time_steps, compare_with_host_build, csr,
                         newton_reaches_reference, newton_states, scalar_bc, use_host_build)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsathm_")
FLUID = ("compressibility", "density", "viscosity", "reference_pressure", "reference_temperature")
THERMAL = ("thermal_expansion", "heat_capacity", "conductivity")


def _constants(d):
    fluid = {k: float(d[k]) for k in FLUID}
    fluid.update({k: float(d["fluid_" + k]) for k in THERMAL})
    solid = {k: float(d[k]) for k in ("reference_porosity", "biot_coefficient", "bulk_modulus")}
    solid.update({k: float(d["solid_" + k]) for k in THERMAL + ("density",)})
    return fluid, solid


def _problem(name):
    c = load_case(name)
    d, g = c.raw, c.g
    nf = g.num_faces
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(d["K"]),
                                           "bc": scalar_bc(d, "flow", nf)})
    pb.initialize_data(data, "fourier", {"bc": scalar_bc(d, "fourier", nf)})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(d["mu"], d["lmbda"]),
                                           "bc": c.bc})
    fluid, solid = _constants(d)
    prob = TpsaThermoporomechanics(g, data, fluid, solid, d["flow_bc_values"], d["fourier_bc_values"], d["bc_values"],
                                   scalar_bc(d, "ff", nf), d["ff_values"], scalar_bc(d, "ef", nf), d["ef_values"],
                                   body_force=d["body_force"], angular_source=d["angular_source"],
                                   mass_source=d["mass_source"], fluid_source=d["fluid_source"])
    prob.column_map, prob.row_map = d["column_map"], d["row_map"]
    return prob, d


def _linearizations(prob, d):
    return check_linearizations(prob, d, newton_states(d), 1e-12, OWN, float(d["dt"]))


@pytest.fixture()
def host_build(monkeypatch):
    use_host_build(monkeypatch)


def test_fixtures_present():
    assert {int(load_case(n).raw["dim"]) for n in CASES} == {2, 3}


@pytest.mark.parametrize("name", CASES)
def test_fixtures_couple_the_fields(name):
    """The reference's Jacobians couple mass to T and energy to p_t and p; the mechanics rows have no T column."""
    d = load_case(name).raw
    nd = int(d["dim"])
    B = nd + (3 if nd == 3 else 1) + 3
    for jk in ("J0", "s0_J", "s1_J"):
        J = csr(d, jk)[d["row_map"]][:, d["column_map"]].tocsr()
        blk = lambda rows, col: J[rows::B][:, col::B]  # noqa: E731
        assert abs(blk(B - 2, B - 1)).max() > 0, jk                  # mass, T
        assert abs(blk(B - 1, B - 3)).max() > 0, jk                  # energy, p_t
        assert abs(blk(B - 1, B - 2)).max() > 0, jk                  # energy, p
        mech = J[np.flatnonzero(np.arange(J.shape[0]) % B < B - 2)]
        assert mech[:, B - 1::B].nnz == 0 or not mech[:, B - 1::B].data.any(), jk


@pytest.mark.parametrize("name", CASES)
def test_host_build_matches_reference(name, host_build):
    prob, d = _problem(name)
    _linearizations(prob, d)
    check_time_steps(prob, d, 1e-10)


def test_refusals_host():
    g = pb.cart_grid_2d([3, 2])
    nf = g.num_faces
    fluid = dict(compressibility=0.1, density=1.0, viscosity=1.0, thermal_expansion=0.1, heat_capacity=1.0,
                 conductivity=1.0, reference_temperature=0.3)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.5, bulk_modulus=2.0, thermal_expansion=0.1,
                 heat_capacity=1.0, conductivity=1.0, density=2.0)
    args = (np.zeros(nf), np.zeros(nf), np.zeros(2 * nf), None, np.zeros(nf), None, np.zeros(nf))
    for k in ("compressibility", "density", "viscosity"):
        for bad in (0.0, -1.0, np.nan):
            with pytest.raises(ValueError, match="must be finite and > 0"):
                TpsaThermoporomechanics(g, {}, dict(fluid, **{k: bad}), solid, *args)
    with pytest.raises(ValueError, match="fluid heat_capacity must be finite"):
        TpsaThermoporomechanics(g, {}, dict(fluid, heat_capacity=np.inf), solid, *args)
    with pytest.raises(ValueError, match="fourier_bc_values must have"):
        TpsaThermoporomechanics(g, {}, fluid, solid, np.zeros(nf), np.zeros(2), *args[2:])
    with pytest.raises(ValueError, match="no dof maps"):
        TpsaThermoporomechanics(g, {}, fluid, solid, *args).to_model_order(sps.eye(6 * g.num_cells))
    assert TpsaThermoporomechanics(g, {}, fluid, solid, *args).num_dofs == 6 * g.num_cells
    from porepy_b200 import model_bridge
    check_single_grid_refusals(model_bridge.tpsa_thermoporomechanics_from_model,
                               model_bridge.tpsa_poromechanics_from_model,
                               ["mass_balance_equation", "energy_balance_equation"],
                               "tpsa_thermoporomechanics_from_model")


# ---- the stock model through the plugin's bridge -----------------------------------------------------------------


def _stock_model(pp, nd):
    from make_tpsa_thm_golden import ThermalSetup

    class Stock(ThermalSetup, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Thermoporomechanics):
        pass
    fluid = pp.FluidComponent(compressibility=0.02, viscosity=0.7, density=1.1, thermal_expansion=0.15,
                              specific_heat_capacity=1.8, thermal_conductivity=0.6)
    solid = pp.SolidConstants(porosity=0.15, biot_coefficient=0.6, lame_lambda=1.5, shear_modulus=1.0, permeability=2.0,
                              thermal_expansion=0.05, specific_heat_capacity=1.2, thermal_conductivity=0.9, density=2.2)
    m = Stock({"times_to_export": [], "tpsa_nd": nd, "cell_size": 0.25, "seed": 9,
               "material_constants": {"fluid": fluid, "solid": solid},
               "reference_variable_values": pp.ReferenceVariableValues(pressure=0.1, temperature=0.2)})
    m.prepare_simulation()
    rng = np.random.default_rng(nd)
    x = 0.1 * rng.standard_normal(m.equation_system.num_dofs())
    m.equation_system.set_variable_values(x, iterate_index=0)
    m.equation_system.set_variable_values(0.5 * x, time_step_index=0)
    m.update_derived_quantities()         # upwind directions of the iterate, as after a Newton update
    return m


def _check_bridge(nd):
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    prob, cols, rows = plugin(pp).tpsa_thermoporomechanics_from_model(m)
    assert prob.num_dofs == m.equation_system.num_dofs()
    check_bridge_linearization(m, prob, cols, rows, float(m.time_manager.dt))
    with pytest.raises(NotImplementedError, match="tpsa_thermoporomechanics_from_model"):
        plugin(pp).tpsa_poromechanics_from_model(m)


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
    check_time_steps(prob, d, 1e-10)
    compare_with_host_build(lambda: _linearizations(*_problem(name)), dev)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_newton_with_block_jacobi(name):
    """The Newton loop with the device 6 x 6 / 9 x 9 block-Jacobi BiCGStab reaches the reference's converged states."""
    newton_reaches_reference(*_problem(name), 1e-10)


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("nd", [2, 3])
def test_gpu_bridge(nd):
    _check_bridge(nd)


@pytest.mark.gpu
def test_gpu_refusals():
    import torch
    prob, d = _problem(CASES[0])
    prob.discretize()
    fg, nc = prob._fg, prob.nc
    b = torch.zeros(prob.num_dofs, dtype=torch.float64, device="cuda")
    r = torch.zeros(2 * nc, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="2 num_cells x 3 num_cells"):
        fg.tpsa_thm_balance_rows(prob.A, pb.DeviceCsr(sps.csr_matrix((2 * nc, 2 * nc))), r, b)
    with pytest.raises(ValueError, match="not the TPSA thermo-poromechanics system"):
        fg.tpsa_thm_balance_rows(pb.DeviceCsr(sps.eye(prob.num_dofs, format="csr")),
                                 pb.DeviceCsr(sps.csr_matrix((2 * nc, 3 * nc))), r, b)
    # the handle holds the five-field pattern: the four-field row writer refuses it
    with pytest.raises(ValueError, match="pb_tpsa_poro_system has not been called"):
        fg.tpsa_poro_fluid_rows(prob.A, pb.DeviceCsr(sps.csr_matrix((nc, 2 * nc))), r[:nc], b)


@pytest.mark.gpu
def test_gpu_full_size_matches_device_ad_assembly():
    """998,250 tetrahedra, seeded inputs: J of the second linearization of a time step against the field-ordered
    porepy_b200.ad bmat assembly of the same matrices (mechanics rows from pb.Tpsa, mass and energy rows from the AD
    chain) permuted to the cell-interleaved order; two linearizations bit-identical."""
    from porepy_b200 import ad
    from porepy_b200.sparse import DeviceCsr

    def balance_rows(prob, x, x_prev, dt):
        jf, nc = ad.assemble(prob.balance_equations(x, x_prev, dt))[0].to_scipy(), prob.nc
        return [[DeviceCsr(jf[i * nc:(i + 1) * nc, j * nc:(j + 1) * nc].tocsr()) for j in range(3)] for i in range(2)]
    check_full_size_linearization("thermoporomechanics", 31, balance_rows)
