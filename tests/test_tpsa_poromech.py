"""TPSA poromechanics (``porepy_b200.TpsaPoromechanics``, ``pb_tpsa_poro_system`` / ``pb_tpsa_poro_fluid_rows``,
csrc/tpsa_system.cuh) against the unmodified reference's ``pp.Poromechanics`` + ``TpsaPoromechanicsMixin``: Jacobian and
-R at the zero state and at an intermediate Newton iterate of two time steps, the residual histories and converged
states (fixtures of tools/make_tpsa_poromech_golden.py), a live stock model through the bridge, the refusals and the
bench-size mesh.  The checks themselves are those of tpsa_checks.py.
CPU: host build of tpsa_system.cuh + the scipy stand-in for the device sparse algebra."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.tpsa_poromech import TpsaPoromechanics
from golden_io import case_names, load_case
from tpsa_checks import (OWN, check_bridge_linearization, check_full_size_linearization, check_linearizations,
                         check_single_grid_refusals, check_time_steps, compare_with_host_build,
                         newton_reaches_reference, newton_states, scalar_bc, use_host_build)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsaporo_")


def _problem(name):
    c = load_case(name)
    d, g = c.raw, c.g
    nf = g.num_faces
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(d["K"]),
                                           "bc": scalar_bc(d, "flow", nf)})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(d["mu"], d["lmbda"]),
                                           "bc": c.bc})
    fluid = {k: float(d[k]) for k in ("compressibility", "density", "viscosity", "reference_pressure")}
    solid = {k: float(d[k]) for k in ("reference_porosity", "biot_coefficient", "bulk_modulus")}
    prob = TpsaPoromechanics(g, data, fluid, solid, d["flow_bc_values"], d["bc_values"], scalar_bc(d, "ff", nf),
                             d["ff_values"], body_force=d["body_force"], angular_source=d["angular_source"],
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
def test_host_build_matches_reference(name, host_build):
    prob, d = _problem(name)
    _linearizations(prob, d)
    check_time_steps(prob, d, 1e-10)


def test_refusals_host():
    g1 = SimpleNamespace(dim=1, num_cells=2, num_faces=3)
    fluid = dict(compressibility=0.1, density=1.0, viscosity=1.0)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.5, bulk_modulus=2.0)
    with pytest.raises(NotImplementedError, match="only implemented for 2d and 3d"):
        TpsaPoromechanics(g1, {}, fluid, solid, np.zeros(3), np.zeros(3), None, np.zeros(3))
    g = pb.cart_grid_2d([3, 2])
    nf = g.num_faces
    args = (np.zeros(nf), np.zeros(2 * nf), None, np.zeros(nf))
    for k in ("compressibility", "density", "viscosity"):
        for bad in (0.0, -1.0, np.nan):
            with pytest.raises(ValueError, match="must be finite and > 0"):
                TpsaPoromechanics(g, {}, dict(fluid, **{k: bad}), solid, *args)
    for bad in (np.nan, np.inf):
        with pytest.raises(ValueError, match="Biot coefficient"):
            TpsaPoromechanics(g, {}, fluid, dict(solid, biot_coefficient=bad), *args)
    with pytest.raises(ValueError, match="mech_bc_values must have"):
        TpsaPoromechanics(g, {}, fluid, solid, np.zeros(nf), np.zeros(nf), None, np.zeros(nf))
    with pytest.raises(ValueError, match="no dof maps"):
        TpsaPoromechanics(g, {}, fluid, solid, *args).to_model_order(sps.eye(5 * g.num_cells))
    from porepy_b200 import model_bridge
    check_single_grid_refusals(model_bridge.tpsa_poromechanics_from_model, model_bridge.tpsa_momentum_from_model,
                               ["mass_balance_equation"], "tpsa_poromechanics_from_model")


# ---- the stock model through the plugin's bridge -----------------------------------------------------------------


def _stock_model(pp, nd):
    from make_tpsa_poromech_golden import Setup

    class Stock(Setup, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Poromechanics):
        pass
    fluid = pp.FluidComponent(compressibility=0.02, viscosity=0.7, density=1.1)
    solid = pp.SolidConstants(porosity=0.15, biot_coefficient=0.6, lame_lambda=1.5, shear_modulus=1.0, permeability=2.0)
    m = Stock({"times_to_export": [], "tpsa_nd": nd, "cell_size": 0.25, "seed": 9,
               "material_constants": {"fluid": fluid, "solid": solid},
               "reference_variable_values": pp.ReferenceVariableValues(pressure=0.1)})
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
    check_bridge_linearization(m, *plugin(pp).tpsa_poromechanics_from_model(m), float(m.time_manager.dt))


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
    # patterns not compared: the device SpGEMM keeps exact cancellations of div @ flux in the fluid rows, scipy drops them
    compare_with_host_build(lambda: _linearizations(*_problem(name)), dev)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_newton_with_block_jacobi(name):
    """The Newton loop with the device block-Jacobi BiCGStab reproduces the reference's converged states."""
    newton_reaches_reference(*_problem(name), 1e-8)


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
    g, fg = prob.sd, prob._fg
    nc = g.num_cells
    codes, rob = fv.tpsa_bc_arrays(prob.data[pb.PARAMETERS]["mechanics"]["bc"], 2, g.num_faces)
    flags = np.zeros(g.num_faces, np.uint8)
    flags[g.get_all_boundary_faces()] = 1
    fp = prob._operands().div.matmul(prob._operands().flux)
    args = [d["mu"], d["lmbda"], np.full(nc, 0.5), g.cell_volumes, codes, rob, flags, g.face_areas, fp]
    for i, what in ((1, "first Lame parameter"), (2, "Biot coefficient")):
        bad = np.array(args[i], float)
        bad[3] = np.nan
        with pytest.raises(ValueError, match=what):
            fg.tpsa_poro_system(2, *args[:i], bad, *args[i + 1:])
    with pytest.raises(ValueError, match="only implemented for 2d and 3d"):
        fg.tpsa_poro_system(1, *args)
    with pytest.raises(ValueError, match="flux pattern"):
        fg.tpsa_poro_system(2, *args[:-1], pb.DeviceCsr(sps.eye(nc + 1, format="csr")))
    b = torch.zeros(prob.num_dofs, dtype=torch.float64, device="cuda")
    r = torch.zeros(nc, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="num_cells x 2 num_cells"):
        fg.tpsa_poro_fluid_rows(prob.A, pb.DeviceCsr(sps.eye(nc, format="csr")), r, b)
    with pytest.raises(ValueError, match="not the TPSA poromechanics system"):
        fg.tpsa_poro_fluid_rows(pb.DeviceCsr(sps.eye(prob.num_dofs, format="csr")),
                                pb.DeviceCsr(sps.csr_matrix((nc, 2 * nc))), r, b)


@pytest.mark.gpu
def test_gpu_full_size_matches_device_ad_assembly():
    """998,250 tetrahedra, seeded inputs: J of the second linearization of a time step against the field-ordered
    porepy_b200.ad bmat assembly of the same matrices (mechanics rows from pb.Tpsa, fluid rows from the AD chain) permuted
    to the cell-interleaved order; two linearizations bit-identical."""
    from porepy_b200.sparse import DeviceCsr

    def fluid_rows(prob, x, x_prev, dt):
        jf = prob.fluid_equation(x, x_prev, dt).jac.to_scipy()
        return [[DeviceCsr(jf[:, :prob.nc]), DeviceCsr(jf[:, prob.nc:])]]
    check_full_size_linearization("poromechanics", 29, fluid_rows)
