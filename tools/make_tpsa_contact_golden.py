"""Generate tests/golden/tpsacontact_*.npz: TPSA elasticity with a fracture in frictional contact, the unmodified
reference's ``pp.MomentumBalance`` with ``TpsaMomentumBalanceMixin`` on the fractured domains of
tools/make_contact_golden.py (``Model``: the unit cube, 4^3 cells, one plane fracture; ``Model2d``: the unit square,
8 x 8 cells, one line fracture), under the four loads ``sliding``, ``sticking``, ``open`` and ``mixed``.  Each fixture
holds the keys of ``contact_model.npz`` (grid, bc, mortar projections, local coordinates, contact constants, the
Jacobian / -R at the second Newton iterate, the residual history and the converged state), the TPSA inputs of
``tpsa_model_*.npz`` (mu, lmbda, the evaluated boundary operator, body force and sources), the row map and the Jacobian
and -R at the zero state.  ``column_map`` / ``row_map`` give the model dof / row of every unknown / equation in the order
[u_c, r_c, p_c per cell | contact traction | interface displacement] / [three balances per cell | interface force
balance | normal law | tangential law].  Every case asserts the contact regime it is meant to exercise.  The prefix
``tpsacontact_`` (as ``tpsaporo_`` / ``tpsathm_``) keeps these fixtures out of the ``tpsa_*`` set that
tests/test_tpsa.py and tests/test_tpsa_system.py read as discretization fixtures.
   python tools/make_tpsa_contact_golden.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_contact_golden import OUT, Model, Model2d, pp  # noqa: E402
from make_golden import grid_arrays  # noqa: E402
from make_mdflow_golden import put_csr  # noqa: E402
from make_tpsa_model_golden import interleave  # noqa: E402


def regimes(t, nd, mu):
    """(open, sticking, sliding) masks of the fracture cells of the converged traction t (nk x nd, local frame)."""
    tn, tt = t[:, nd - 1], np.linalg.norm(t[:, :nd - 1], axis=1)
    is_open = np.abs(tn) < 1e-12
    sliding = ~is_open & (tt >= mu * np.abs(tn) * (1 - 1e-8))
    return is_open, ~is_open & ~sliding, sliding


def case(scenario, name, base):
    solid = pp.SolidConstants(lame_lambda=2.0, shear_modulus=1.5, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1)
    M = type("TpsaContact", (pp.models.momentum_balance.TpsaMomentumBalanceMixin, base), {})
    m = M({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 1.0, constant_dt=True),
           "material_constants": {"solid": solid}})
    m.scenario = scenario
    m.prepare_simulation()
    es, mdg = m.equation_system, m.mdg
    nd = m.nd
    nr = m.rotation_dimension()
    mat, frac, intf = mdg.subdomains(dim=nd)[0], mdg.subdomains(dim=nd - 1)[0], mdg.interfaces()[0]
    nc = mat.num_cells

    def dofs(name):
        return es.dofs_of([v for v in es.variables if v.name == name])

    def ev(op):
        v = es.evaluate(op)
        return np.asarray(getattr(v, "val", v), float)

    def scalar(op):
        return float(np.atleast_1d(ev(op))[0])
    d = {f"matrix__{k}": v for k, v in grid_arrays(mat).items()}
    prm = mdg.subdomain_data(mat)[pp.PARAMETERS][m.stress_keyword]
    bc, C = prm["bc"], prm["fourth_order_tensor"]
    J0, rhs0 = es.assemble()
    idx = es.assembled_equation_indices
    solid_mass = [eq for eq in es.equations if eq.startswith("solid_mass_equation")][0]
    cols = np.concatenate([interleave([dofs(m.displacement_variable), dofs(m.rotation_stress_variable),
                                       dofs(m.total_pressure_variable)], nd, nr, nc),
                           dofs(m.contact_traction_variable), dofs(m.interface_displacement_variable)])
    rows = np.concatenate([interleave([idx["momentum_balance_equation"], idx["angular_momentum_balance_equation"],
                                       idx[solid_mass]], nd, nr, nc)]
                          + [idx[eq] for eq in ("interface_force_balance_equation",
                                                "normal_fracture_deformation_equation",
                                                "tangential_fracture_deformation_equation")])
    assert np.array_equal(np.sort(cols), np.arange(es.num_dofs()))
    assert np.array_equal(np.sort(rows), np.arange(es.num_dofs()))
    bmask = np.zeros(mat.num_faces, bool)
    bmask[mat.get_all_boundary_faces()] = True
    d.update(dim=np.int64(nd), mu=C.mu, lmbda=C.lmbda, boundary_faces=bmask, bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu,
             bc_is_rob=bc.is_rob, bc_is_internal=np.asarray(bc.is_internal, bool),
             bc_robin_weight=np.asarray(bc.robin_weight, float), bc_basis=np.asarray(bc.basis, float),
             bc_values=ev(m.combine_boundary_operators_mechanical_stress([mat])), body_force=ev(m.body_force([mat])),
             angular_source=np.broadcast_to(ev(m.source_angular_momentum([mat])), (nr * nc,)).copy(),
             mass_source=np.broadcast_to(ev(m.solid_mass_source([mat])), (nc,)).copy(),
             rhs0=np.asarray(rhs0, float), column_map=cols, row_map=rows)
    put_csr(d, "J0", J0)
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(30):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 1:
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-14 * norms[0]:      # to round-off: the stored state is the yardstick of the device solves
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    assert norms[-1] < 1e-14 * norms[0], norms
    rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             mortar_sign=sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), mortar_volumes=intf.cell_volumes,
             numerical_constant=np.float64(scalar(m.contact_mechanics_numerical_constant([frac]))),
             characteristic_traction=np.float64(scalar(m.characteristic_contact_traction([frac]))),
             friction_coefficient=np.float64(scalar(m.friction_coefficient([frac]))),
             dilation_angle=np.float64(m.solid.dilation_angle), reference_gap=np.float64(m.solid.fracture_gap),
             open_state_tolerance=np.float64(m.numerical.open_state_tolerance))
    put_csr(d, "local_coordinates", rot)
    for key in ("mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg", "secondary_to_mortar_int"):
        put_csr(d, key, getattr(intf, key)())
    t = d["solution"][dofs(m.contact_traction_variable)].reshape(-1, nd)
    is_open, sticking, sliding = regimes(t, nd, float(d["friction_coefficient"]))
    want = {"sliding": sliding.any(), "sticking": sticking.any() and not is_open.any(), "open": is_open.all(),
            "mixed": is_open.any() and (~is_open).any()}[scenario]
    assert want, (name, is_open, sticking, sliding)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "dofs", es.num_dofs(), "Newton residuals", ["%.1e" % v for v in norms], "open / sticking / sliding",
          int(is_open.sum()), int(sticking.sum()), int(sliding.sum()))


if __name__ == "__main__":
    for scen in ("sliding", "sticking", "open", "mixed"):
        case(scen, f"tpsacontact_{scen}", Model)
    for scen in ("sliding", "mixed"):
        case(scen, f"tpsacontact_2d_{scen}", Model2d)
