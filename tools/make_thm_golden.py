"""Generate tests/golden/thm_model.npz: Jacobian, residual, residual history and converged state of one implicit time step
of the unmodified reference's ``pp.Thermoporomechanics`` (momentum, mass and energy balance; Biot and thermal stress
coupling through ``pp.Biot``; compressible, thermally expanding fluid; upwinded mass and enthalpy fluxes; Fourier flux
discretized at the reference porosity, the model's default) on a small 3-D grid -- BASELINE config[4] without
the fractures -- and tests/golden/thm_model_2d.npz, the same on the 2-D grid of ``make_poromech_golden.Model2d``.  Run in
the build container:  python tools/make_thm_golden.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_porepy  # noqa: E402
from make_golden import grid_arrays  # noqa: E402
from make_mdflow_golden import put_csr  # noqa: E402
import make_poromech_golden as pm  # noqa: E402

pp = load_porepy()
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
# geometry, permeability, stiffness and the flow / mechanics boundary conditions of the poromechanics fixture
Shared = type("Shared", (), {k: v for k, v in pm.Model.__dict__.items() if callable(v) and not k.startswith("__")})


class Model(Shared, pp.Thermoporomechanics):
    def bc_type_fourier_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_type_enthalpy_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_values_temperature(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros(bg.num_cells)
        v[s.west] = 0.5 + 0.2 * bg.cell_centers[2, s.west]
        return v


Shared2d = type("Shared2d", (), {k: v for k, v in pm.Model2d.__dict__.items() if callable(v) and not k.startswith("__")})


class Model2d(Shared2d, Model):
    def bc_values_temperature(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros(bg.num_cells)
        v[s.west] = 0.5 + 0.2 * bg.cell_centers[1, s.west]
        return v


def main(model_class=Model, name="thm_model"):
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7, thermal_expansion=0.03,
                              specific_heat_capacity=2.0, thermal_conductivity=0.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0,
                              thermal_expansion=0.02, specific_heat_capacity=1.5, thermal_conductivity=1.1, density=2.5)
    m = model_class({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 0.25, constant_dt=True),
               "material_constants": {"fluid": fluid, "solid": solid}})
    m.prepare_simulation()
    es = m.equation_system
    sd = m.mdg.subdomains()[0]
    assert [v.name for v in es.variables] == ["u", "pressure", "temperature"]
    data = m.mdg.subdomain_data(sd)
    d = grid_arrays(sd)
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(15):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 2:
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-12 * norms[0]:
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    fl, so = m.fluid.reference_component, m.solid
    bg = m.mdg.subdomain_to_boundary_grid(sd)
    proj = bg.projection()
    proj3 = sps.kron(proj, sps.eye(sd.dim)).tocsr()
    prm = data[pp.PARAMETERS]
    p_ref, t_ref = m.reference_variable_values.pressure, m.reference_variable_values.temperature
    pb_, tb = proj.T @ m.bc_values_pressure(bg), proj.T @ m.bc_values_temperature(bg)
    rho_b = fl.density * np.exp(fl.compressibility * (pb_ - p_ref) - fl.thermal_expansion * (tb - t_ref))
    kb = so.lame_lambda + 2 * so.shear_modulus / 3
    bcf, bct, bcm = prm["flow"]["bc"], prm["fourier_discretization"]["bc"], prm["mechanics"]["bc"]
    bff, bfe = m.bc_type_fluid_flux(sd), m.bc_type_enthalpy_flux(sd)
    svm = prm["mechanics"]["scalar_vector_mappings"]
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             dt=np.float64(m.time_manager.dt),
             compressibility=np.float64(fl.compressibility), density=np.float64(fl.density), viscosity=np.float64(fl.viscosity),
             fluid_thermal_expansion=np.float64(fl.thermal_expansion), fluid_heat_capacity=np.float64(fl.specific_heat_capacity),
             fluid_conductivity=np.float64(fl.thermal_conductivity), reference_pressure=np.float64(p_ref),
             reference_temperature=np.float64(t_ref), reference_porosity=np.float64(so.porosity),
             biot_coefficient=np.float64(so.biot_coefficient), solid_thermal_expansion=np.float64(so.thermal_expansion),
             solid_heat_capacity=np.float64(so.specific_heat_capacity), solid_conductivity=np.float64(so.thermal_conductivity),
             solid_density=np.float64(so.density),
             n_inv=np.float64((so.biot_coefficient - so.porosity) * (1 - so.biot_coefficient) / kb),
             K=prm["flow"]["second_order_tensor"].values, C=prm["mechanics"]["fourth_order_tensor"].values,
             alpha_flow=svm["flow"].values, alpha_thermal=svm[m.enthalpy_keyword].values,
             flow_is_dir=bcf.is_dir, flow_is_neu=bcf.is_neu,
             flow_bc_values=np.where(bcf.is_dir, pb_, proj.T @ m.bc_values_darcy_flux(bg)),
             fourier_is_dir=bct.is_dir, fourier_is_neu=bct.is_neu,
             fourier_bc_values=np.where(bct.is_dir, tb, proj.T @ m.bc_values_fourier_flux(bg)),
             ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             ff_values=np.where(bff.is_dir, rho_b / fl.viscosity, proj.T @ m.bc_values_fluid_flux(bg)),
             ef_is_dir=bfe.is_dir, ef_is_neu=bfe.is_neu,
             ef_values=np.where(bfe.is_dir, fl.specific_heat_capacity * (tb - t_ref) * rho_b / fl.viscosity,
                                proj.T @ m.bc_values_enthalpy_flux(bg)),
             mech_is_dir=bcm.is_dir, mech_is_neu=bcm.is_neu, mech_is_rob=bcm.is_rob, mech_is_internal=bcm.is_internal,
             mech_bc_values=np.where(bcm.is_dir.ravel("F"), proj3.T @ m.bc_values_displacement(bg),
                                     proj3.T @ m.bc_values_stress(bg)))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "cells", sd.num_cells, "dofs", es.num_dofs(), "Newton residuals", ["%.2e" % v for v in norms])


if __name__ == "__main__":
    main()
    main(Model2d, "thm_model_2d")
