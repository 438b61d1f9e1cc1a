"""Generate tests/golden/poromech_model.npz: the Jacobian, residual, residual history and converged state of one implicit
time step of the unmodified reference's ``pp.Poromechanics`` (Biot coupling through ``pp.Biot``, compressible fluid,
upwinded mobility, stabilised poromechanical porosity) on a small 3-D grid -- BASELINE config[3] in miniature -- and
tests/golden/poromech_model_2d.npz, the same on a 10 x 8 Cartesian grid in 2-D (``Model2d``).  Run in the build
container:  python tools/make_poromech_golden.py"""
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

pp = load_porepy()
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


class Model(pp.Poromechanics):
    def set_domain(self):
        self._domain = pp.Domain({"xmin": 0, "xmax": 1.25, "ymin": 0, "ymax": 1, "zmin": 0, "zmax": 1})

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": 0.25}

    def permeability(self, subdomains):
        vals = []
        for sd in subdomains:
            rng = np.random.default_rng(sd.num_cells)
            nc = sd.num_cells
            t = np.zeros((3, 3, nc))
            t[0, 0], t[1, 1], t[2, 2] = 1 + rng.random((3, nc))
            o = 0.3 * rng.random((3, nc))
            t[0, 1] = t[1, 0] = o[0]
            t[0, 2] = t[2, 0] = o[1]
            t[1, 2] = t[2, 1] = o[2]
            vals.append(t.reshape(9, nc).ravel("F"))
        return pp.wrap_as_dense_ad_array(np.hstack(vals) if vals else np.zeros(0), name="permeability")

    def stiffness_tensor(self, sd):
        rng = np.random.default_rng(7 + sd.num_cells)
        return pp.FourthOrderTensor(1.5 * np.exp(0.3 * rng.standard_normal(sd.num_cells)),
                                    2.0 * np.exp(0.3 * rng.standard_normal(sd.num_cells)))

    def bc_type_darcy_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_type_fluid_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_values_pressure(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros(bg.num_cells)
        v[s.west] = 1.0 + bg.cell_centers[1, s.west]
        return v

    def bc_type_mechanics(self, sd):
        s = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, s.west + s.bottom, "dir")
        bc.internal_to_dirichlet(sd)
        return bc

    def bc_values_stress(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((3, bg.num_cells))
        v[2, s.top] = -0.05 * bg.cell_volumes[s.top]
        return v.ravel("F")

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((3, bg.num_cells))
        v[0, s.west] = 0.01 * bg.cell_centers[2, s.west]
        return v.ravel("F")


def permeability_2d(sd, seed):
    """Seeded heterogeneous, anisotropic in-plane permeability of a 2-D (or 1-D) grid: k_xx, k_yy, k_xy; k_zz = 1."""
    rng = np.random.default_rng(seed)
    nc = sd.num_cells
    t = np.zeros((3, 3, nc))
    t[0, 0], t[1, 1] = 1 + rng.random((2, nc))
    t[0, 1] = t[1, 0] = 0.3 * rng.random(nc)
    t[2, 2] = 1.0
    return t


class Model2d(Model):
    """The 2-D counterpart of ``Model``: the same kind of loads on a 1.25 x 1 rectangle with 10 x 8 cells (west: Dirichlet
    pressure and displacement, south: fixed, north: a compressive traction)."""

    def set_domain(self):
        self._domain = pp.Domain({"xmin": 0, "xmax": 1.25, "ymin": 0, "ymax": 1})

    def meshing_arguments(self):
        return {"cell_size": 0.125}

    def permeability(self, subdomains):
        vals = [permeability_2d(sd, sd.num_cells).reshape(9, sd.num_cells).ravel("F") for sd in subdomains]
        return pp.wrap_as_dense_ad_array(np.hstack(vals) if vals else np.zeros(0), name="permeability")

    def bc_type_mechanics(self, sd):
        s = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, s.west + s.south, "dir")
        bc.internal_to_dirichlet(sd)
        return bc

    def bc_values_stress(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((2, bg.num_cells))
        v[1, s.north] = -0.05 * bg.cell_volumes[s.north]
        return v.ravel("F")

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((2, bg.num_cells))
        v[0, s.west] = 0.01 * bg.cell_centers[1, s.west]
        return v.ravel("F")


def main(model_class=Model, name="poromech_model"):
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0)
    m = model_class({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 0.25, constant_dt=True),
               "material_constants": {"fluid": fluid, "solid": solid}})
    m.prepare_simulation()
    es = m.equation_system
    sd = m.mdg.subdomains()[0]
    nc = sd.num_cells
    assert [v.name for v in es.variables] == ["pressure", "u"] and es.dofs_of([es.variables[0]])[0] == 0
    data = m.mdg.subdomain_data(sd)
    d = grid_arrays(sd)
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(12):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 1:
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-13 * norms[0]:
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    fl = m.fluid.reference_component
    bg = m.mdg.subdomain_to_boundary_grid(sd)
    proj = bg.projection()
    proj3 = sps.kron(proj, sps.eye(sd.dim)).tocsr()
    bcf = data[pp.PARAMETERS]["flow"]["bc"]
    bcm = data[pp.PARAMETERS]["mechanics"]["bc"]
    bff = m.bc_type_fluid_flux(sd)
    p_ref = m.reference_variable_values.pressure
    pb_ = proj.T @ m.bc_values_pressure(bg)
    kb = m.solid.lame_lambda + 2 * m.solid.shear_modulus / 3      # bulk modulus of the solid constants (constitutive_laws
    alpha, phi = m.solid.biot_coefficient, m.solid.porosity        # ``bulk_modulus``): enters the porosity law only
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             dt=np.float64(m.time_manager.dt), compressibility=np.float64(fl.compressibility), density=np.float64(fl.density),
             viscosity=np.float64(fl.viscosity), reference_pressure=np.float64(p_ref), reference_porosity=np.float64(phi),
             biot_coefficient=np.float64(alpha), n_inv=np.float64((alpha - phi) * (1 - alpha) / kb),
             K=data[pp.PARAMETERS]["flow"]["second_order_tensor"].values,
             C=data[pp.PARAMETERS]["mechanics"]["fourth_order_tensor"].values,
             flow_is_dir=bcf.is_dir, flow_is_neu=bcf.is_neu,
             flow_bc_values=np.where(bcf.is_dir, pb_, proj.T @ m.bc_values_darcy_flux(bg)),
             ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             ff_values=np.where(bff.is_dir, fl.density * np.exp(fl.compressibility * (pb_ - p_ref)) / fl.viscosity,
                                proj.T @ m.bc_values_fluid_flux(bg)),
             mech_is_dir=bcm.is_dir, mech_is_neu=bcm.is_neu, mech_is_rob=bcm.is_rob, mech_is_internal=bcm.is_internal,
             mech_bc_values=np.where(bcm.is_dir.ravel("F"), proj3.T @ m.bc_values_displacement(bg),
                                     proj3.T @ m.bc_values_stress(bg)))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "cells", nc, "dofs", es.num_dofs(), "Newton residuals", ["%.2e" % v for v in norms])


if __name__ == "__main__":
    main()
    main(Model2d, "poromech_model_2d")
