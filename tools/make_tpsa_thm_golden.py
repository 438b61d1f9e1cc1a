"""Generate tests/golden/tpsathm_*.npz from the unmodified reference's TPSA thermo-poromechanics model
(``pp.Thermoporomechanics`` with ``TpsaPoromechanicsMixin``: displacement, rotation stress, total pressure, fluid pressure
and temperature), run in the build container where the reference is importable.

The grids, stiffness, mechanical and Darcy boundary conditions and the fluid source are those of
``make_tpsa_poromech_golden.Setup``.  On top of them every model has a thermally expanding fluid and solid (beta_f, beta_s
non-zero), heat capacities and conductivities, a non-zero reference temperature, Dirichlet temperatures that differ on
the west and east sides (Fourier and enthalpy flux), and the flow source between the two Dirichlet pressure sides, so
the upwind direction of the mass and enthalpy fluxes changes inside the domain.  Each fixture holds the fields of
``tpsaporo_*`` (grid, coefficients, boundary data, ``J0`` / ``rhs0``, for time steps s = 0, 1 ``s{s}_previous``,
``s{s}_iterate`` with ``s{s}_J`` / ``s{s}_rhs``, ``s{s}_residual_norms``, ``s{s}_solution``) plus the Fourier and
enthalpy-flux boundary data and the thermal constants; ``column_map`` / ``row_map`` are in the cell-interleaved order
[u_c, r_c, p_t_c, p_c, T_c].

    python tools/make_tpsa_thm_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import OUT, grid_arrays, pp  # noqa: E402
from make_mdflow_golden import put_csr  # noqa: E402
from make_tpsa_poromech_golden import Setup  # noqa: E402


class ThermalSetup(Setup):
    def bc_type_fourier_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_type_enthalpy_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_values_temperature(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.full(bg.num_cells, self.reference_variable_values.temperature)
        v[s.west] = 0.9 + 0.3 * bg.cell_centers[1, s.west]
        v[s.east] = 0.1
        return v


class Model(ThermalSetup, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Thermoporomechanics):
    pass


def interleave(blocks, nd, nr, nc):
    u, r, pt, p, t = blocks
    out = np.empty((nc, nd + nr + 3), np.int64)
    out[:, :nd] = np.asarray(u).reshape(nc, nd)
    out[:, nd:nd + nr] = np.asarray(r).reshape(nc, nr)
    out[:, nd + nr] = pt
    out[:, nd + nr + 1] = p
    out[:, nd + nr + 2] = t
    return out.reshape(-1)


def constants():
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7, thermal_expansion=0.2,
                              specific_heat_capacity=2.0, thermal_conductivity=0.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=0.8,
                              thermal_expansion=0.1, specific_heat_capacity=1.5, thermal_conductivity=1.1, density=2.5)
    return fluid, solid


def case(name, nd, cell_size, seed):
    fluid, solid = constants()
    m = Model({"times_to_export": [], "tpsa_nd": nd, "cell_size": cell_size, "seed": seed,
               "time_manager": pp.TimeManager([0, 0.5], 0.25, constant_dt=True),
               "material_constants": {"fluid": fluid, "solid": solid},
               "reference_variable_values": pp.ReferenceVariableValues(pressure=0.3, temperature=0.4)})
    m.prepare_simulation()
    es = m.equation_system
    sd = m.mdg.subdomains()[0]
    nc, nf = sd.num_cells, sd.num_faces
    nr = m.rotation_dimension()
    assert np.all(es.get_variable_values(iterate_index=0) == 0)
    data = m.mdg.subdomain_data(sd)
    mk, fk, tk = m.stress_keyword, m.darcy_keyword, m.fourier_keyword
    bc, C = data[pp.PARAMETERS][mk]["bc"], data[pp.PARAMETERS][mk]["fourth_order_tensor"]
    bcf, bct = data[pp.PARAMETERS][fk]["bc"], data[pp.PARAMETERS][tk]["bc"]
    bff, bfe = m.bc_type_fluid_flux(sd), m.bc_type_enthalpy_flux(sd)
    bg = m.mdg.subdomain_to_boundary_grid(sd)
    proj = bg.projection()
    fl, so = m.fluid.reference_component, m.solid
    p_ref, t_ref = m.reference_variable_values.pressure, m.reference_variable_values.temperature
    pbv, tbv = proj.T @ m.bc_values_pressure(bg), proj.T @ m.bc_values_temperature(bg)
    rho_b = fl.density * np.exp(fl.compressibility * (pbv - p_ref) - fl.thermal_expansion * (tbv - t_ref))

    def ev(op, n):
        v = es.evaluate(op)
        return np.broadcast_to(np.asarray(getattr(v, "val", v), float), (n,)).copy()

    def dofs(var):
        return es.dofs_of([v for v in es.variables if v.name == var])
    d = grid_arrays(sd)
    d.update(kind=np.array("tpsa_thm"), mu=C.mu, lmbda=C.lmbda,
             K=data[pp.PARAMETERS][fk]["second_order_tensor"].values,
             bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=np.asarray(bc.is_internal, bool), bc_robin_weight=np.asarray(bc.robin_weight, float),
             bc_basis=np.asarray(bc.basis, float),
             flow_is_dir=bcf.is_dir, flow_is_neu=bcf.is_neu, ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             fourier_is_dir=bct.is_dir, fourier_is_neu=bct.is_neu, ef_is_dir=bfe.is_dir, ef_is_neu=bfe.is_neu,
             bc_values=ev(m.combine_boundary_operators_mechanical_stress([sd]), nd * nf),
             body_force=ev(m.body_force([sd]), nd * nc), angular_source=ev(m.source_angular_momentum([sd]), nr * nc),
             mass_source=ev(m.solid_mass_source([sd]), nc), fluid_source=ev(m.fluid_source([sd]), nc),
             energy_source=ev(m.energy_source([sd]), nc),
             flow_bc_values=np.where(bcf.is_dir, pbv, proj.T @ m.bc_values_darcy_flux(bg)),
             fourier_bc_values=np.where(bct.is_dir, tbv, proj.T @ m.bc_values_fourier_flux(bg)),
             ff_values=np.where(bff.is_dir, rho_b / fl.viscosity, proj.T @ m.bc_values_fluid_flux(bg)),
             ef_values=np.where(bfe.is_dir, fl.specific_heat_capacity * (tbv - t_ref) * rho_b / fl.viscosity,
                                proj.T @ m.bc_values_enthalpy_flux(bg)),
             compressibility=np.float64(fl.compressibility), density=np.float64(fl.density),
             viscosity=np.float64(fl.viscosity), reference_pressure=np.float64(p_ref),
             fluid_thermal_expansion=np.float64(fl.thermal_expansion),
             fluid_heat_capacity=np.float64(fl.specific_heat_capacity),
             fluid_conductivity=np.float64(fl.thermal_conductivity), reference_temperature=np.float64(t_ref),
             reference_porosity=np.float64(so.porosity), biot_coefficient=np.float64(so.biot_coefficient),
             bulk_modulus=np.float64(so.lame_lambda + 2 * so.shear_modulus / 3),
             solid_thermal_expansion=np.float64(so.thermal_expansion),
             solid_heat_capacity=np.float64(so.specific_heat_capacity),
             solid_conductivity=np.float64(so.thermal_conductivity), solid_density=np.float64(so.density))
    d["column_map"] = interleave([dofs(m.displacement_variable), dofs(m.rotation_stress_variable),
                                  dofs(m.total_pressure_variable), dofs(m.pressure_variable),
                                  dofs(m.temperature_variable)], nd, nr, nc)
    for s in range(2):
        m.time_manager.increase_time()
        m.time_manager.increase_time_index()
        m.before_nonlinear_loop()
        d[f"s{s}_previous"] = es.get_variable_values(time_step_index=0)
        norms = []
        for it in range(15):
            m.before_nonlinear_iteration()
            m.assemble_linear_system()
            A, b = m.linear_system
            norms.append(np.linalg.norm(b))
            if s == 0 and it == 0:
                put_csr(d, "J0", A)
                d["rhs0"] = b.copy()
                idx = es.assembled_equation_indices
                d["row_map"] = interleave([idx["momentum_balance_equation"], idx["angular_momentum_balance_equation"],
                                           idx["Solid_mass_equation_poromechanics"], idx["mass_balance_equation"],
                                           idx["energy_balance_equation"]], nd, nr, nc)
            if it == 1:
                d[f"s{s}_iterate"] = es.get_variable_values(iterate_index=0)
                d[f"s{s}_rhs"] = b.copy()
                put_csr(d, f"s{s}_J", A)
            if norms[-1] < 1e-13 * norms[0]:
                break
            m.after_nonlinear_iteration(m.solve_linear_system())
        assert len(norms) >= 3, norms
        d[f"s{s}_residual_norms"] = np.array(norms)
        d[f"s{s}_solution"] = es.get_variable_values(iterate_index=0)
        m.after_nonlinear_convergence()
        print(name, "step", s, "Newton residuals", ["%.2e" % v for v in norms])
    d["dt"] = np.float64(m.time_manager.dt)
    assert not np.any(d["energy_source"])
    # the flux changes direction inside the domain: the source drives flow towards both Dirichlet sides
    q = ev(m.darcy_flux([sd]), nf)
    inner = np.flatnonzero(np.diff(sd.cell_faces.tocsr().indptr) == 2)
    xn = sd.face_normals[0, inner]
    assert np.any(q[inner][xn > 0] > 0) and np.any(q[inner][xn > 0] < 0)
    assert bc.is_dir.any() and bc.is_neu.any() and not bc.is_rob.any()
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print(name, "nc", nc, "dofs", es.num_dofs(), f"{os.path.getsize(path) / 1e3:.0f} kB")


CASES = [
    ("tpsathm_cart2d", 2, 0.125, 401),
    ("tpsathm_cart3d", 3, 0.25, 402),
]


def main():
    os.makedirs(OUT, exist_ok=True)
    for name, nd, h, seed in CASES:
        case(name, nd, h, seed)


if __name__ == "__main__":
    main()
