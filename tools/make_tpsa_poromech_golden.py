"""Generate tests/golden/tpsaporo_*.npz from the unmodified reference's TPSA poromechanics model
(``pp.Poromechanics`` with ``TpsaPoromechanicsMixin``: displacement, rotation stress, total pressure and fluid pressure),
run in the build container where the reference is importable.

Every model has heterogeneous mu and lambda, a Biot coefficient below one, a compressible fluid with a non-zero reference
pressure, a flow source in the middle of the domain between two Dirichlet pressure sides (so the upwind direction
changes inside the domain), and mechanical Dirichlet (west), roller (south) and Neumann (elsewhere) faces.  Each fixture
holds
  * the grid (``make_golden.grid_arrays``), mu, lambda, the permeability and both boundary conditions;
  * the inputs of ``porepy_b200.TpsaPoromechanics``: the evaluated mechanical boundary operator, body force, angular and
    solid-mass sources, the Darcy boundary values, the fluid-flux boundary weights, the fluid source and the constants;
  * ``J0`` / ``rhs0``: the model's ``equation_system.assemble()`` at the zero state (the first linearization of step 0);
  * for time steps s = 0, 1: ``s{s}_previous``, ``s{s}_iterate`` (the second Newton iterate) with ``s{s}_J`` / ``s{s}_rhs``
    there, ``s{s}_residual_norms`` and the converged ``s{s}_solution``;
  * ``column_map`` / ``row_map``: the model dof / row of each unknown / equation in the cell-interleaved order
    [u_c, r_c, p_t_c, p_c], from ``dofs_of`` and ``assembled_equation_indices``.

    python tools/make_tpsa_poromech_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import OUT, grid_arrays, pp  # noqa: E402
from make_mdflow_golden import put_csr  # noqa: E402


class Setup:
    def set_domain(self):
        box = {"xmin": 0, "xmax": 1.25, "ymin": 0, "ymax": 1}
        if self.params["tpsa_nd"] == 3:
            box.update(zmin=0, zmax=1)
        self._domain = pp.Domain(box)

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": self.params["cell_size"]}

    def stiffness_tensor(self, sd):
        rng = np.random.default_rng(self.params["seed"])
        mu = 1.5 * np.exp(0.5 * rng.standard_normal(sd.num_cells))
        mu[sd.cell_centers[0] < 0.5] *= 10.0
        lmbda = 2.0 * np.exp(0.5 * rng.standard_normal(sd.num_cells))
        return pp.FourthOrderTensor(mu, lmbda)

    def bc_type_mechanics(self, sd):
        """Dirichlet west, a roller south (Dirichlet in y), Neumann elsewhere."""
        s = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, s.west, "dir")
        south = s.south & ~s.west
        bc.is_dir[1, south] = True
        bc.is_neu[1, south] = False
        return bc

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[0, s.west] = 0.01 * bg.cell_centers[1, s.west]
        v[self.nd - 1, s.west] = -0.005
        return v.ravel("F")

    def bc_values_stress(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[1, s.north] = -1e-2 * bg.cell_volumes[s.north]
        v[0, s.east] = 5e-3 * bg.cell_volumes[s.east]
        return v.ravel("F")

    def bc_type_darcy_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_type_fluid_flux(self, sd):
        s = self.domain_boundary_sides(sd)
        return pp.BoundaryCondition(sd, s.west + s.east, "dir")

    def bc_values_pressure(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.full(bg.num_cells, self.reference_variable_values.pressure)
        v[s.west] = 0.6 + 0.2 * bg.cell_centers[1, s.west]
        v[s.east] = 0.2
        return v

    def fluid_source(self, subdomains):
        vals = []
        for sd in subdomains:
            x = sd.cell_centers
            vals.append(30.0 * np.exp(-20.0 * ((x[0] - 0.7) ** 2 + (x[1] - 0.5) ** 2)))
        src = pp.wrap_as_dense_ad_array(np.hstack(vals), name="fluid_source_density")
        return super().fluid_source(subdomains) + self.volume_integral(src, subdomains, dim=1)


class Model(Setup, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Poromechanics):
    pass


def interleave(blocks, nd, nr, nc):
    u, r, pt, p = blocks
    out = np.empty((nc, nd + nr + 2), np.int64)
    out[:, :nd] = np.asarray(u).reshape(nc, nd)
    out[:, nd:nd + nr] = np.asarray(r).reshape(nc, nr)
    out[:, nd + nr] = pt
    out[:, nd + nr + 1] = p
    return out.reshape(-1)


def case(name, nd, cell_size, seed):
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.7, lame_lambda=2.0, shear_modulus=1.5,
                              permeability=0.8)
    m = Model({"times_to_export": [], "tpsa_nd": nd, "cell_size": cell_size, "seed": seed,
               "time_manager": pp.TimeManager([0, 0.5], 0.25, constant_dt=True),
               "material_constants": {"fluid": fluid, "solid": solid},
               "reference_variable_values": pp.ReferenceVariableValues(pressure=0.3)})
    m.prepare_simulation()
    es = m.equation_system
    sd = m.mdg.subdomains()[0]
    nc, nf = sd.num_cells, sd.num_faces
    nr = m.rotation_dimension()
    assert np.all(es.get_variable_values(iterate_index=0) == 0)
    data = m.mdg.subdomain_data(sd)
    mk, fk = m.stress_keyword, m.darcy_keyword
    bc, C = data[pp.PARAMETERS][mk]["bc"], data[pp.PARAMETERS][mk]["fourth_order_tensor"]
    bcf, bff = data[pp.PARAMETERS][fk]["bc"], m.bc_type_fluid_flux(sd)
    bg = m.mdg.subdomain_to_boundary_grid(sd)
    proj = bg.projection()
    fl = m.fluid.reference_component
    p_ref = m.reference_variable_values.pressure
    pbv = proj.T @ m.bc_values_pressure(bg)

    def ev(op, n):
        v = es.evaluate(op)
        return np.broadcast_to(np.asarray(getattr(v, "val", v), float), (n,)).copy()

    def dofs(var):
        return es.dofs_of([v for v in es.variables if v.name == var])
    d = grid_arrays(sd)
    d.update(kind=np.array("tpsa_poromech"), mu=C.mu, lmbda=C.lmbda,
             K=data[pp.PARAMETERS][fk]["second_order_tensor"].values,
             bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=np.asarray(bc.is_internal, bool), bc_robin_weight=np.asarray(bc.robin_weight, float),
             bc_basis=np.asarray(bc.basis, float),
             flow_is_dir=bcf.is_dir, flow_is_neu=bcf.is_neu, ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             bc_values=ev(m.combine_boundary_operators_mechanical_stress([sd]), nd * nf),
             body_force=ev(m.body_force([sd]), nd * nc), angular_source=ev(m.source_angular_momentum([sd]), nr * nc),
             mass_source=ev(m.solid_mass_source([sd]), nc), fluid_source=ev(m.fluid_source([sd]), nc),
             flow_bc_values=np.where(bcf.is_dir, pbv, proj.T @ m.bc_values_darcy_flux(bg)),
             ff_values=np.where(bff.is_dir, fl.density * np.exp(fl.compressibility * (pbv - p_ref)) / fl.viscosity,
                                proj.T @ m.bc_values_fluid_flux(bg)),
             compressibility=np.float64(fl.compressibility), density=np.float64(fl.density),
             viscosity=np.float64(fl.viscosity), reference_pressure=np.float64(p_ref),
             reference_porosity=np.float64(m.solid.porosity), biot_coefficient=np.float64(m.solid.biot_coefficient),
             bulk_modulus=np.float64(m.solid.lame_lambda + 2 * m.solid.shear_modulus / 3))
    d["column_map"] = interleave([dofs(m.displacement_variable), dofs(m.rotation_stress_variable),
                                  dofs(m.total_pressure_variable), dofs(m.pressure_variable)], nd, nr, nc)
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
                                           idx["Solid_mass_equation_poromechanics"], idx["mass_balance_equation"]], nd, nr, nc)
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
    ("tpsaporo_cart2d", 2, 0.125, 301),
    ("tpsaporo_cart3d", 3, 0.25, 302),
]


def main():
    os.makedirs(OUT, exist_ok=True)
    for name, nd, h, seed in CASES:
        case(name, nd, h, seed)


if __name__ == "__main__":
    main()
