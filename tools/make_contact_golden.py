"""Generate tests/golden/contact_model.npz: frictional contact on a fracture, the unmodified reference's
``pp.MomentumBalance`` (MPSA elasticity in the matrix with the fracture faces as internal Dirichlet boundary, interface
displacements, contact traction; force balance on the interface; the semismooth normal / tangential complementarity laws of
models/contact_mechanics.py:80-245 with Coulomb friction and shear dilation) -- the contact part of BASELINE config[4] in
miniature: a compressed and sheared fracture in the sliding regime.  Stored: grids, parameters, the geometric pieces of the
interface (scalar mortar projections, side signs, local fracture coordinates), the Jacobian / right-hand side at the second
Newton iterate, the residual history and the converged state.  ``Model2d`` is the 2-D counterpart (an 8 x 8 Cartesian unit
square cut by a vertical line fracture that does not reach the boundary; fixtures ``*_2d``).
   python tools/make_contact_golden.py"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_porepy  # noqa: E402
from make_golden import grid_arrays  # noqa: E402
from make_mdflow_golden import put_csr, rect  # noqa: E402

pp = load_porepy()
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


class Model(pp.MomentumBalance):
    def set_domain(self):
        self._domain = pp.Domain({"xmin": 0, "xmax": 1, "ymin": 0, "ymax": 1, "zmin": 0, "zmax": 1})

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": 0.25}

    def set_fractures(self):
        self._fractures = [pp.PlaneFracture(rect(0, 0.5, 0.25, 0.75))]

    def stiffness_tensor(self, sd):
        rng = np.random.default_rng(11 + sd.num_cells)
        return pp.FourthOrderTensor(1.5 * np.exp(0.2 * rng.standard_normal(sd.num_cells)),
                                    2.0 * np.exp(0.2 * rng.standard_normal(sd.num_cells)))

    def bc_type_mechanics(self, sd):
        s = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, s.west + s.east, "dir")
        bc.internal_to_dirichlet(sd)
        return bc

    scenario = "sliding"

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((3, bg.num_cells))
        if self.scenario == "sliding":
            v[0, s.east] = -0.01 * (1 + 0.3 * bg.cell_centers[2, s.east])     # compress across the fracture, unevenly
            v[1, s.east] = 0.02                                                # and shear it
            v[2, s.east] = 0.005 * bg.cell_centers[1, s.east]
        elif self.scenario == "sticking":                                      # strong compression, little shear
            v[0, s.east] = -0.02
            v[1, s.east] = 0.002 * bg.cell_centers[2, s.east]
        elif self.scenario == "open":                                          # pull the fracture open (+ some shear)
            v[0, s.east] = 0.01 * (1 + 0.5 * bg.cell_centers[1, s.east])
            v[2, s.east] = 0.004
        elif self.scenario == "mixed":                                         # a rotation-like load: part closes, part opens
            v[0, s.east] = 0.03 * (bg.cell_centers[2, s.east] - 0.5)
            v[1, s.east] = 0.01
        return v.ravel("F")


class Model2d(Model):
    """The 2-D counterpart of ``Model``: the unit square, 8 x 8 cells, the line fracture x = 0.5, 0.25 <= y <= 0.75; the
    east side is pushed and sheared as in 3-D, with the variation along y.  The grid is built by ``pp.meshing.cart_grid``
    directly (the fracture network of the default ``set_geometry`` needs shapely for a 2-D domain)."""

    def set_domain(self):
        self._domain = pp.Domain({"xmin": 0, "xmax": 1, "ymin": 0, "ymax": 1})

    def set_geometry(self):
        self.set_domain()
        self.mdg = pp.meshing.cart_grid([np.array([[0.5, 0.5], [0.25, 0.75]])], [8, 8], physdims=[1, 1])
        self.nd = self.mdg.dim_max()
        pp.set_local_coordinate_projections(self.mdg)
        self.set_well_network()

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((2, bg.num_cells))
        y = bg.cell_centers[1, s.east]
        if self.scenario == "sliding":
            v[0, s.east] = -0.01 * (1 + 0.3 * y)                               # compress across the fracture, unevenly
            v[1, s.east] = 0.02                                                # and shear it
        elif self.scenario == "mixed":                                         # a rotation-like load: the lower part
            v[0, s.east] = 0.03 * (y - 0.5)                                    # closes and slides, the upper part opens
            v[1, s.east] = 0.01
        return v.ravel("F")


def main(scenario="sliding", name="contact_model", base=Model):
    solid = pp.SolidConstants(lame_lambda=2.0, shear_modulus=1.5, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1)
    m = base({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 1.0, constant_dt=True),
               "material_constants": {"solid": solid}})
    m.scenario = scenario
    m.prepare_simulation()
    es, mdg = m.equation_system, m.mdg
    nd = m.nd
    mat, frac, intf = mdg.subdomains(dim=nd)[0], mdg.subdomains(dim=nd - 1)[0], mdg.interfaces()[0]
    assert list(es.equations) == ["momentum_balance_equation", "interface_force_balance_equation",
                                  "normal_fracture_deformation_equation", "tangential_fracture_deformation_equation"]

    def dofs(name):
        return es.dofs_of([v for v in es.variables if v.name == name])
    d = {f"matrix__{k}": v for k, v in grid_arrays(mat).items()}
    d.update({f"fracture__{k}": v for k, v in grid_arrays(frac).items()})
    data = mdg.subdomain_data(mat)
    bcm = data[pp.PARAMETERS]["mechanics"]["bc"] if "bc" in data[pp.PARAMETERS].get("mechanics", {}) else m.bc_type_mechanics(mat)
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(20):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 1:
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-11 * norms[0]:
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    bcm = mdg.subdomain_data(mat)[pp.PARAMETERS]["mechanics"]["bc"]
    bg = mdg.subdomain_to_boundary_grid(mat)
    proj3 = sps.kron(bg.projection(), sps.eye(nd)).tocsr()

    def scalar(op):
        v = es.evaluate(op)
        return float(np.atleast_1d(getattr(v, "val", v))[0])
    rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             column_map=np.concatenate([dofs("u"), dofs("contact_traction"), dofs("u_interface")]),
             C=mdg.subdomain_data(mat)[pp.PARAMETERS]["mechanics"]["fourth_order_tensor"].values,
             mech_is_dir=bcm.is_dir, mech_is_neu=bcm.is_neu, mech_is_rob=bcm.is_rob, mech_is_internal=bcm.is_internal,
             mech_bc_values=np.where(bcm.is_dir.ravel("F"), proj3.T @ m.bc_values_displacement(bg),
                                     proj3.T @ m.bc_values_stress(bg)),
             mortar_sign=sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), mortar_volumes=intf.cell_volumes,
             numerical_constant=np.float64(scalar(m.contact_mechanics_numerical_constant([frac]))),
             characteristic_traction=np.float64(scalar(m.characteristic_contact_traction([frac]))),
             friction_coefficient=np.float64(scalar(m.friction_coefficient([frac]))),
             dilation_angle=np.float64(m.solid.dilation_angle), reference_gap=np.float64(m.solid.fracture_gap),
             open_state_tolerance=np.float64(m.numerical.open_state_tolerance))
    put_csr(d, "local_coordinates", rot)
    for key in ("mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg", "secondary_to_mortar_int"):
        put_csr(d, key, getattr(intf, key)())
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    t = d["solution"][dofs("contact_traction")].reshape(-1, nd)
    print(name, "dofs", es.num_dofs(), "Newton residuals", ["%.2e" % v for v in norms])
    print("   contact traction (tangential, normal) per fracture cell:\\n", t, "\\n   |t_t| / (mu |t_n|):",
          np.linalg.norm(t[:, :nd - 1], axis=1) / (0.4 * np.abs(t[:, nd - 1])))


def permeability(model, subdomains):
    """Seeded heterogeneous, anisotropic permeability; 20 times larger in the fractures.  In 2-D the tensor is in-plane
    (k_zz = 1, no out-of-plane coupling)."""
    vals = []
    for sd in subdomains:
        rng = np.random.default_rng(5 + sd.num_cells)
        nc = sd.num_cells
        t = np.zeros((3, 3, nc))
        scale = 1.0 if sd.dim == model.nd else 20.0
        if model.nd == 3:
            t[0, 0], t[1, 1], t[2, 2] = scale * (1 + rng.random((3, nc)))
            o = 0.3 * scale * rng.random((3, nc))
            t[0, 1] = t[1, 0] = o[0]
            t[0, 2] = t[2, 0] = o[1]
            t[1, 2] = t[2, 1] = o[2]
        else:
            t[0, 0], t[1, 1] = scale * (1 + rng.random((2, nc)))
            t[0, 1] = t[1, 0] = 0.3 * scale * rng.random(nc)
            t[2, 2] = 1.0
        vals.append(t.reshape(9, nc).ravel("F"))
    return pp.wrap_as_dense_ad_array(np.hstack(vals) if vals else np.zeros(0), name="permeability")


def _geometry(base):
    """The geometry, stiffness and mechanical loads of ``base`` (``Model`` or ``Model2d``) as a mixin."""
    keys = ("set_domain", "grid_type", "meshing_arguments", "set_fractures", "stiffness_tensor", "bc_type_mechanics",
            "bc_values_displacement") + (("set_geometry",) if base is Model2d else ())
    return type("Geometry", (), {k: getattr(base, k) for k in keys})


def main_poromechanics(scenario="sliding", name="contact_poromech", base=Model):
    """``pp.Poromechanics`` on the same fractured domain: Biot poromechanics in the matrix, compressible flow in the
    fracture (aperture = residual aperture + normal jump), the interface Darcy law with that aperture, the fluid pressure
    in the interface force balance, frictional contact -- BASELINE configs[3] + [4] in one model."""
    class PoroModel(_geometry(base), pp.Poromechanics):
        permeability = permeability

        def bc_type_darcy_flux(self, sd):
            s = self.domain_boundary_sides(sd)
            return pp.BoundaryCondition(sd, s.south + s.north, "dir")

        def bc_type_fluid_flux(self, sd):
            s = self.domain_boundary_sides(sd)
            return pp.BoundaryCondition(sd, s.south + s.north, "dir")

        def bc_values_pressure(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros(bg.num_cells)
            v[s.south] = 0.02 * (1 + bg.cell_centers[0, s.south])
            return v
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0,
                              normal_permeability=2.0, residual_aperture=0.05, friction_coefficient=0.4,
                              fracture_gap=1e-4, dilation_angle=0.1)
    m = PoroModel({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 0.25, constant_dt=True),
                   "material_constants": {"fluid": fluid, "solid": solid}})
    m.scenario = scenario
    m.prepare_simulation()
    es, mdg = m.equation_system, m.mdg
    nd = m.nd
    mat, frac, intf = mdg.subdomains(dim=nd)[0], mdg.subdomains(dim=nd - 1)[0], mdg.interfaces()[0]

    def dofs(name, g=None):
        return es.dofs_of([v for v in es.variables if v.name == name and (g is None or v.domain is g)])
    d = {f"matrix__{k}": v for k, v in grid_arrays(mat).items()}
    d.update({f"fracture__{k}": v for k, v in grid_arrays(frac).items()})
    d["fracture__tip_faces"] = np.asarray(frac.tags["tip_faces"], bool)
    d["fracture__domain_boundary_faces"] = np.asarray(frac.tags["domain_boundary_faces"], bool)
    d["matrix__domain_boundary_faces"] = np.asarray(mat.tags["domain_boundary_faces"], bool)
    # the flux discretizations are those of the initial state (the reference re-discretizes only the upwinding)
    for key, sd in (("matrix", mat), ("fracture", frac)):
        prm = mdg.subdomain_data(sd)[pp.PARAMETERS]["flow"]
        d[f"{key}__K"] = prm["second_order_tensor"].values.copy()
        for f in ("is_dir", "is_neu", "is_rob", "is_internal"):
            d[f"{key}__flow_{f}"] = getattr(prm["bc"], f)
    rows, r0 = {}, 0
    layout = {"normal_fracture_deformation_equation": [(frac, 1)], "tangential_fracture_deformation_equation": [(frac, nd - 1)],
              "mass_balance_equation": [(mat, 1), (frac, 1)], "interface_darcy_flux_equation": [(intf, 1)],
              "momentum_balance_equation": [(mat, nd)], "interface_force_balance_equation": [(intf, nd)]}
    for eq in es.equations:
        for g, k in layout.get(eq, []):
            rows[(eq, id(g))] = np.arange(r0, r0 + k * g.num_cells)
            r0 += k * g.num_cells
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(25):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 0:            # the zero state: every tie rule of maximum / l2_norm / upwinding is active here
            d["initial_rhs"] = b.copy()
            put_csr(d, "initial_jacobian", A)
        if it == 1:
            d["iterate1"] = es.get_variable_values(iterate_index=0)
            d["iterate1_rhs"] = b.copy()
        if it == 2:
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-11 * norms[0]:
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    bg = mdg.subdomain_to_boundary_grid(mat)
    proj = bg.projection()
    proj3 = sps.kron(proj, sps.eye(nd)).tocsr()
    bcm = mdg.subdomain_data(mat)[pp.PARAMETERS]["mechanics"]["bc"]
    bcf = mdg.subdomain_data(mat)[pp.PARAMETERS]["flow"]["bc"]
    bff = m.bc_type_fluid_flux(mat)
    fl, so = m.fluid.reference_component, m.solid
    p_ref = m.reference_variable_values.pressure
    pb_ = proj.T @ m.bc_values_pressure(bg)

    def scalar(op):
        v = es.evaluate(op)
        return float(np.atleast_1d(getattr(v, "val", v))[0])
    kb = so.lame_lambda + 2 * so.shear_modulus / 3
    rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
    order_c = [dofs("pressure", mat), dofs("pressure", frac), dofs("u"), dofs("contact_traction"),
               dofs("interface_darcy_flux"), dofs("u_interface")]
    order_r = [("mass_balance_equation", mat), ("mass_balance_equation", frac), ("momentum_balance_equation", mat),
               ("interface_darcy_flux_equation", intf), ("interface_force_balance_equation", intf),
               ("normal_fracture_deformation_equation", frac), ("tangential_fracture_deformation_equation", frac)]
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             column_map=np.concatenate(order_c), row_map=np.concatenate([rows[(eq, id(g))] for eq, g in order_r]),
             dt=np.float64(m.time_manager.dt),
             C=mdg.subdomain_data(mat)[pp.PARAMETERS]["mechanics"]["fourth_order_tensor"].values,
             biot_coefficient=np.float64(so.biot_coefficient), reference_porosity=np.float64(so.porosity),
             n_inv=np.float64((so.biot_coefficient - so.porosity) * (1 - so.biot_coefficient) / kb),
             compressibility=np.float64(fl.compressibility), density=np.float64(fl.density),
             viscosity=np.float64(fl.viscosity), reference_pressure=np.float64(p_ref),
             residual_aperture=np.float64(so.residual_aperture),
             normal_permeability=np.broadcast_to(np.asarray(getattr(es.evaluate(m.normal_permeability([intf])), "val",
                                                                    es.evaluate(m.normal_permeability([intf]))), float),
                                                 (intf.num_cells,)).copy(),
             mech_is_dir=bcm.is_dir, mech_is_neu=bcm.is_neu, mech_is_rob=bcm.is_rob, mech_is_internal=bcm.is_internal,
             mech_bc_values=np.where(bcm.is_dir.ravel("F"), proj3.T @ m.bc_values_displacement(bg),
                                     proj3.T @ m.bc_values_stress(bg)),
             flow_bc_values=np.where(bcf.is_dir, pb_, proj.T @ m.bc_values_darcy_flux(bg)),
             ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             ff_values=np.where(bff.is_dir, fl.density * np.exp(fl.compressibility * (pb_ - p_ref)) / fl.viscosity,
                                proj.T @ m.bc_values_fluid_flux(bg)),
             mortar_sign=sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), mortar_volumes=intf.cell_volumes,
             numerical_constant=np.float64(scalar(m.contact_mechanics_numerical_constant([frac]))),
             characteristic_traction=np.float64(scalar(m.characteristic_contact_traction([frac]))),
             friction_coefficient=np.float64(scalar(m.friction_coefficient([frac]))),
             dilation_angle=np.float64(so.dilation_angle), reference_gap=np.float64(so.fracture_gap),
             open_state_tolerance=np.float64(m.numerical.open_state_tolerance))
    put_csr(d, "local_coordinates", rot)
    for key in ("mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg", "secondary_to_mortar_int",
                "mortar_to_primary_int", "primary_to_mortar_avg", "mortar_to_secondary_int", "secondary_to_mortar_avg"):
        put_csr(d, key, getattr(intf, key)())
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    t = d["solution"][dofs("contact_traction")].reshape(-1, nd)
    print(name, "dofs", es.num_dofs(), "Newton residuals", ["%.2e" % v for v in norms])
    print("   contact traction:", np.array2string(t, precision=4).replace("\n", ";"))


def main_thm(scenario="sliding", name="contact_thm", base=Model):
    """``pp.Thermoporomechanics`` on the fractured domain: BASELINE config[4] (thermo-poromechanics + frictional contact, full
    Newton loop) on one fracture."""
    class ThmModel(_geometry(base), pp.Thermoporomechanics):
        permeability = permeability

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
            v[s.south] = 0.3 + 0.1 * bg.cell_centers[2 if self.nd == 3 else 0, s.south]      # varies along z, x in 2-D
            return v
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7, thermal_expansion=0.03,
                              specific_heat_capacity=2.0, thermal_conductivity=0.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0,
                              normal_permeability=2.0, residual_aperture=0.05, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1, thermal_expansion=0.02, specific_heat_capacity=1.5,
                              thermal_conductivity=1.1, density=2.5)
    m = ThmModel({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 0.25, constant_dt=True),
                  "material_constants": {"fluid": fluid, "solid": solid}})
    m.scenario = scenario
    m.prepare_simulation()
    es, mdg = m.equation_system, m.mdg
    nd = m.nd
    mat, frac, intf = mdg.subdomains(dim=nd)[0], mdg.subdomains(dim=nd - 1)[0], mdg.interfaces()[0]

    def dofs(name, g=None):
        return es.dofs_of([v for v in es.variables if v.name == name and (g is None or v.domain is g)])
    d = {f"matrix__{k}": v for k, v in grid_arrays(mat).items()}
    d.update({f"fracture__{k}": v for k, v in grid_arrays(frac).items()})
    d["fracture__tip_faces"] = np.asarray(frac.tags["tip_faces"], bool)
    d["fracture__domain_boundary_faces"] = np.asarray(frac.tags["domain_boundary_faces"], bool)
    d["matrix__domain_boundary_faces"] = np.asarray(mat.tags["domain_boundary_faces"], bool)
    for key, sd in (("matrix", mat), ("fracture", frac)):
        for short, kw in (("flow", "flow"), ("fourier", "fourier_discretization")):
            prm = mdg.subdomain_data(sd)[pp.PARAMETERS][kw]
            d[f"{key}__{short}_K"] = prm["second_order_tensor"].values.copy()       # at the initial state
            for f in ("is_dir", "is_neu", "is_rob", "is_internal"):
                d[f"{key}__{short}_{f}"] = getattr(prm["bc"], f)
    svm = mdg.subdomain_data(mat)[pp.PARAMETERS]["mechanics"]["scalar_vector_mappings"]
    d["alpha_flow"], d["alpha_thermal"] = svm["flow"].values, svm[m.enthalpy_keyword].values
    layout = {"normal_fracture_deformation_equation": [(frac, 1)], "tangential_fracture_deformation_equation": [(frac, nd - 1)],
              "momentum_balance_equation": [(mat, nd)], "interface_force_balance_equation": [(intf, nd)],
              "mass_balance_equation": [(mat, 1), (frac, 1)], "interface_darcy_flux_equation": [(intf, 1)],
              "energy_balance_equation": [(mat, 1), (frac, 1)], "interface_fourier_flux_equation": [(intf, 1)],
              "interface_enthalpy_flux_equation": [(intf, 1)]}
    rows, r0 = {}, 0
    for eq in es.equations:
        for g, k in layout.get(eq, []):
            rows[(eq, id(g))] = np.arange(r0, r0 + k * g.num_cells)
            r0 += k * g.num_cells
    m.time_manager.increase_time()
    m.time_manager.increase_time_index()
    m.before_nonlinear_loop()
    x_prev = es.get_variable_values(time_step_index=0)
    norms = []
    for it in range(25):
        m.before_nonlinear_iteration()
        m.assemble_linear_system()
        A, b = m.linear_system
        norms.append(np.linalg.norm(b))
        if it == 0:
            d["initial_rhs"] = b.copy()
            put_csr(d, "initial_jacobian", A)
        if it == 3:                       # aperture off its residual value here: the re-discretized fracture fluxes matter
            d["iterate"] = es.get_variable_values(iterate_index=0)
            d["iterate_rhs"] = b.copy()
            put_csr(d, "iterate_jacobian", A)
        if norms[-1] < 1e-11 * norms[0]:
            break
        m.after_nonlinear_iteration(m.solve_linear_system())
    bg = mdg.subdomain_to_boundary_grid(mat)
    proj = bg.projection()
    proj3 = sps.kron(proj, sps.eye(nd)).tocsr()
    prm = mdg.subdomain_data(mat)[pp.PARAMETERS]
    bcm, bcf, bct = prm["mechanics"]["bc"], prm["flow"]["bc"], prm["fourier_discretization"]["bc"]
    bff, bfe = m.bc_type_fluid_flux(mat), m.bc_type_enthalpy_flux(mat)
    fl, so = m.fluid.reference_component, m.solid
    p_ref, t_ref = m.reference_variable_values.pressure, m.reference_variable_values.temperature
    pb_, tb = proj.T @ m.bc_values_pressure(bg), proj.T @ m.bc_values_temperature(bg)
    rho_b = fl.density * np.exp(fl.compressibility * (pb_ - p_ref) - fl.thermal_expansion * (tb - t_ref))

    def scalar(op):
        v = es.evaluate(op)
        return float(np.atleast_1d(getattr(v, "val", v))[0])

    def field(op, n):
        v = es.evaluate(op)
        v = getattr(v, "val", v)
        return np.full(n, float(v)) if np.ndim(v) == 0 else np.asarray(v, float)
    kb = so.lame_lambda + 2 * so.shear_modulus / 3
    rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
    order_c = [dofs("pressure", mat), dofs("pressure", frac), dofs("temperature", mat), dofs("temperature", frac), dofs("u"),
               dofs("contact_traction"), dofs("interface_darcy_flux"), dofs("interface_fourier_flux"),
               dofs("interface_enthalpy_flux"), dofs("u_interface")]
    order_r = [("mass_balance_equation", mat), ("mass_balance_equation", frac), ("energy_balance_equation", mat),
               ("energy_balance_equation", frac), ("momentum_balance_equation", mat), ("interface_darcy_flux_equation", intf),
               ("interface_fourier_flux_equation", intf), ("interface_enthalpy_flux_equation", intf),
               ("interface_force_balance_equation", intf), ("normal_fracture_deformation_equation", frac),
               ("tangential_fracture_deformation_equation", frac)]
    d.update(previous=x_prev, solution=es.get_variable_values(iterate_index=0), residual_norms=np.array(norms),
             column_map=np.concatenate(order_c), row_map=np.concatenate([rows[(eq, id(g))] for eq, g in order_r]),
             dt=np.float64(m.time_manager.dt),
             C=prm["mechanics"]["fourth_order_tensor"].values,
             biot_coefficient=np.float64(so.biot_coefficient), reference_porosity=np.float64(so.porosity),
             n_inv=np.float64((so.biot_coefficient - so.porosity) * (1 - so.biot_coefficient) / kb),
             compressibility=np.float64(fl.compressibility), density=np.float64(fl.density), viscosity=np.float64(fl.viscosity),
             fluid_thermal_expansion=np.float64(fl.thermal_expansion), fluid_heat_capacity=np.float64(fl.specific_heat_capacity),
             fluid_conductivity=np.float64(fl.thermal_conductivity), solid_thermal_expansion=np.float64(so.thermal_expansion),
             solid_heat_capacity=np.float64(so.specific_heat_capacity), solid_conductivity=np.float64(so.thermal_conductivity),
             solid_density=np.float64(so.density), reference_pressure=np.float64(p_ref), reference_temperature=np.float64(t_ref),
             residual_aperture=np.float64(so.residual_aperture),
             normal_permeability=field(m.normal_permeability([intf]), intf.num_cells),
             normal_thermal_conductivity=field(m.normal_thermal_conductivity([intf]), intf.num_cells),
             mech_is_dir=bcm.is_dir, mech_is_neu=bcm.is_neu, mech_is_rob=bcm.is_rob, mech_is_internal=bcm.is_internal,
             mech_bc_values=np.where(bcm.is_dir.ravel("F"), proj3.T @ m.bc_values_displacement(bg),
                                     proj3.T @ m.bc_values_stress(bg)),
             flow_bc_values=np.where(bcf.is_dir, pb_, proj.T @ m.bc_values_darcy_flux(bg)),
             fourier_bc_values=np.where(bct.is_dir, tb, proj.T @ m.bc_values_fourier_flux(bg)),
             ff_is_dir=bff.is_dir, ff_is_neu=bff.is_neu,
             ff_values=np.where(bff.is_dir, rho_b / fl.viscosity, proj.T @ m.bc_values_fluid_flux(bg)),
             ef_is_dir=bfe.is_dir, ef_is_neu=bfe.is_neu,
             ef_values=np.where(bfe.is_dir, fl.specific_heat_capacity * (tb - t_ref) * rho_b / fl.viscosity,
                                proj.T @ m.bc_values_enthalpy_flux(bg)),
             mortar_sign=sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), mortar_volumes=intf.cell_volumes,
             numerical_constant=np.float64(scalar(m.contact_mechanics_numerical_constant([frac]))),
             characteristic_traction=np.float64(scalar(m.characteristic_contact_traction([frac]))),
             friction_coefficient=np.float64(scalar(m.friction_coefficient([frac]))),
             dilation_angle=np.float64(so.dilation_angle), reference_gap=np.float64(so.fracture_gap),
             open_state_tolerance=np.float64(m.numerical.open_state_tolerance))
    put_csr(d, "local_coordinates", rot)
    for key in ("mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg", "secondary_to_mortar_int",
                "mortar_to_primary_int", "primary_to_mortar_avg", "mortar_to_secondary_int", "secondary_to_mortar_avg"):
        put_csr(d, key, getattr(intf, key)())
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(name, "dofs", es.num_dofs(), "Newton residuals", ["%.2e" % v for v in norms])


if __name__ == "__main__":
    main_thm("sliding", "contact_thm")
    main_thm("mixed", "contact_thm_mixed")
    main_poromechanics("sliding", "contact_poromech")
    main_poromechanics("mixed", "contact_poromech_mixed")
    main("sliding", "contact_model")
    main("sticking", "contact_sticking")
    main("open", "contact_open")
    main("mixed", "contact_mixed")
    main_thm("sliding", "contact_thm_2d", Model2d)
    main_poromechanics("sliding", "contact_poromech_2d", Model2d)
    main("sliding", "contact_2d", Model2d)
    main("mixed", "contact_2d_mixed", Model2d)
