"""From a prepared PorePy model to the device problems of this package: the glue a PorePy user needs to hand a live
``pp.SinglePhaseFlow`` / ``pp.MassAndEnergyBalance`` (on a fracture network) or ``pp.Poromechanics`` /
``pp.Thermoporomechanics`` (one 2-D or 3-D subdomain, or such a matrix cut by non-intersecting fractures of one dimension
less) over to ``porepy_b200`` -- grids, parameter dictionaries and mortar projections
of ``model.mdg`` as they are; boundary data, coefficients and constants evaluated from the model's own methods
(``bc_values_*``, ``bc_type_*``, ``normal_permeability``, ``aperture``, ``specific_volume``, ``porosity``, the fluid and
solid constants).  Reached through ``porepy_plugin.plugin(pp)``: ``b200.compressible_flow_from_model(model)`` etc.

The model's data dictionaries are not modified: every problem gets its own dictionaries (the parameter entries are shared,
the discretization matrices and the upwind parameters are the problem's own).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps

from .layout import BlockLayout
from .params import DISCRETIZATION_MATRICES, PARAMETERS


def _dofs(model, name, grid):
    """Dofs of the variable ``name`` on ``grid`` in the model's ``EquationSystem``."""
    es = model.equation_system
    return es.dofs_of([v for v in es.variables if v.name == name and v.domain is grid])


def _column_map(model, layout, grids):
    """Dof of the model of every unknown of ``layout``: block ``name`` is the model's ``{name}_variable``, the part on
    domain d lives on ``grids[d]``."""
    return np.concatenate([_dofs(model, getattr(model, f"{name}_variable"), grids[d]) for name, d, _, _ in
                           layout.items()])


def _row_map(model, layout):
    """Row of the model of every equation of ``layout``: the model numbers its equations in the order of
    ``equation_system.equations``, the parts of one equation in the layout's order."""
    rows, r0 = {}, 0
    for eq in model.equation_system.equations:
        for name, d, n, w in layout.items():
            if name == eq:
                rows[(name, d)] = np.arange(r0, r0 + n * w)
                r0 += n * w
    return np.concatenate([rows[(name, d)] for name, d, _, _ in layout.items()])


def _evaluated(model, op, n):
    v = model.equation_system.evaluate(op)
    v = getattr(v, "val", v)
    return np.full(n, float(v)) if np.ndim(v) == 0 else np.asarray(v, float)


def _own_data(data: dict, keywords) -> dict:
    return {PARAMETERS: {kw: dict(data[PARAMETERS][kw]) for kw in keywords if kw in data.get(PARAMETERS, {})},
            DISCRETIZATION_MATRICES: {}}


def _face_values(model, sd, bc, dirichlet, neumann):
    """Boundary operator of a flux law on ``sd``: ``dirichlet(bg)`` on the Dirichlet faces of ``bc``, ``neumann(bg)``
    elsewhere (``_combine_boundary_operators`` of the models), as a face array."""
    bg = model.mdg.subdomain_to_boundary_grid(sd)
    if bg is None or bg.num_cells == 0:
        return np.zeros(sd.num_faces)
    proj = bg.projection()
    return np.where(bc.is_dir, proj.T @ dirichlet(bg), proj.T @ neumann(bg))


def _fluid(model, thermal: bool) -> dict:
    fl = model.fluid.reference_component
    out = dict(compressibility=fl.compressibility, density=fl.density, viscosity=fl.viscosity,
               reference_pressure=model.reference_variable_values.pressure)
    if thermal:
        out.update(thermal_expansion=fl.thermal_expansion, heat_capacity=fl.specific_heat_capacity,
                   conductivity=fl.thermal_conductivity, reference_temperature=model.reference_variable_values.temperature)
    return out


def _boundary_weights(model, sd, fluid: dict, thermal: bool):
    """(rho / mu, c_f (T - T0) rho / mu) of the boundary pressure / temperature, as functions of a boundary grid."""
    def rho(bg):
        e = fluid["compressibility"] * (model.bc_values_pressure(bg) - fluid["reference_pressure"])
        if thermal:
            e = e - fluid["thermal_expansion"] * (model.bc_values_temperature(bg) - fluid["reference_temperature"])
        return fluid["density"] * np.exp(e)

    def w(bg):
        return rho(bg) / fluid["viscosity"]

    def we(bg):
        return fluid["heat_capacity"] * (model.bc_values_temperature(bg) - fluid["reference_temperature"]) * w(bg)
    return w, we


def _interfaces(model, thermal: bool):
    from .mdflow import MdInterface
    mdg = model.mdg
    index = {id(sd): i for i, sd in enumerate(mdg.subdomains())}
    out, kappa_t = [], []
    for it in mdg.interfaces():
        if getattr(it, "codim", 1) != 1:
            continue
        h, l = mdg.interface_to_subdomain_pair(it)
        out.append(MdInterface(index[id(h)], index[id(l)], it.mortar_to_primary_int(), it.primary_to_mortar_avg(),
                               it.mortar_to_secondary_int(), it.secondary_to_mortar_avg(),
                               _evaluated(model, model.normal_permeability([it]), it.num_cells),
                               np.asarray(it.cell_volumes, float) * _evaluated(model, model.specific_volume([it]), it.num_cells),
                               _evaluated(model, model.aperture([l]), l.num_cells)))
        if thermal:
            kappa_t.append(_evaluated(model, model.normal_thermal_conductivity([it]), it.num_cells))
    return out, kappa_t


def compressible_flow_from_model(model):
    """``pp.SinglePhaseFlow`` (compressible fluid) on ``model.mdg`` -> ``CompressibleMixedDimensionalFlow``; unknowns and
    equations in the model's own order."""
    from .mdflow import MdSubdomain
    from .mdflow_nl import CompressibleMixedDimensionalFlow
    mdg, kw = model.mdg, model.darcy_keyword
    fluid = _fluid(model, False)
    subs, storage, bcs, weights = [], [], [], []
    for sd in mdg.subdomains():
        data = _own_data(mdg.subdomain_data(sd), [kw])
        n = sd.num_cells
        storage.append(np.asarray(sd.cell_volumes, float) * _evaluated(model, model.specific_volume([sd]), n)
                       * _evaluated(model, model.porosity([sd]), n))
        if sd.num_faces == 0:
            subs.append(MdSubdomain(sd, data))
            bcs.append(None)
            weights.append(None)
            continue
        w, _ = _boundary_weights(model, sd, fluid, False)
        bc_ff = model.bc_type_fluid_flux(sd)
        subs.append(MdSubdomain(sd, data, _face_values(model, sd, data[PARAMETERS][kw]["bc"], model.bc_values_pressure,
                                                       model.bc_values_darcy_flux)))
        bcs.append(bc_ff)
        weights.append(_face_values(model, sd, bc_ff, w, model.bc_values_fluid_flux))
    intfs, _ = _interfaces(model, False)
    prob = CompressibleMixedDimensionalFlow(subs, intfs, fluid, storage, bcs, weights, keyword=kw)
    prob.mobility_keyword = "b200_mobility"
    return prob


def mass_energy_from_model(model):
    """``pp.MassAndEnergyBalance`` on ``model.mdg`` -> (``MixedDimensionalMassEnergy``, column_map, row_map): unknown k
    of the problem is dof ``column_map[k]`` of the model's ``EquationSystem``, equation k its row ``row_map[k]``."""
    from .mdflow import MdSubdomain
    from .mdthermal import MixedDimensionalMassEnergy
    mdg = model.mdg
    fk, tk = model.darcy_keyword, model.fourier_keyword
    fluid = _fluid(model, True)
    solid = dict(density=model.solid.density, heat_capacity=model.solid.specific_heat_capacity)
    sds = list(mdg.subdomains())
    subs, volume, porosity, bcv, bct = [], [], [], [], []
    for sd in sds:
        data = _own_data(mdg.subdomain_data(sd), [fk, tk])
        n = sd.num_cells
        volume.append(np.asarray(sd.cell_volumes, float) * _evaluated(model, model.specific_volume([sd]), n))
        porosity.append(_evaluated(model, model.porosity([sd]), n))
        subs.append(MdSubdomain(sd, data))
        if sd.num_faces == 0:
            bcv.append(None)
            bct.append(None)
            continue
        w, we = _boundary_weights(model, sd, fluid, True)
        ff, ef = model.bc_type_fluid_flux(sd), model.bc_type_enthalpy_flux(sd)
        prm = data[PARAMETERS]
        bcv.append(dict(flow=_face_values(model, sd, prm[fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
                        fourier=_face_values(model, sd, prm[tk]["bc"], model.bc_values_temperature, model.bc_values_fourier_flux),
                        fluid_flux=_face_values(model, sd, ff, w, model.bc_values_fluid_flux),
                        enthalpy_flux=_face_values(model, sd, ef, we, model.bc_values_enthalpy_flux)))
        bct.append(dict(fluid_flux=ff, enthalpy_flux=ef))
    intfs, kappa_t = _interfaces(model, True)
    prob = MixedDimensionalMassEnergy(subs, intfs, fluid, solid, volume, porosity, bcv, bct, kappa_t, flow_keyword=fk,
                                      fourier_keyword=tk)
    prob.mobility_keyword, prob.enthalpy_upwind_keyword = "b200_mobility", "b200_enthalpy_upwind"
    its = [it for it in mdg.interfaces() if getattr(it, "codim", 1) == 1]
    grids = {**{("subdomain", i): sd for i, sd in enumerate(sds)}, **{("interface", j): it for j, it in enumerate(its)}}
    return prob, _column_map(model, prob.unknown_layout, grids), _row_map(model, prob.equation_layout)


def _mechanics_boundary(model, sd, data, mk):
    """Displacement on the Dirichlet faces of the vectorial ``bc``, traction elsewhere: nd nf, face-major."""
    bg = model.mdg.subdomain_to_boundary_grid(sd)
    proj = sps.kron(bg.projection(), sps.identity(int(sd.dim))).tocsr()
    bc = data[PARAMETERS][mk]["bc"]
    return np.where(np.asarray(bc.is_dir).ravel("F"), proj.T @ model.bc_values_displacement(bg),
                    proj.T @ model.bc_values_stress(bg))


def _single_matrix(model):
    """The one subdomain of a model without fractures; it must be 2-D or 3-D."""
    sds = list(model.mdg.subdomains())
    if len(sds) != 1:
        raise NotImplementedError(f"one subdomain without fractures is expected, the model has {len(sds)} (of dimensions "
                                  f"{sorted({int(sd.dim) for sd in sds}, reverse=True)})")
    if sds[0].dim not in (2, 3):
        raise NotImplementedError(f"the mechanics equations need a 2-D or 3-D subdomain, the model's is {sds[0].dim}-D")
    return sds[0]


def _matrix_and_fractures(model):
    """(matrix, fractures, the grids of the layout domains ``("matrix",)``, ``("fracture", j)``, ``("interface", j)``) of
    a model with one nd-D matrix (nd = 2 or 3) and fractures of dimension nd - 1 that do not intersect; anything else --
    intersection lines or points, a 1-D matrix, several matrices -- raises ``NotImplementedError``."""
    mdg = model.mdg
    nd = int(mdg.dim_max())
    if nd not in (2, 3):
        raise NotImplementedError(f"a {nd}-D matrix: the contact mechanics equations need a 2-D or 3-D matrix with "
                                  f"fractures of one dimension less")
    mats = list(mdg.subdomains(dim=nd))
    if len(mats) != 1:
        raise NotImplementedError(f"one {nd}-D matrix subdomain is expected, the model has {len(mats)}")
    low = sorted({int(sd.dim) for sd in mdg.subdomains() if sd.dim < nd - 1}, reverse=True)
    if low:
        raise NotImplementedError(f"{low[0]}-D subdomains (fracture intersections) in a {nd}-D matrix: only {nd - 1}-D "
                                  f"fractures without intersections are supported")
    fracs = list(mdg.subdomains(dim=nd - 1))
    grids = {("matrix",): mats[0]}
    for j, f in enumerate(fracs):
        grids[("fracture", j)] = f
        grids[("interface", j)] = [it for it in mdg.interfaces() if mdg.interface_to_subdomain_pair(it)[1] is f][0]
    return mats[0], fracs, grids


def _n_inv(model):
    so = model.solid
    bulk = so.lame_lambda + 2.0 * so.shear_modulus / 3.0          # ``bulk_modulus`` of the solid constants
    return (so.biot_coefficient - so.porosity) * (1.0 - so.biot_coefficient) / bulk


def poromechanics_from_model(model):
    """``pp.Poromechanics`` on one 2-D or 3-D subdomain without fractures -> ``Poromechanics`` (unknowns [p | u], the
    model's own order)."""
    from .poromech import Poromechanics
    sd = _single_matrix(model)
    fk, mk = model.darcy_keyword, model.stress_keyword
    data = _own_data(model.mdg.subdomain_data(sd), [fk, mk])
    fluid = _fluid(model, False)
    w, _ = _boundary_weights(model, sd, fluid, False)
    bc_ff = model.bc_type_fluid_flux(sd)
    prob = Poromechanics(sd, data, fluid, dict(reference_porosity=model.solid.porosity, n_inv=_n_inv(model)),
                         _face_values(model, sd, data[PARAMETERS][fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
                         _mechanics_boundary(model, sd, data, mk), bc_ff,
                         _face_values(model, sd, bc_ff, w, model.bc_values_fluid_flux), flow_keyword=fk, mechanics_keyword=mk)
    prob.mobility_keyword = "b200_mobility"
    return prob


def thermoporomechanics_from_model(model):
    """``pp.Thermoporomechanics`` on one 2-D or 3-D subdomain without fractures -> ``Thermoporomechanics`` (unknowns
    [u | p | T], the model's own order)."""
    from .thermoporomech import Thermoporomechanics
    sd = _single_matrix(model)
    fk, tk, mk, ck = model.darcy_keyword, model.fourier_keyword, model.stress_keyword, model.enthalpy_keyword
    data = _own_data(model.mdg.subdomain_data(sd), [fk, tk, mk])
    fluid = _fluid(model, True)
    so = model.solid
    solid = dict(reference_porosity=so.porosity, n_inv=_n_inv(model), biot_coefficient=so.biot_coefficient,
                 thermal_expansion=so.thermal_expansion, heat_capacity=so.specific_heat_capacity,
                 conductivity=so.thermal_conductivity, density=so.density)
    w, we = _boundary_weights(model, sd, fluid, True)
    ff, ef = model.bc_type_fluid_flux(sd), model.bc_type_enthalpy_flux(sd)
    prm = data[PARAMETERS]
    bc = dict(flow=_face_values(model, sd, prm[fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
              fourier=_face_values(model, sd, prm[tk]["bc"], model.bc_values_temperature, model.bc_values_fourier_flux),
              mechanics=_mechanics_boundary(model, sd, data, mk),
              fluid_flux=_face_values(model, sd, ff, w, model.bc_values_fluid_flux),
              enthalpy_flux=_face_values(model, sd, ef, we, model.bc_values_enthalpy_flux),
              fluid_flux_type=ff, enthalpy_flux_type=ef)
    prob = Thermoporomechanics(sd, data, fluid, solid, bc, flow_keyword=fk, fourier_keyword=tk, mechanics_keyword=mk,
                               thermal_keyword=ck)
    prob.mobility_keyword, prob.enthalpy_upwind_keyword = "b200_mobility", "b200_enthalpy_upwind"
    return prob


def fractured_momentum_from_model(model):
    """``pp.MomentumBalance`` with fractures in frictional contact -> (``FracturedMomentumBalance``, column_map): one
    nd-D matrix subdomain (nd = 2 or 3), any number of (nd - 1)-D fractures without intersections (each with its
    two-sided interface); unknown k of the problem is dof ``column_map[k]`` of the model ([u | contact tractions |
    interface displacements])."""
    from .contact import FractureContact, FracturedMomentumBalance
    mat, fracs, grids = _matrix_and_fractures(model)
    mdg = model.mdg
    mk = model.stress_keyword
    data = _own_data(mdg.subdomain_data(mat), [mk])
    contacts = []
    for j, frac in enumerate(fracs):
        intf = grids[("interface", j)]
        rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
        contacts.append(FractureContact(intf.mortar_to_primary_avg(), intf.primary_to_mortar_int(),
                                        intf.mortar_to_secondary_avg(), intf.secondary_to_mortar_int(),
                                        sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), intf.cell_volumes, rot))
    prob = FracturedMomentumBalance(mat, data, _mechanics_boundary(model, mat, data, mk), contacts,
                                    _contact_constants(model, fracs), keyword=mk)
    return prob, _column_map(model, prob.unknown_layout, grids)


def _contact_constants(model, fracs):
    def scalar(op):
        return float(np.atleast_1d(_evaluated(model, op, 1))[0])
    return dict(numerical_constant=scalar(model.contact_mechanics_numerical_constant(fracs)),
                characteristic_traction=scalar(model.characteristic_contact_traction(fracs)),
                friction_coefficient=scalar(model.friction_coefficient(fracs)),
                dilation_angle=model.solid.dilation_angle, reference_gap=model.solid.fracture_gap,
                open_state_tolerance=model.numerical.open_state_tolerance)


def _fractured_problem(model, thermal: bool):
    """Shared part of the two fractured (thermo-)poromechanics bridges."""
    from .fractured_poromech import FractureCoupling
    mat, fracs, grids = _matrix_and_fractures(model)
    mdg = model.mdg
    fk, mk = model.darcy_keyword, model.stress_keyword
    kws = [fk, mk] + ([model.fourier_keyword] if thermal else [])
    data = _own_data(mdg.subdomain_data(mat), kws)
    a_res = model.solid.residual_aperture
    couplings, kappa_t = [], []
    for j, frac in enumerate(fracs):
        intf = grids[("interface", j)]
        fdata = _own_data(mdg.subdomain_data(frac), [fk] + ([model.fourier_keyword] if thermal else []))
        k_now = np.asarray(fdata[PARAMETERS][fk]["second_order_tensor"].values, float)
        a_now = _evaluated(model, model.specific_volume([frac]), frac.num_cells)       # the tensor holds k x specific volume
        proj = {name: getattr(intf, name)() for name in (
            "mortar_to_primary_avg", "primary_to_mortar_int", "mortar_to_secondary_avg", "secondary_to_mortar_int",
            "mortar_to_primary_int", "primary_to_mortar_avg", "mortar_to_secondary_int", "secondary_to_mortar_avg")}
        rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
        fbc = None
        if np.any(np.asarray(frac.tags["domain_boundary_faces"], bool)):      # the fracture reaches the domain boundary
            fl_ = _fluid(model, thermal)
            wf_, wef_ = _boundary_weights(model, frac, fl_, thermal)
            fft = model.bc_type_fluid_flux(frac)
            fbc = dict(flow=_face_values(model, frac, fdata[PARAMETERS][fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
                       fluid_flux=_face_values(model, frac, fft, wf_, model.bc_values_fluid_flux), fluid_flux_type=fft)
            if thermal:
                eft = model.bc_type_enthalpy_flux(frac)
                fbc.update(fourier=_face_values(model, frac, fdata[PARAMETERS][model.fourier_keyword]["bc"],
                                                model.bc_values_temperature, model.bc_values_fourier_flux),
                           enthalpy_flux=_face_values(model, frac, eft, wef_, model.bc_values_enthalpy_flux),
                           enthalpy_flux_type=eft)
        couplings.append(FractureCoupling(frac, fdata, proj, sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(),
                                          intf.cell_volumes, rot, _evaluated(model, model.normal_permeability([intf]), intf.num_cells),
                                          k_now / a_now[None, None, :], bc=fbc))
        if thermal:
            kappa_t.append(_evaluated(model, model.normal_thermal_conductivity([intf]), intf.num_cells))
    fluid = _fluid(model, thermal)
    so = model.solid
    solid = dict(reference_porosity=so.porosity, n_inv=_n_inv(model), residual_aperture=a_res)
    w, we = _boundary_weights(model, mat, fluid, thermal)
    ff = model.bc_type_fluid_flux(mat)
    prm = data[PARAMETERS]
    bc = dict(flow=_face_values(model, mat, prm[fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
              mechanics=_mechanics_boundary(model, mat, data, mk),
              fluid_flux=_face_values(model, mat, ff, w, model.bc_values_fluid_flux), fluid_flux_type=ff)
    return mat, fracs, data, couplings, fluid, solid, bc, kappa_t, (w, we), grids


def fractured_poromechanics_from_model(model):
    """``pp.Poromechanics`` on a fractured medium with frictional contact -> (``FracturedPoromechanics``, column_map,
    row_map)."""
    from .fractured_poromech import FracturedPoromechanics
    mat, fracs, data, couplings, fluid, solid, bc, _, _, grids = _fractured_problem(model, False)
    prob = FracturedPoromechanics(mat, data, couplings, fluid, solid, _contact_constants(model, fracs), bc,
                                  flow_keyword=model.darcy_keyword, mechanics_keyword=model.stress_keyword)
    prob.mobility_keyword = "b200_mobility"
    return prob, _column_map(model, prob.unknown_layout, grids), _row_map(model, prob.equation_layout)


def fractured_thermoporomechanics_from_model(model):
    """``pp.Thermoporomechanics`` on a fractured medium with frictional contact (BASELINE config[4]) ->
    (``FracturedThermoporomechanics``, column_map, row_map)."""
    from .fractured_thm import FracturedThermoporomechanics
    mat, fracs, data, couplings, fluid, solid, bc, kappa_t, (w, we), grids = _fractured_problem(model, True)
    so = model.solid
    solid.update(biot_coefficient=so.biot_coefficient, thermal_expansion=so.thermal_expansion,
                 heat_capacity=so.specific_heat_capacity, conductivity=so.thermal_conductivity, density=so.density)
    tk = model.fourier_keyword
    ef = model.bc_type_enthalpy_flux(mat)
    bc.update(fourier=_face_values(model, mat, data[PARAMETERS][tk]["bc"], model.bc_values_temperature, model.bc_values_fourier_flux),
              enthalpy_flux=_face_values(model, mat, ef, we, model.bc_values_enthalpy_flux), enthalpy_flux_type=ef)
    prob = FracturedThermoporomechanics(mat, data, couplings, fluid, solid, _contact_constants(model, fracs), bc, kappa_t,
                                        flow_keyword=model.darcy_keyword, fourier_keyword=tk,
                                        mechanics_keyword=model.stress_keyword, thermal_keyword=model.enthalpy_keyword)
    prob.mobility_keyword, prob.enthalpy_upwind_keyword = "b200_mobility", "b200_enthalpy_upwind"
    return prob, _column_map(model, prob.unknown_layout, grids), _row_map(model, prob.equation_layout)


def _tpsa_grid(model, name: str, other=None):
    """The one 2-D or 3-D subdomain of a TPSA model without fractures, for the problem class ``name``.  ``other``:
    (equation, message) of a model family the class does not solve, refused when the model has that equation."""
    mdg = model.mdg
    sds = list(mdg.subdomains())
    if any(sd.dim < model.nd for sd in sds) or any(True for _ in mdg.interfaces()):
        raise NotImplementedError(f"{name}: fractures are not supported")
    if len(sds) != 1:
        raise NotImplementedError(f"{name}: one subdomain is expected")
    if other is not None and other[0] in model.equation_system.equations:
        raise NotImplementedError(f"{name}: {other[1]}")
    if sds[0].dim not in (2, 3):
        raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")
    return sds[0]


def _tpsa_mechanics(model, sd) -> tuple:
    """(the mechanical boundary operator, {body_force, angular_source, mass_source}) of ``sd``: the model's own
    ``combine_boundary_operators_mechanical_stress``, ``body_force``, ``source_angular_momentum`` and
    ``solid_mass_source``, evaluated."""
    nd, nc = int(sd.dim), sd.num_cells
    g = _evaluated(model, model.combine_boundary_operators_mechanical_stress([sd]), nd * sd.num_faces)
    return g, dict(body_force=_evaluated(model, model.body_force([sd]), nd * nc),
                   angular_source=_evaluated(model, model.source_angular_momentum([sd]),
                                             model.rotation_dimension() * nc),
                   mass_source=_evaluated(model, model.solid_mass_source([sd]), nc))


def _tpsa_maps(model, prob, grids) -> tuple:
    """Set and return (column_map, row_map) of a TPSA problem: the model's dofs of ``prob.fields`` and rows of
    ``prob.balances`` on the matrix, interleaved cell by cell, then those of the blocks behind the cell block of its
    layouts.  The poromechanics models call the solid-mass equation ``Solid_mass_equation_poromechanics``."""
    from .tpsa_elasticity import interleave
    nc, equations = prob.nc, model.equation_system.equations

    def cell_interleaved(cell_blocks, tail, model_order):
        layout = BlockLayout([(name, [(("matrix",), nc, w)]) for name, w in cell_blocks] + tail)
        idx, ends, k = model_order(layout), layout.offsets, len(cell_blocks)
        return np.concatenate([interleave([idx[a:b] for a, b in zip(ends[:k], ends[1:k + 1])], prob.nd, prob.nr, nc),
                               idx[ends[k]:]])

    prob.column_map = cell_interleaved(prob.fields, prob.unknown_layout.blocks[1:],
                                       lambda layout: _column_map(model, layout, grids))
    balances = [(name if name in equations else next(eq for eq in equations if eq.lower().startswith(name)), w)
                for name, w in prob.balances]
    prob.row_map = cell_interleaved(balances, prob.equation_layout.blocks[1:], lambda layout: _row_map(model, layout))
    return prob.column_map, prob.row_map


def tpsa_momentum_from_model(model):
    """A prepared ``pp.MomentumBalance`` with ``TpsaMomentumBalanceMixin`` on one 2-D or 3-D grid without fractures ->
    (``TpsaElasticity``, column_map, row_map): unknown k of the problem (cell-interleaved [u_c, r_c, p_c]) is dof
    ``column_map[k]`` of the model's ``EquationSystem``, equation k its row ``row_map[k]``.  The boundary operator g is
    the model's own ``combine_boundary_operators_mechanical_stress``, evaluated; f is its ``body_force``, s_r / s_p its
    ``source_angular_momentum`` / ``solid_mass_source``."""
    from .tpsa_elasticity import TpsaElasticity
    sd = _tpsa_grid(model, "TpsaElasticity", ("mass_balance_equation", "the TPSA poromechanics model (four fields) is "
                                              "not supported; use tpsa_poromechanics_from_model"))
    mk = model.stress_keyword
    g, sources = _tpsa_mechanics(model, sd)
    prob = TpsaElasticity(sd, _own_data(model.mdg.subdomain_data(sd), [mk]), mk, g, **sources)
    return (prob, *_tpsa_maps(model, prob, {("matrix",): sd}))


def _tpsa_solid(model, sd, thermal: bool) -> dict:
    so, nc = model.solid, sd.num_cells
    solid = dict(reference_porosity=so.porosity, biot_coefficient=_evaluated(model, model.biot_coefficient([sd]), nc),
                 bulk_modulus=float(np.atleast_1d(_evaluated(model, model.bulk_modulus([sd]), 1))[0]))
    if thermal:
        solid.update(thermal_expansion=so.thermal_expansion, heat_capacity=so.specific_heat_capacity,
                     conductivity=so.thermal_conductivity, density=so.density)
    return solid


def tpsa_poromechanics_from_model(model):
    """A prepared ``pp.Poromechanics`` with ``TpsaPoromechanicsMixin`` on one 2-D or 3-D grid without fractures ->
    (``TpsaPoromechanics``, column_map, row_map): unknown k of the problem (cell-interleaved [u_c, r_c, p_t_c, p_c]) is
    dof ``column_map[k]`` of the model's ``EquationSystem``, equation k its row ``row_map[k]``.  The mechanical boundary
    operator, body force, sources, Darcy and fluid-flux boundary data are the model's own operators, evaluated."""
    from .tpsa_poromech import TpsaPoromechanics
    sd = _tpsa_grid(model, "TpsaPoromechanics", ("energy_balance_equation", "the TPSA thermo-poromechanics model (five "
                                                 "fields) is not supported; use tpsa_thermoporomechanics_from_model"))
    fk, mk = model.darcy_keyword, model.stress_keyword
    data = _own_data(model.mdg.subdomain_data(sd), [fk, mk])
    fluid = _fluid(model, False)
    w, _ = _boundary_weights(model, sd, fluid, False)
    bc_ff = model.bc_type_fluid_flux(sd)
    g, sources = _tpsa_mechanics(model, sd)
    prob = TpsaPoromechanics(
        sd, data, fluid, _tpsa_solid(model, sd, False),
        _face_values(model, sd, data[PARAMETERS][fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
        g, bc_ff, _face_values(model, sd, bc_ff, w, model.bc_values_fluid_flux), **sources,
        fluid_source=_evaluated(model, model.fluid_source([sd]), sd.num_cells), flow_keyword=fk, mechanics_keyword=mk)
    prob.mobility_keyword = "b200_mobility"
    return (prob, *_tpsa_maps(model, prob, {("matrix",): sd}))


def tpsa_thermoporomechanics_from_model(model):
    """A prepared ``pp.Thermoporomechanics`` with ``TpsaPoromechanicsMixin`` on one 2-D or 3-D grid without fractures ->
    (``TpsaThermoporomechanics``, column_map, row_map): unknown k of the problem (cell-interleaved
    [u_c, r_c, p_t_c, p_c, T_c]) is dof ``column_map[k]`` of the model's ``EquationSystem``, equation k its row
    ``row_map[k]``.  The mechanical boundary operator, body force, sources, Darcy, Fourier, fluid- and enthalpy-flux
    boundary data are the model's own operators, evaluated.  The Fourier conductivity is the one of the zero state, which
    the model discretizes with when its initial values are zero (its default); for other initial values set
    ``prob.conductivity`` before ``discretize``."""
    from .tpsa_thermoporomech import TpsaThermoporomechanics
    sd = _tpsa_grid(model, "TpsaThermoporomechanics")
    fk, tk, mk = model.darcy_keyword, model.fourier_keyword, model.stress_keyword
    data = _own_data(model.mdg.subdomain_data(sd), [fk, tk, mk])
    fluid = _fluid(model, True)
    w, we = _boundary_weights(model, sd, fluid, True)
    ff, ef = model.bc_type_fluid_flux(sd), model.bc_type_enthalpy_flux(sd)
    prm = data[PARAMETERS]
    g, sources = _tpsa_mechanics(model, sd)
    prob = TpsaThermoporomechanics(
        sd, data, fluid, _tpsa_solid(model, sd, True),
        _face_values(model, sd, prm[fk]["bc"], model.bc_values_pressure, model.bc_values_darcy_flux),
        _face_values(model, sd, prm[tk]["bc"], model.bc_values_temperature, model.bc_values_fourier_flux),
        g, ff, _face_values(model, sd, ff, w, model.bc_values_fluid_flux), ef,
        _face_values(model, sd, ef, we, model.bc_values_enthalpy_flux), **sources,
        fluid_source=_evaluated(model, model.fluid_source([sd]), sd.num_cells), flow_keyword=fk, fourier_keyword=tk,
        mechanics_keyword=mk)
    prob.mobility_keyword, prob.enthalpy_upwind_keyword = "b200_mobility", "b200_enthalpy_upwind"
    return (prob, *_tpsa_maps(model, prob, {("matrix",): sd}))


def tpsa_fractured_momentum_from_model(model):
    """A prepared ``pp.MomentumBalance`` with ``TpsaMomentumBalanceMixin`` on one 2-D or 3-D matrix with fractures in
    frictional contact (one dimension less, no intersections, matching mortar grids) ->
    (``TpsaFracturedMomentumBalance``, column_map, row_map): unknown k of the problem ([u_c, r_c, p_c per matrix cell |
    contact traction | interface displacement]) is dof ``column_map[k]`` of the model's ``EquationSystem``, equation k its
    row ``row_map[k]``.  The boundary operator is the model's own ``combine_boundary_operators_mechanical_stress``,
    evaluated; the body force and the angular and solid-mass sources are its own operators, evaluated."""
    from .contact import FractureContact
    from .tpsa_contact import TpsaFracturedMomentumBalance
    if "mass_balance_equation" in model.equation_system.equations:
        raise NotImplementedError("TpsaFracturedMomentumBalance: fractured TPSA poromechanics is not supported")
    mat, fracs, grids = _matrix_and_fractures(model)
    if getattr(mat, "periodic_face_map", None) is not None:
        raise NotImplementedError("periodic faces are not supported by porepy_b200")
    mdg = model.mdg
    mk = model.stress_keyword
    contacts = []
    for j, frac in enumerate(fracs):
        intf = grids[("interface", j)]
        rot = mdg.subdomain_data(frac)["tangential_normal_projection"].project_tangential_normal(frac.num_cells)
        contacts.append(FractureContact(intf.mortar_to_primary_avg(), intf.primary_to_mortar_int(),
                                        intf.mortar_to_secondary_avg(), intf.secondary_to_mortar_int(),
                                        sps.csr_matrix(intf.sign_of_mortar_sides(1)).diagonal(), intf.cell_volumes, rot))
    g, sources = _tpsa_mechanics(model, mat)
    prob = TpsaFracturedMomentumBalance(mat, _own_data(mdg.subdomain_data(mat), [mk]), g, contacts,
                                        _contact_constants(model, fracs), **sources, keyword=mk)
    return (prob, *_tpsa_maps(model, prob, grids))
