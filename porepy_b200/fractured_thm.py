"""Thermo-poromechanics of a fractured medium with frictional contact -- BASELINE config[4] ("thermo-poromechanics +
frictional contact, fracture network, full Newton loop") as the reference states it: ``pp.Thermoporomechanics`` on a matrix
cut by fractures, every term and its Jacobian by ``DeviceAdArray`` on device-resident matrices.

The union of ``porepy_b200.fractured_poromech`` (poromechanics, fracture flow with jump-dependent aperture, contact),
``porepy_b200.thermoporomech`` (thermal stress, thermally expanding fluid, thermo-poromechanical porosity, internal energy)
and ``porepy_b200.mdthermal`` (Fourier and enthalpy fluxes on subdomains and interfaces), with the aperture in the
fracture's internal energy and in the interface Fourier law:

* fracture energy        vol a (rho c_f (T - T0) - p)        (porosity 1, specific volume a)
* interface Fourier law  eta - vol kappa_T (2 Pi (1 / a)) (Pi tr T - Pi T_f)                constitutive_laws.py:2342-2386
* fracture conductivity  k_f a: the fracture's Fourier flux is re-discretized with the iterate's aperture like its Darcy
                         flux (measured on the reference: both flux matrices x 1.002 at the second iterate); the matrix's
                         flux matrices stay those of the initial state.

Unknowns and equations: those of ``FracturedPoromechanics`` with the temperatures, the interface Fourier and enthalpy
fluxes and their equations inserted (``unknown_layout``, ``equation_layout``).  ``tests/golden/contact_thm*.npz`` pin
the Jacobian at the zero state and at the fourth Newton iterate, the residual history of the semismooth Newton loop and
the converged state.  The Newton updates are solved on the device by ``krylov.gmres_solver(prob.preconditioner_groups())``
(3 nd + 8 unknowns per fracture-cell group: 17 in 3-D, 14 in 2-D).  A 2-D matrix with line fractures is handled as the
3-D one (``contact_thm_2d.npz``).
"""
from __future__ import annotations

import numpy as np

from . import ad
from .advection import advective_flux
from .contact import contact_laws, fracture_parts, interface_parts
from .fractured_poromech import FracturedPoromechanics
from .fv import Mpfa
from .params import DISCRETIZATION_MATRICES, PARAMETERS, SecondOrderTensor


class FracturedThermoporomechanics(FracturedPoromechanics):
    """As ``FracturedPoromechanics``, plus: ``data[parameters][fourier_keyword]`` (``bc``) for the matrix and for every
    fracture (``FractureCoupling.data``); ``scalar_vector_mappings`` of the mechanics parameters hold the thermal-stress
    tensor under ``thermal_keyword``; ``fluid`` adds ``thermal_expansion, heat_capacity, conductivity,
    reference_temperature``; ``solid`` adds ``biot_coefficient, thermal_expansion, heat_capacity, conductivity, density``;
    ``bc`` adds the face arrays ``fourier``, ``enthalpy_flux`` and the object ``enthalpy_flux_type``;
    ``normal_thermal_conductivity``: one array per fracture interface."""

    enthalpy_upwind_keyword = "enthalpy_upwind"

    def __init__(self, sd, data: dict, fractures, fluid: dict, solid: dict, contact: dict, bc: dict,
                 normal_thermal_conductivity, flow_keyword: str = "flow", fourier_keyword: str = "fourier",
                 mechanics_keyword: str = "mechanics", thermal_keyword: str = "thermal"):
        super().__init__(sd, data, fractures, fluid, solid, contact, bc, flow_keyword, mechanics_keyword)
        self.tk, self.ck = fourier_keyword, thermal_keyword
        self.kappa_t = [np.asarray(v, float) for v in normal_thermal_conductivity]
        scalar = [(("matrix",), self.nc, 1)] + fracture_parts(self.fractures, 1)
        flux = interface_parts(self.fractures, 1)
        self.unknown_layout = self.unknown_layout.insert("pressure", [("temperature", scalar)]).insert(
            "interface_darcy_flux", [("interface_fourier_flux", flux), ("interface_enthalpy_flux", flux)])
        self.equation_layout = self.equation_layout.insert("mass_balance_equation", [("energy_balance_equation", scalar)]
                                                           ).insert("interface_darcy_flux_equation", [
            ("interface_fourier_flux_equation", flux), ("interface_enthalpy_flux_equation", flux)])

    # ``preconditioner_groups()``: nd + 2 unknowns per matrix cell; per fracture cell k, those of ``FracturedPoromechanics``
    # plus the fracture energy balance of k and the Fourier and enthalpy laws of its mortar cells (3 nd + 8: 17 in 3-D)
    matrix_group = ([("mass_balance_equation", "c"), ("energy_balance_equation", "c"),
                     ("momentum_balance_equation", "c")], [("pressure", "c"), ("temperature", "c"), ("displacement", "c")])
    fracture_group = (FracturedPoromechanics.fracture_group[0] + [
                          ("energy_balance_equation", "k"), ("interface_fourier_flux_equation", "m1"),
                          ("interface_fourier_flux_equation", "m2"), ("interface_enthalpy_flux_equation", "m1"),
                          ("interface_enthalpy_flux_equation", "m2")],
                      FracturedPoromechanics.fracture_group[1] + [
                          ("temperature", "k"), ("interface_fourier_flux", "m1"), ("interface_fourier_flux", "m2"),
                          ("interface_enthalpy_flux", "m1"), ("interface_enthalpy_flux", "m2")])

    # ---- discretizations
    def _matrix_conductivity(self):
        phi = self.so.reference_porosity
        return np.full(self.nc, phi * self.fl.conductivity + (1.0 - phi) * self.so.conductivity)

    def _discretize_fracture(self, fc, aperture) -> None:
        super()._discretize_fracture(fc, aperture)
        fc.data.setdefault(PARAMETERS, {}).setdefault(self.tk, {})["second_order_tensor"] = SecondOrderTensor(
            self.fl.conductivity * np.asarray(aperture, float))          # porosity 1 in the fracture, specific volume a
        fc.data[PARAMETERS][self.tk].setdefault("ambient_dimension", self.nd)
        Mpfa(self.tk).discretize(fc.sd, fc.data)

    def discretize(self) -> None:
        self.data[PARAMETERS][self.tk]["second_order_tensor"] = SecondOrderTensor(self._matrix_conductivity())
        Mpfa(self.tk).discretize(self.sd, self.data)
        super().discretize()

    def _operands(self):
        fresh = self._const is None
        k = super()._operands()
        if fresh:
            csr, dev = ad.as_device_csr, ad.device_vector
            Fo = self.data[DISCRETIZATION_MATRICES][self.tk]
            M = self.data[DISCRETIZATION_MATRICES][self.mk]
            k.Fo = {key: csr(Fo[key]) for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face")}
            k.grad_t = csr(M["scalar_gradient"][self.ck])
            k.bct, k.bce = dev(self.bc["fourier"]), dev(self.bc["enthalpy_flux"])
            for j, fc in enumerate(self.fractures):
                k.fr[j].coef_t = dev(fc.volumes * self.kappa_t[j] * 2.0)
        return k

    # ---- constitutive laws
    def _density(self, p, t=None):
        fl = self.fl
        e = (p - fl.reference_pressure) * fl.compressibility
        if t is not None:
            e = e - (t - fl.reference_temperature) * fl.thermal_expansion
        return e.exp() * fl.density

    def _porosity(self, p, t, u, uj, k):
        so = self.so
        return super()._porosity(p, u, uj, k) \
            - (t - self.fl.reference_temperature) * ((so.biot_coefficient - so.reference_porosity) * so.thermal_expansion)

    def _upwind_keywords(self):
        return super()._upwind_keywords() + [(self.enthalpy_upwind_keyword, "enthalpy_flux_type")]

    def equations(self, x, x_prev, dt: float) -> list:
        k, fl, so = self._operands(), self.fl, self.so
        csr = ad.as_device_csr
        nfr = len(self.fractures)
        mk, ek = self.mobility_keyword, self.enthalpy_upwind_keyword
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var, prev = self.unknown_layout.variables(x), self.unknown_layout.parts(x_prev)
        (p3, *pf), (t3, *tf), (u,) = var["pressure"], var["temperature"], var["displacement"]
        lam, eta, eps = var["interface_darcy_flux"], var["interface_fourier_flux"], var["interface_enthalpy_flux"]
        t, uj = var["contact_traction"], var["interface_displacement"]
        (p3n, *pfn), (t3n, *tfn), (un,) = prev["pressure"], prev["temperature"], prev["displacement"]
        ujn = prev["interface_displacement"]
        t0 = fl.reference_temperature

        def weights(p, tt):
            w = self._density(p, tt) * (1.0 / fl.viscosity)
            return w, w * (tt - t0) * fl.heat_capacity
        w3, we3 = weights(p3, t3)
        wf, wef = zip(*[weights(pf[j], tf[j]) for j in range(nfr)]) if nfr else ((), ())
        ifl, enthalpy, b_flow, b_heat, b_mech = [], [], k.bcq, k.bct, k.ubc
        for j in range(nfr):
            q = k.fr[j]
            U = self._intf_data[j][DISCRETIZATION_MATRICES][mk]
            up, us = csr(U["upwind_primary"]), csr(U["upwind_secondary"])

            def upwinded(a3, af):
                return (up @ (q.p2m @ (k.trace @ a3))) + (us @ (q.s2m @ af))
            ifl.append(lam[j] * upwinded(w3, wf[j]))
            enthalpy.append(eps[j] - lam[j] * upwinded(we3, wef[j]))
            b_flow = (q.m2p @ lam[j]) + b_flow
            b_heat = (q.m2p @ eta[j]) + b_heat
            b_mech = (q.m2p_nd @ uj[j]) + b_mech
        # ---- matrix
        Tm, Te = self.data[DISCRETIZATION_MATRICES][mk], self.data[DISCRETIZATION_MATRICES][ek]
        q3 = (k.F["flux"] @ p3) + (k.F["bound_flux"] @ b_flow)
        neu_m, neu_e = k.bcw, k.bce
        for j in range(nfr):
            neu_m = (k.fr[j].m2p @ ifl[j]) + neu_m
            neu_e = (k.fr[j].m2p @ eps[j]) + neu_e
        ff3 = advective_flux(Tm, q3, w3, k.bcw, neu_m)
        fe3 = advective_flux(Te, q3, we3, k.bce, neu_e)
        fo3 = (k.Fo["flux"] @ t3) + (k.Fo["bound_flux"] @ b_heat)
        phi, phi_n = self._porosity(p3, t3, u, uj, k), self._porosity(p3n, t3n, un, ujn, k)
        rho3, rho3n = self._density(p3, t3), self._density(p3n, t3n)
        mass3 = (rho3 * phi - rho3n * phi_n) * (k.vol * (1.0 / dt)) + (k.div @ ff3)

        def energy(p, tt, rho, por):
            dtm = tt - t0
            return (rho * dtm * fl.heat_capacity - p) * por + (dtm * (so.density * so.heat_capacity)) * (-por + 1.0)
        energy3 = (energy(p3, t3, rho3, phi) - energy(p3n, t3n, rho3n, phi_n)) * (k.vol * (1.0 / dt)) + (k.div @ (fe3 + fo3))
        stress = (k.stress @ u) + (k.bound @ b_mech) + (k.grad_p @ (p3 - fl.reference_pressure)) + (k.grad_t @ (t3 - t0))
        momentum = -(k.div_nd @ stress)
        trace_p = (k.F["bound_pressure_cell"] @ p3) + (k.F["bound_pressure_face"] @ b_flow)
        trace_t = (k.Fo["bound_pressure_cell"] @ t3) + (k.Fo["bound_pressure_face"] @ b_heat)
        mass_f, energy_f, darcy, fourier, force, normal, tangential = [], [], [], [], [], [], []
        for j, fc in enumerate(self.fractures):
            q = k.fr[j]
            a, a_n = self._aperture(uj[j], q), self._aperture(ujn[j], q)
            Tf, Tef = fc.data[DISCRETIZATION_MATRICES][mk], fc.data[DISCRETIZATION_MATRICES][ek]
            qf = self._fracture_flux(fc, q, pf[j])
            fof = self._fracture_flux(fc, q, tf[j], self.tk, "fourier")
            bw, be = self._fracture_bc(q, "fluid_flux"), self._fracture_bc(q, "enthalpy_flux")
            rhof, rhofn = self._density(pf[j], tf[j]), self._density(pfn[j], tfn[j])
            mass_f.append((a * rhof - a_n * rhofn) * (q.vol * (1.0 / dt))
                          + (q.div @ advective_flux(Tf, qf, wf[j], bw, bw)) - (q.m2s @ ifl[j]))
            ef = rhof * (tf[j] - t0) * fl.heat_capacity - pf[j]                  # porosity 1: no solid part
            efn = rhofn * (tfn[j] - t0) * fl.heat_capacity - pfn[j]
            energy_f.append((a * ef - a_n * efn) * (q.vol * (1.0 / dt))
                            + (q.div @ (advective_flux(Tef, qf, wef[j], be, be) + fof))
                            - (q.m2s @ (eta[j] + eps[j])))
            inv_a = q.s2m @ a.reciprocal()
            darcy.append(lam[j] - ((q.p2m @ trace_p) - (q.s2m @ pf[j])) * inv_a * q.coef)
            fourier.append(eta[j] - ((q.p2m @ trace_t) - (q.s2m @ tf[j])) * inv_a * q.coef_t)
            force.append((q.p2m_nd @ (stress * k.outward)) + (q.traction @ t[j]) + (q.pressure_load @ pf[j]))
            nrm, tan = contact_laws(q, t[j], uj[j], ujn[j], self.ct)
            normal.append(nrm)
            tangential.append(tan)
        return self.equation_layout.stack({
            "mass_balance_equation": [mass3] + mass_f, "energy_balance_equation": [energy3] + energy_f,
            "momentum_balance_equation": [momentum], "interface_darcy_flux_equation": darcy,
            "interface_fourier_flux_equation": fourier, "interface_enthalpy_flux_equation": enthalpy,
            "interface_force_balance_equation": force, "normal_fracture_deformation_equation": normal,
            "tangential_fracture_deformation_equation": tangential})
