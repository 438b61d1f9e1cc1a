"""Mass and energy balance in a fracture network, the reference's ``pp.MassAndEnergyBalance`` on the device AD chain --
the thermal half of BASELINE config[4] on a mixed-dimensional grid (the mechanical half on a 3-D subdomain:
``porepy_b200.thermoporomech``; frictional contact on a fracture: ``porepy_b200.contact``).

Per subdomain: pressure and temperature; per interface: Darcy flux ``lambda``, Fourier flux ``eta``, enthalpy flux ``eps``.

* density, weights         rho = rho0 exp(c (p - p0) - beta (T - T0)),  w = rho / mu,  w_e = c_f (T - T0) w
* mass balance             vol phi (rho - rho_n) / dt + div [q (U w) + B_dir (q w_b) + B_neu (w_b + Pi lambda (U_h tr w + U_l w))]
                           - Pi^int (lambda ...) - source                       models/fluid_mass_balance.py:147-345
* energy balance           vol (E - E_n) / dt + div [Fourier + enthalpy flux] - Pi^int (eta + eps),
                           E = (rho c_f (T - T0) - p) phi + rho_s c_s (T - T0) (1 - phi)      models/energy_balance.py:165-352
* Fourier flux             flux_T T + bound_flux_T (T_b + Pi eta)   (``porepy_b200.Mpfa`` on every subdomain)
* interface laws           lambda - vol kappa   (2 / a) (Pi tr(p) - Pi p_l)     constitutive_laws.py:1032-1076
                           eta    - vol kappa_T (2 / a) (Pi tr(T) - Pi T_l)     constitutive_laws.py:2342-2386
                           eps    - lambda (U_h Pi tr(w_e) + U_l Pi w_e)        energy_balance.py:353-376

Unknowns and equations: ``unknown_layout``, ``equation_layout`` (the reference interleaves both per grid;
``tests/golden/mdthermal_*.npz`` carry the index maps).  Upwinding (``porepy_b200.Upwind`` / ``UpwindCoupling``, shared
by the mass and the enthalpy flux: same Darcy flux) is re-discretized from the iterate in front of every linearization.
Every Newton step eliminates the three interface unknown sets (``mdflow_nl.schur_solver``).
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps

from . import ad
from .advection import advective_flux, rediscretize_upwind, rediscretize_upwind_coupling
from .fv import Mpfa
from .layout import BlockLayout, LayoutModel
from .mdflow_nl import equation_system, schur_solver
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES


class MixedDimensionalMassEnergy(LayoutModel):
    """``subdomains``: ``mdflow.MdSubdomain`` records whose data dictionaries hold ``parameters[flow_keyword]`` and
    ``parameters[fourier_keyword]`` (``second_order_tensor``, ``bc``, ``ambient_dimension``); ``interfaces``:
    ``mdflow.MdInterface`` records.  Per subdomain (lists): ``volume`` (cell volume x specific volume), ``porosity``,
    ``bc_values`` = dict(flow=, fourier=, fluid_flux=, enthalpy_flux=) face arrays, ``bc_types`` = dict(fluid_flux=,
    enthalpy_flux=) boundary-condition objects of the two upwind schemes.  ``normal_thermal_conductivity``: one array per
    interface.  ``fluid``: ``compressibility, density, viscosity, thermal_expansion, heat_capacity, reference_pressure,
    reference_temperature``; ``solid``: ``density, heat_capacity``."""

    mobility_keyword = "mobility"
    enthalpy_upwind_keyword = "enthalpy_upwind"

    def __init__(self, subdomains, interfaces, fluid: dict, solid: dict, volume, porosity, bc_values, bc_types,
                 normal_thermal_conductivity, sources=None, flow_keyword: str = "flow", fourier_keyword: str = "fourier"):
        self.subdomains, self.interfaces = list(subdomains), list(interfaces)
        self.fk, self.tk = flow_keyword, fourier_keyword
        self.fl = SimpleNamespace(**{k: float(v) for k, v in fluid.items()})
        self.so = SimpleNamespace(**{k: float(v) for k, v in solid.items()})
        self.volume = [np.asarray(v, float) for v in volume]
        self.porosity = [np.asarray(v, float) for v in porosity]
        self.bc_values, self.bc_types = list(bc_values), list(bc_types)
        self.kappa_t = [np.asarray(v, float) for v in normal_thermal_conductivity]
        self.sources = [np.zeros(s.sd.num_cells) if (sources is None or sources[i] is None) else np.asarray(sources[i], float)
                        for i, s in enumerate(self.subdomains)]
        sub = [(("subdomain", i), int(s.sd.num_cells), 1) for i, s in enumerate(self.subdomains)]
        intf = [(("interface", j), it.num_cells, 1) for j, it in enumerate(self.interfaces)]
        self.unknown_layout = BlockLayout([("pressure", sub), ("temperature", sub), ("interface_darcy_flux", intf),
                                           ("interface_fourier_flux", intf), ("interface_enthalpy_flux", intf)])
        self.equation_layout = BlockLayout([
            ("mass_balance_equation", sub), ("energy_balance_equation", sub), ("interface_darcy_flux_equation", intf),
            ("interface_fourier_flux_equation", intf), ("interface_enthalpy_flux_equation", intf)])
        self._intf_data = [{} for _ in self.interfaces]
        self._const = None

    def discretize(self) -> None:
        """Darcy and Fourier flux of every subdomain with faces (``porepy_b200.Mpfa``; lines: TPFA), once."""
        for s in self.subdomains:
            if s.sd.num_faces > 0:
                Mpfa(self.fk).discretize(s.sd, s.data)
                Mpfa(self.tk).discretize(s.sd, s.data)
        self._const = None

    def _operands(self):
        if self._const is None:
            csr, dev = ad.as_device_csr, ad.device_vector
            k = SimpleNamespace(div=[], trace=[], vol=[], phi=[], src=[], bc=[], F=[], Fo=[], m2p=[], p2m=[], m2s=[], s2m=[],
                                coef=[], coef_t=[])
            for i, s in enumerate(self.subdomains):
                has = s.sd.num_faces > 0
                k.div.append(csr(sps.csr_matrix(s.sd.cell_faces.T)) if has else None)
                k.trace.append(csr(abs(sps.csr_matrix(s.sd.cell_faces))) if has else None)
                k.vol.append(dev(self.volume[i]))
                k.phi.append(dev(self.porosity[i]))
                k.src.append(dev(self.sources[i]))
                k.bc.append({key: dev(v) for key, v in self.bc_values[i].items()} if has else None)
                mats = s.data[DISCRETIZATION_MATRICES] if has else None
                k.F.append({key: csr(mats[self.fk][key]) for key in ("flux", "bound_flux", "bound_pressure_cell",
                                                                      "bound_pressure_face")} if has else None)
                k.Fo.append({key: csr(mats[self.tk][key]) for key in ("flux", "bound_flux", "bound_pressure_cell",
                                                                       "bound_pressure_face")} if has else None)
            for j, it in enumerate(self.interfaces):
                k.m2p.append(csr(it.mortar_to_primary_int))
                k.p2m.append(csr(it.primary_to_mortar_avg))
                k.m2s.append(csr(it.mortar_to_secondary_int))
                k.s2m.append(csr(it.secondary_to_mortar_avg))
                geo = it.coefficient() / np.asarray(it.normal_permeability, float)      # vol * 2 / a
                k.coef.append(dev(it.coefficient()))
                k.coef_t.append(dev(geo * self.kappa_t[j]))
            self._const = k
        return self._const

    def _density(self, p, t):
        fl = self.fl
        return ((p - fl.reference_pressure) * fl.compressibility
                - (t - fl.reference_temperature) * fl.thermal_expansion).exp() * fl.density

    def _energy(self, p, t, phi):
        dtm = t - self.fl.reference_temperature
        return (self._density(p, t) * dtm * self.fl.heat_capacity - p) * phi \
            + (dtm * (self.so.density * self.so.heat_capacity)) * (-phi + 1.0)

    def _boundary(self, i, key, flux, k):
        """bc + sum of the projected interface fluxes: what bound_flux / bound_pressure_face act on."""
        b = k.bc[i][key]
        for j, it in enumerate(self.interfaces):
            if it.primary == i:
                b = (k.m2p[j] @ flux[j]) + b
        return b

    def update_upwind(self, x) -> None:
        x = ad.device_vector(x)
        k = self._operands()
        parts = self.unknown_layout.parts(x)
        p, lam = parts["pressure"], parts["interface_darcy_flux"]
        for i, s in enumerate(self.subdomains):
            if s.sd.num_faces == 0:
                continue
            q = ((k.F[i]["flux"] @ p[i]) + (k.F[i]["bound_flux"] @ self._boundary(i, "flow", lam, k))).cpu().numpy()
            for kw, key in ((self.mobility_keyword, "fluid_flux"), (self.enthalpy_upwind_keyword, "enthalpy_flux")):
                rediscretize_upwind(s.sd, s.data, kw, q, self.bc_types[i][key])
        for j, it in enumerate(self.interfaces):
            h, l = self.subdomains[it.primary], self.subdomains[it.secondary]
            rediscretize_upwind_coupling(h.sd, l.sd, it.num_cells, h.data, l.data, self._intf_data[j],
                                         self.mobility_keyword, lam[j].cpu().numpy())

    def equations(self, x, x_prev, dt: float) -> list:
        k = self._operands()
        csr = ad.as_device_csr
        fl = self.fl
        nsd = len(self.subdomains)
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var, prev = self.unknown_layout.variables(x), self.unknown_layout.parts(x_prev)
        p, t = var["pressure"], var["temperature"]
        lam, eta, eps = var["interface_darcy_flux"], var["interface_fourier_flux"], var["interface_enthalpy_flux"]
        pn, tn = prev["pressure"], prev["temperature"]
        w = [self._density(p[i], t[i]) * (1.0 / fl.viscosity) for i in range(nsd)]
        we = [w[i] * (t[i] - fl.reference_temperature) * fl.heat_capacity for i in range(nsd)]
        ifl, enthalpy_law = [], []
        for j, it in enumerate(self.interfaces):
            U = self._intf_data[j][DISCRETIZATION_MATRICES][self.mobility_keyword]
            up, us = csr(U["upwind_primary"]), csr(U["upwind_secondary"])
            h, l = it.primary, it.secondary

            def upwinded(wh, wl):
                return (up @ (k.p2m[j] @ (k.trace[h] @ wh))) + (us @ (k.s2m[j] @ wl))
            ifl.append(lam[j] * upwinded(w[h], w[l]))
            enthalpy_law.append(eps[j] - lam[j] * upwinded(we[h], we[l]))
        mass, energy, bq, bt = [], [], [None] * nsd, [None] * nsd
        for i, s in enumerate(self.subdomains):
            rho, rho_n = self._density(p[i], t[i]), self._density(pn[i], tn[i])
            m_eq = (rho - rho_n) * (k.vol[i] * k.phi[i] * (1.0 / dt))
            e_eq = (self._energy(p[i], t[i], k.phi[i]) - self._energy(pn[i], tn[i], k.phi[i])) * (k.vol[i] * (1.0 / dt))
            if s.sd.num_faces > 0:
                bq[i], bt[i] = self._boundary(i, "flow", lam, k), self._boundary(i, "fourier", eta, k)
                Tm = s.data[DISCRETIZATION_MATRICES][self.mobility_keyword]
                Te = s.data[DISCRETIZATION_MATRICES][self.enthalpy_upwind_keyword]
                q = (k.F[i]["flux"] @ p[i]) + (k.F[i]["bound_flux"] @ bq[i])
                ff = advective_flux(Tm, q, w[i], k.bc[i]["fluid_flux"], self._boundary(i, "fluid_flux", ifl, k))
                fe = advective_flux(Te, q, we[i], k.bc[i]["enthalpy_flux"], self._boundary(i, "enthalpy_flux", eps, k))
                fo = (k.Fo[i]["flux"] @ t[i]) + (k.Fo[i]["bound_flux"] @ bt[i])
                m_eq = m_eq + (k.div[i] @ ff)
                e_eq = e_eq + (k.div[i] @ (fe + fo))
            for j, it in enumerate(self.interfaces):
                if it.secondary == i:
                    m_eq = m_eq - (k.m2s[j] @ ifl[j])
                    e_eq = e_eq - (k.m2s[j] @ (eta[j] + eps[j]))
            mass.append(m_eq - k.src[i])
            energy.append(e_eq)
        darcy_law, fourier_law = [], []
        for j, it in enumerate(self.interfaces):
            h, l = it.primary, it.secondary
            for laws, mats, hv, lv, bnd, flux, coef in ((darcy_law, k.F[h], p[h], p[l], bq[h], lam[j], k.coef[j]),
                                                        (fourier_law, k.Fo[h], t[h], t[l], bt[h], eta[j], k.coef_t[j])):
                trace = (mats["bound_pressure_cell"] @ hv) + (mats["bound_pressure_face"] @ bnd)
                laws.append(flux - ((k.p2m[j] @ trace) - (k.s2m[j] @ lv)) * coef)
        return self.equation_layout.stack({
            "mass_balance_equation": mass, "energy_balance_equation": energy,
            "interface_darcy_flux_equation": darcy_law, "interface_fourier_flux_equation": fourier_law,
            "interface_enthalpy_flux_equation": enthalpy_law})

    def linearize(self, x, x_prev, dt: float):
        self.update_upwind(x)
        return ad.assemble(self.equations(x, x_prev, dt))

    def time_step(self, x_prev, dt: float, tol: float = 1e-10, max_iterations: int = 20, linear_tol: float = 1e-10,
                  verbose: bool = False):
        """One implicit time step by Newton's method; every step on the Schur complement of the subdomain unknowns."""
        x_prev = ad.device_vector(x_prev)

        def linearize(x):
            self.update_upwind(x)
            return equation_system(self.equations(x, x_prev, dt))
        solver = schur_solver(self.unknown_layout, self.equation_layout, linear_tol)
        return newton_loop(linearize, x_prev, solver, tol, max_iterations, verbose)
