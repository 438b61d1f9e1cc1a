"""TPSA thermo-poromechanics on the device: the reference's ``pp.Thermoporomechanics`` with ``TpsaPoromechanicsMixin``
(models/poromechanics.py:177-213, "Can also be used to define a THM model with Tpsa"; constitutive_laws.py:3299-3374,
4799-4839; energy_balance.py:184-352) on one 2-D or 3-D grid without fractures.

Unknowns and equations per cell, cell by cell: the displacement u (nd), the rotation stress r (nr), the total pressure
p_t, the fluid pressure p and the temperature T, ``[u_c, r_c, p_t_c, p_c, T_c]``; the diagonal blocks of the Jacobian
are the (nd + nr + 3)^2 cell blocks (6 x 6 in 2-D, 9 x 9 in 3-D).

* momentum, angular momentum,    exactly the rows of ``TpsaPoromechanics``: ``ConstitutiveLawsTpsaPoromechanics.stress``
  solid mass                     is the mechanical stress alone, so the thermal stress of ``ThermoPressureStress`` never
                                 reaches the momentum balance, and the solid-mass row subtracts vol alpha / lambda p
                                 only.  These rows have no T column.
* porosity                       phi = phi0 + N^-1 (p - p0) + alpha / lambda (p_t + alpha p) - (alpha - phi0) beta_s (T - T0)
                                 (the TPSA displacement term, constitutive_laws.py:3345-3374, in
                                 ``ThermoPoroMechanicsPorosity``)
* density                        rho = rho0 exp(c (p - p0) - beta_f (T - T0))
* fluid mass balance             as in ``TpsaPoromechanics`` with this density and porosity
* energy balance                 as in ``Thermoporomechanics``: internal energy (rho c_f (T - T0) - p) phi
                                 + rho_s c_s (T - T0) (1 - phi), the Fourier flux (MPFA with the conductivity
                                 phi k_f + (1 - phi) k_s, discretized once, constitutive_laws.py:2120-2150) and the
                                 upwinded enthalpy flux with weight c_f (T - T0) rho / mu

The reference evaluates the conductivity's porosity when it discretizes, at its initial state.  With MPSA that
porosity needs a discretization matrix not yet computed, so the reference falls back on the reference porosity; the
TPSA porosity needs none, so it is the porosity of the initial state.  ``conductivity`` takes the per-cell value the
model discretized with; by default it is the one of the zero state, the reference's default initial state.

The mechanics rows are linear and constant: ``pb_tpsa_thm_system`` writes them once per ``discretize``.  At every
linearization the mass and energy balances are evaluated on the device AD chain in the variables [p_t | p | T], and
``pb_tpsa_thm_balance_rows`` writes their Jacobian rows into a fixed pattern: the whole own block plus the p and T
columns of every cell in the union of the Darcy and Fourier div @ flux patterns.  Mobility and enthalpy upwinding are
re-discretized from the iterate's Darcy flux in front of every linearization.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from . import ad
from .advection import advective_flux, rediscretize_upwind
from .fv import Mpfa
from .params import DISCRETIZATION_MATRICES, PARAMETERS, SecondOrderTensor
from .thermoporomech import Thermoporomechanics
from .tpsa_poromech import TpsaPoromechanics


class TpsaThermoporomechanics(TpsaPoromechanics):
    """As ``TpsaPoromechanics``, plus the energy balance.  ``data`` also holds ``parameters[fourier_keyword]`` with the
    ``bc`` of the Fourier flux (its conductivity tensor is written by ``discretize``).  ``fluid`` also has
    ``thermal_expansion, heat_capacity, conductivity, reference_temperature``; ``solid`` also ``thermal_expansion,
    heat_capacity, conductivity, density``.  Face data: ``fourier_bc_values`` (temperature on Dirichlet faces, flux
    elsewhere), ``bc_enthalpy_flux`` + ``enthalpy_flux_values`` (the boundary operator of the enthalpy flux).
    ``conductivity``: the cell conductivities of the Fourier flux (None: phi k_f + (1 - phi) k_s at the zero state)."""

    enthalpy_upwind_keyword = "enthalpy_upwind"
    scalar_fields = TpsaPoromechanics.scalar_fields + ("temperature",)
    scalar_balances = TpsaPoromechanics.scalar_balances + ("energy_balance_equation",)
    bridge = "tpsa_thermoporomechanics_from_model"
    outside_pattern = "mass or energy Jacobian entries outside the TPSA thermo-poromechanics row pattern"

    # the density and internal energy of the MPSA thermo-poromechanics model
    _density = Thermoporomechanics._density
    _energy = Thermoporomechanics._energy

    def __init__(self, sd, data: dict, fluid: dict, solid: dict, flow_bc_values, fourier_bc_values, mech_bc_values,
                 bc_fluid_flux, fluid_flux_values, bc_enthalpy_flux, enthalpy_flux_values, body_force=None,
                 angular_source=None, mass_source=None, fluid_source=None, flow_keyword: str = "flow",
                 fourier_keyword: str = "fourier", mechanics_keyword: str = "mechanics", conductivity=None) -> None:
        super().__init__(sd, data, fluid, solid, flow_bc_values, mech_bc_values, bc_fluid_flux, fluid_flux_values,
                         body_force=body_force, angular_source=angular_source, mass_source=mass_source,
                         fluid_source=fluid_source, flow_keyword=flow_keyword, mechanics_keyword=mechanics_keyword)
        self.tk = fourier_keyword
        self.fl = SimpleNamespace(**{k: float(v) for k, v in fluid.items()})
        self.fl.reference_pressure = self.p_ref
        self.fl.reference_temperature = float(fluid.get("reference_temperature", 0.0))
        self.so = SimpleNamespace(**{k: float(solid[k]) for k in ("thermal_expansion", "heat_capacity",
                                                                  "conductivity", "density")})
        self.so.reference_porosity = self.phi_ref
        for name, v in (("fluid thermal_expansion", self.fl.thermal_expansion),
                        ("fluid heat_capacity", self.fl.heat_capacity), ("fluid conductivity", self.fl.conductivity),
                        ("solid thermal_expansion", self.so.thermal_expansion),
                        ("solid heat_capacity", self.so.heat_capacity), ("solid conductivity", self.so.conductivity),
                        ("solid density", self.so.density), ("reference_temperature", self.fl.reference_temperature)):
            if not np.isfinite(v):
                raise ValueError(f"{name} must be finite")
        self.fourier_bc = self._vector(fourier_bc_values, self.nf, "fourier_bc_values")
        self.bc_enthalpy_flux = bc_enthalpy_flux
        self.ef_values = self._vector(enthalpy_flux_values, self.nf, "enthalpy_flux_values")
        if conductivity is None:
            zero = np.zeros(self.nc)
            k = SimpleNamespace(n_inv=self.n_inv, alpha=self.alpha, a_lam=0.0,
                                a_beta=(self.alpha - self.phi_ref) * self.so.thermal_expansion)
            phi = self._porosity(zero, zero, zero, k)
            conductivity = phi * self.fl.conductivity + (1.0 - phi) * self.so.conductivity
        self.conductivity = np.ascontiguousarray(np.broadcast_to(np.asarray(conductivity, float), (self.nc,)))
        if not np.all(np.isfinite(self.conductivity) & (self.conductivity > 0)):
            raise ValueError("the Fourier conductivity must be finite and > 0")

    def _mechanics_rows(self, mu, codes, robin, flags, pattern):
        return self._fg.tpsa_thm_system(self.nd, mu, self.lmbda, self.alpha, self.sd.cell_volumes, codes, robin,
                                        flags, self.sd.face_areas, pattern)

    def _rhs(self):
        return self._fg.tpsa_thm_rhs(self.num_dofs, self.bc_values, self.body_force, self.angular_source,
                                     self.mass_source)

    def _write_rows(self, jac, neg_res, rhs):
        self._fg.tpsa_thm_balance_rows(self.A, jac, neg_res, rhs, self._missing)

    def _discretize_fluxes(self) -> None:
        super()._discretize_fluxes()
        self.data[PARAMETERS][self.tk]["second_order_tensor"] = SecondOrderTensor(self.conductivity)
        Mpfa(self.tk).discretize(self.sd, self.data)

    def _balance_pattern(self, k):
        """The union of the Darcy and Fourier div @ flux patterns."""
        return k.div.matmul(k.flux) + k.div.matmul(k.fourier)

    def _operands(self):
        if self._const is None:
            csr, dev = ad.as_device_csr, ad.device_vector
            k = super()._operands()
            Fo = self.data[DISCRETIZATION_MATRICES][self.tk]
            k.fourier = csr(Fo["flux"])
            k.fo_b = csr(Fo["bound_flux"]) @ dev(self.fourier_bc)
            k.bce = dev(self.ef_values)
            k.a_beta = dev((self.alpha - self.phi_ref) * self.so.thermal_expansion)
        return self._const

    def _porosity(self, pt, p, t, k):
        """phi(p_t, p, T) for tensors or ``DeviceAdArray`` operands."""
        return super()._porosity(pt, p, k) - (t - self.fl.reference_temperature) * k.a_beta

    def update_upwind(self, p) -> None:
        k = self._operands()
        q = ((k.flux @ ad.device_vector(p)) + k.q_b).cpu().numpy()
        rediscretize_upwind(self.sd, self.data, self.mobility_keyword, q, self.bc_fluid_flux)
        rediscretize_upwind(self.sd, self.data, self.enthalpy_upwind_keyword, q, self.bc_enthalpy_flux)

    def balance_equations(self, x, x_prev, dt: float) -> list:
        """[mass, energy] balance as ``DeviceAdArray`` in the variables [p_t | p | T] at the iterate ``x``."""
        k = self._operands()
        pt, p, t = ad.variables(list(self._fields(x)))
        ptn, pn, tn = self._fields(x_prev)
        DM = self.data[DISCRETIZATION_MATRICES]
        fl = self.fl
        phi, phi_n = self._porosity(pt, p, t, k), self._porosity(ptn, pn, tn, k)
        rho, rho_n = self._density(p, t), self._density(pn, tn)
        q = (k.flux @ p) + k.q_b
        w = rho * (1.0 / fl.viscosity)
        ff = advective_flux(DM[self.mobility_keyword], q, w, k.bcw, k.bcw)
        mass = (rho * phi * k.vol - rho_n * phi_n * k.vol) * (1.0 / dt) + (k.div @ ff) - k.src
        fe = advective_flux(DM[self.enthalpy_upwind_keyword], q, w * (t - fl.reference_temperature) * fl.heat_capacity,
                            k.bce, k.bce)
        fo = (k.fourier @ t) + k.fo_b
        energy = (self._energy(p, t, phi) - self._energy(pn, tn, phi_n)) * (k.vol * (1.0 / dt)) + (k.div @ (fe + fo))
        return [mass, energy]

    def balance_rows(self, x, x_prev, dt: float):
        """(field-ordered Jacobian [mass | energy] x [p_t | p | T], -R) of the balance rows at the iterate ``x``."""
        return ad.assemble(self.balance_equations(x, x_prev, dt))

    def fluid_equation(self, x, x_prev, dt: float):
        """The fluid mass balance as a ``DeviceAdArray`` in the variables [p_t | p | T] at the iterate ``x``."""
        return self.balance_equations(x, x_prev, dt)[0]
