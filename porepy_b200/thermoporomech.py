"""Thermo-poromechanics, the reference's model equations on the device AD chain -- BASELINE config[4] ("thermo-
poromechanics ..., full Newton loop") on a 2-D or 3-D subdomain (``nd = sd.dim``) without fractures: momentum, mass and
energy balance of ``pp.Thermoporomechanics``, every term from the device-resident outputs of ``porepy_b200.Mpfa`` (Darcy
and Fourier) and ``porepy_b200.Biot`` (two coupling tensors: Biot's and the thermal stress), value and Jacobian by
``DeviceAdArray``.

* density                  rho = rho0 exp(c (p - p0) - beta_f (T - T0))                    fluid_property_library.py
* porosity                 poromechanical porosity of ``porepy_b200.poromech`` - (alpha - phi0) beta_s (T - T0)
                           constitutive_laws.py:4799-4839
* stress                   + scalar_gradient[thermal] (T - T0)   (``thermal_stress``)       constitutive_laws.py:3569-3591
* internal energy          (rho c_f (T - T0) - p) phi + rho_s c_s (T - T0) (1 - phi)        energy_balance.py:184-234
* energy flux              Fourier (MPFA with the conductivity phi k_f + (1 - phi) k_s, constitutive_laws.py:2120-2150:
                           discretized once at the reference porosity -- the reference's default adds no nonlinear Fourier
                           discretization, energy_balance.py:1227-1242; ``rediscretize_fourier=True`` follows the iterate's
                           porosity instead, the opt-in of that hook) + upwinded enthalpy flux with weight
                           c_f (T - T0) rho / mu                                            energy_balance.py:236-352
* balance equations        momentum: -div_nd stress - f;  mass / energy: d/dt (vol x) + div flux - source

Unknowns and equations in the order of the reference's ``EquationSystem`` (``unknown_layout``, ``equation_layout``).
``tests/golden/thm_model.npz`` pins Jacobian, residual, residual history and converged state to the
unmodified reference (tools/make_thm_golden.py), ``thm_model_2d.npz`` the same in 2-D.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps

from . import ad, krylov
from .advection import advective_flux, rediscretize_upwind
from .contact import matrix_dimension
from .fv import Biot, Mpfa
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES, PARAMETERS, SecondOrderTensor


class Thermoporomechanics(LayoutModel):
    """``data``: ``parameters[flow_keyword]`` (``second_order_tensor``, ``bc``), ``parameters[fourier_keyword]`` (``bc``; the
    conductivity tensor is written here by ``discretize``), ``parameters[mechanics_keyword]`` (``fourth_order_tensor``,
    vectorial ``bc``, ``scalar_vector_mappings`` = {flow_keyword: Biot tensor, thermal_keyword: thermal-stress tensor}).
    ``fluid``: ``compressibility, density, viscosity, thermal_expansion, heat_capacity, conductivity, reference_pressure,
    reference_temperature``; ``solid``: ``reference_porosity, n_inv, biot_coefficient, thermal_expansion, heat_capacity,
    conductivity, density``.  ``bc``: face arrays ``flow``, ``fourier``, ``mechanics`` (nd nf), ``fluid_flux``,
    ``enthalpy_flux`` and the boundary-condition objects ``fluid_flux_type``, ``enthalpy_flux_type`` of the two upwind
    discretizations."""

    mobility_keyword = "mobility"
    enthalpy_upwind_keyword = "enthalpy_upwind"

    def __init__(self, sd, data: dict, fluid: dict, solid: dict, bc: dict, flow_keyword: str = "flow",
                 fourier_keyword: str = "fourier", mechanics_keyword: str = "mechanics", thermal_keyword: str = "thermal",
                 rediscretize_fourier: bool = False):
        self.nd = matrix_dimension(sd)
        self.sd, self.data = sd, data
        self.fk, self.tk, self.mk, self.ck = flow_keyword, fourier_keyword, mechanics_keyword, thermal_keyword
        self.fl = SimpleNamespace(**{k: float(v) for k, v in fluid.items()})
        self.so = SimpleNamespace(**{k: float(v) for k, v in solid.items()})
        self.bc = bc
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        self.rediscretize_fourier = bool(rediscretize_fourier)
        scalar, vector = [(("matrix",), self.nc, 1)], [(("matrix",), self.nc, self.nd)]
        self.unknown_layout = BlockLayout([("displacement", vector), ("pressure", scalar), ("temperature", scalar)])
        self.equation_layout = BlockLayout([("momentum_balance_equation", vector), ("mass_balance_equation", scalar),
                                            ("energy_balance_equation", scalar)])
        self._const = None

    def _discretize_fourier(self, phi) -> None:
        self.data[PARAMETERS][self.tk]["second_order_tensor"] = SecondOrderTensor(
            phi * self.fl.conductivity + (1.0 - phi) * self.so.conductivity)
        Mpfa(self.tk).discretize(self.sd, self.data)

    def discretize(self) -> None:
        """Darcy flux, the Biot / thermal-stress terms and the Fourier flux at the reference porosity; the upwinding
        follows the iterate (``update_discretizations``)."""
        Mpfa(self.fk).discretize(self.sd, self.data)
        Biot(self.mk).discretize(self.sd, self.data)
        self._discretize_fourier(np.full(self.nc, self.so.reference_porosity))
        self._const = None

    def _operands(self):
        if self._const is None:
            csr, dev = ad.as_device_csr, ad.device_vector
            F = self.data[DISCRETIZATION_MATRICES][self.fk]
            M = self.data[DISCRETIZATION_MATRICES][self.mk]
            vol = np.asarray(self.sd.cell_volumes, float)
            k = SimpleNamespace(
                div=csr(sps.csr_matrix(self.sd.cell_faces.T)),
                div_nd=csr(sps.kron(sps.csr_matrix(self.sd.cell_faces.T), sps.identity(self.nd)).tocsr()),
                flux=csr(F["flux"]), stress=csr(M["stress"]), grad_p=csr(M["scalar_gradient"][self.fk]),
                grad_t=csr(M["scalar_gradient"][self.ck]), div_u=csr(M["displacement_divergence"][self.fk]),
                cons=csr(M["mpsa_consistency"][self.fk]), vol=dev(vol), inv_vol=dev(1.0 / vol),
                bcw=dev(self.bc["fluid_flux"]), bce=dev(self.bc["enthalpy_flux"]), bct=dev(self.bc["fourier"]))
            k.q_b = csr(F["bound_flux"]) @ dev(self.bc["flow"])
            k.stress_b = csr(M["bound_stress"]) @ dev(self.bc["mechanics"])
            k.div_u_b = csr(M["boundary_displacement_divergence"][self.fk]) @ dev(self.bc["mechanics"])
            self._const = k
        return self._const

    # ---- constitutive laws on tensors or DeviceAdArrays
    def _density(self, p, t):
        return ((p - self.fl.reference_pressure) * self.fl.compressibility
                - (t - self.fl.reference_temperature) * self.fl.thermal_expansion).exp() * self.fl.density

    def _porosity(self, u, p, t, k):
        dp, dtm = p - self.fl.reference_pressure, t - self.fl.reference_temperature
        so = self.so
        return (((k.div_u @ u) + (k.cons @ dp) + k.div_u_b) * k.inv_vol + dp * so.n_inv
                - dtm * ((so.biot_coefficient - so.reference_porosity) * so.thermal_expansion) + so.reference_porosity)

    def _energy(self, p, t, phi):
        dtm = t - self.fl.reference_temperature
        fluid = (self._density(p, t) * dtm * self.fl.heat_capacity - p) * phi
        solid = (dtm * (self.so.density * self.so.heat_capacity)) * (-phi + 1.0)
        return fluid + solid

    # ---- what follows the iterate: upwind directions (and, by request, the porosity-weighted conductivity)
    def update_discretizations(self, x) -> None:
        x = ad.device_vector(x)
        k = self._operands()
        parts = self.unknown_layout.parts(x)
        (u,), (p,), (t,) = parts["displacement"], parts["pressure"], parts["temperature"]
        q = ((k.flux @ p) + k.q_b).cpu().numpy()
        for kw, bc in ((self.mobility_keyword, self.bc["fluid_flux_type"]),
                       (self.enthalpy_upwind_keyword, self.bc["enthalpy_flux_type"])):
            rediscretize_upwind(self.sd, self.data, kw, q, bc)
        if self.rediscretize_fourier:
            self._discretize_fourier(self._porosity(u, p, t, k).cpu().numpy())

    def equations(self, x, x_prev, dt: float) -> list:
        """[momentum, mass, energy] balance as ``DeviceAdArray`` at the iterate ``x``."""
        k = self._operands()
        csr = ad.as_device_csr
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var, prev = self.unknown_layout.variables(x), self.unknown_layout.parts(x_prev)
        (u,), (p,), (t,) = var["displacement"], var["pressure"], var["temperature"]
        (un,), (pn,), (tn,) = prev["displacement"], prev["pressure"], prev["temperature"]
        DM = self.data[DISCRETIZATION_MATRICES]
        Tm, Te, Fo = DM[self.mobility_keyword], DM[self.enthalpy_upwind_keyword], DM[self.tk]
        fl = self.fl
        phi, phi_n = self._porosity(u, p, t, k), self._porosity(un, pn, tn, k)
        rho, rho_n = self._density(p, t), self._density(pn, tn)
        stress = (k.stress @ u) + (k.grad_p @ (p - fl.reference_pressure)) + (k.grad_t @ (t - fl.reference_temperature)) \
            + k.stress_b
        momentum = -(k.div_nd @ stress)
        q = (k.flux @ p) + k.q_b
        w = rho * (1.0 / fl.viscosity)
        ff = advective_flux(Tm, q, w, k.bcw, k.bcw)
        mass = (rho * phi - rho_n * phi_n) * (k.vol * (1.0 / dt)) + (k.div @ ff)
        we = w * (t - fl.reference_temperature) * fl.heat_capacity
        fe = advective_flux(Te, q, we, k.bce, k.bce)
        fo = (csr(Fo["flux"]) @ t) + (csr(Fo["bound_flux"]) @ k.bct)
        energy = (self._energy(p, t, phi) - self._energy(pn, tn, phi_n)) * (k.vol * (1.0 / dt)) + (k.div @ (fe + fo))
        return self.equation_layout.stack({"momentum_balance_equation": [momentum], "mass_balance_equation": [mass],
                                           "energy_balance_equation": [energy]})

    def linearize(self, x, x_prev, dt: float):
        """(J as ``DeviceCsr``, -R as a CUDA tensor) at the iterate ``x``."""
        self.update_discretizations(x)
        return ad.assemble(self.equations(x, x_prev, dt))

    def time_step(self, x_prev, dt: float, tol: float = 1e-10, max_iterations: int = 20, linear_tol: float = 1e-10,
                  linear_solver=None, verbose: bool = False):
        """One implicit time step by Newton's method; ``linear_solver(J, rhs) -> dx`` overrides the device Krylov solve
        (fused Jacobi-BiCGStab, csrc/krylov.cu).  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        solver = krylov.bicgstab_solver(linear_tol) if linear_solver is None else linear_solver
        return newton_loop(lambda x: self.linearize(x, x_prev, dt), x_prev, solver, tol, max_iterations, verbose)
