"""Biot poromechanics, the reference's model equations on the device AD chain -- BASELINE config[3] ("Biot poromechanics,
coupled MPFA + MPSA"): mass and momentum balance of ``pp.Poromechanics`` on a 2-D or 3-D subdomain (``nd = sd.dim``),
every term taken from the device-resident outputs of ``porepy_b200.Mpfa`` and ``porepy_b200.Biot``, value and Jacobian by
``DeviceAdArray``.

* ``momentum_balance_equation``   -div_nd (stress u + bound_stress u_b + scalar_gradient (p - p_ref)) - f = 0
                                  models/momentum_balance.py, ``pressure_stress`` constitutive_laws.py
* poromechanical porosity         phi = phi_ref + N^-1 (p - p_ref) + (displacement_divergence u + boundary_displacement_divergence u_b
                                  + mpsa_consistency (p - p_ref)) / vol             constitutive_laws.py:4536-4720
* ``fluid_mass``                  vol rho(p) phi(u, p),   rho = rho0 exp(c (p - p_ref))   fluid_mass_balance.py:167-190
* ``fluid_flux``                  q (U rho/mu) + B_dir (q w_b) + B_neu w_b,   q = flux p + bound_flux p_b
                                  constitutive_laws.py:2521-2569
* ``mass_balance_equation``       (mass - mass_n) / dt + div fluid_flux - source = 0

Unknowns and equations in the order of the reference's ``EquationSystem`` (``unknown_layout``, ``equation_layout``;
displacements cell-major, nd per cell).  ``pb.Upwind`` is re-discretized from the iterate's Darcy flux in front of every
linearization (models/solution_strategy.py:433-441).  The Newton update is solved by the fused Jacobi-BiCGStab
(csrc/krylov.cu) on the coupled Jacobian.  ``tests/golden/poromech_model.npz`` pins Jacobian, residual, residual history
and converged state to the unmodified reference (tools/make_poromech_golden.py), ``poromech_model_2d.npz`` the same in 2-D.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps

from . import ad, krylov
from .advection import advective_flux, rediscretize_upwind
from .contact import matrix_dimension
from .fv import Biot, Mpfa
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES


class Poromechanics(LayoutModel):
    """``data``: PorePy-style dictionary with ``parameters[flow_keyword]`` (``second_order_tensor``, ``bc``) and
    ``parameters[mechanics_keyword]`` (``fourth_order_tensor``, vectorial ``bc``, ``scalar_vector_mappings`` =
    {flow_keyword: Biot coefficient or tensor}).  ``fluid``: ``compressibility, density, viscosity, reference_pressure``;
    ``solid``: ``reference_porosity, n_inv`` (= (alpha - phi_ref)(1 - alpha) / K_bulk).  Face data: ``flow_bc_values``
    (pressure on Dirichlet faces, flux elsewhere), ``mech_bc_values`` (nd nf, face-major: displacement / traction),
    ``bc_fluid_flux`` + ``fluid_flux_values`` (the boundary operator of the advective flux)."""

    mobility_keyword = "mobility"

    def __init__(self, sd, data: dict, fluid: dict, solid: dict, flow_bc_values, mech_bc_values, bc_fluid_flux,
                 fluid_flux_values, source=None, body_force=None, flow_keyword: str = "flow",
                 mechanics_keyword: str = "mechanics"):
        self.nd = matrix_dimension(sd)
        self.sd, self.data = sd, data
        self.fk, self.mk = flow_keyword, mechanics_keyword
        self.c, self.rho0, self.mu = (float(fluid[k]) for k in ("compressibility", "density", "viscosity"))
        self.p_ref = float(fluid.get("reference_pressure", 0.0))
        self.phi_ref, self.n_inv = float(solid["reference_porosity"]), float(solid["n_inv"])
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        self.flow_bc = np.asarray(flow_bc_values, float)
        self.mech_bc = np.asarray(mech_bc_values, float)
        self.bc_fluid_flux = bc_fluid_flux
        self.ff_values = np.asarray(fluid_flux_values, float)
        self.source = np.zeros(self.nc) if source is None else np.asarray(source, float)
        self.body_force = np.zeros(self.nd * self.nc) if body_force is None else np.asarray(body_force, float)
        scalar, vector = [(("matrix",), self.nc, 1)], [(("matrix",), self.nc, self.nd)]
        self.unknown_layout = BlockLayout([("pressure", scalar), ("displacement", vector)])
        self.equation_layout = BlockLayout([("mass_balance_equation", scalar), ("momentum_balance_equation", vector)])
        self._const = None

    def discretize(self) -> None:
        Mpfa(self.fk).discretize(self.sd, self.data)
        Biot(self.mk).discretize(self.sd, self.data)
        self._const = None

    def _coupling(self, key):
        m = self.data[DISCRETIZATION_MATRICES][self.mk][key]
        return m[self.fk] if isinstance(m, dict) else m

    def _operands(self):
        if self._const is None:
            from types import SimpleNamespace
            csr, dev = ad.as_device_csr, ad.device_vector
            F = self.data[DISCRETIZATION_MATRICES][self.fk]
            M = self.data[DISCRETIZATION_MATRICES][self.mk]
            vol = np.asarray(self.sd.cell_volumes, float)
            k = SimpleNamespace(
                div=csr(sps.csr_matrix(self.sd.cell_faces.T)),
                div_nd=csr(sps.kron(sps.csr_matrix(self.sd.cell_faces.T), sps.identity(self.nd)).tocsr()),
                flux=csr(F["flux"]), stress=csr(M["stress"]), grad_p=csr(self._coupling("scalar_gradient")),
                div_u=csr(self._coupling("displacement_divergence")), cons=csr(self._coupling("mpsa_consistency")),
                vol=dev(vol), inv_vol=dev(1.0 / vol), bcw=dev(self.ff_values), src=dev(self.source), f=dev(self.body_force))
            # boundary data enter through constant vectors: one SpMV each, once
            k.q_b = csr(F["bound_flux"]) @ dev(self.flow_bc)
            k.stress_b = csr(M["bound_stress"]) @ dev(self.mech_bc)
            k.div_u_b = csr(self._coupling("boundary_displacement_divergence")) @ dev(self.mech_bc)
            self._const = k
        return self._const

    def _density(self, p):
        return ((p - self.p_ref) * self.c).exp() * self.rho0

    def _porosity(self, p, u, k):
        """phi(u, p) for tensors or ``DeviceAdArray`` operands (constitutive_laws.py:4536-4560)."""
        dp = p - self.p_ref
        return ((k.div_u @ u) + (k.cons @ dp) + k.div_u_b) * k.inv_vol + dp * self.n_inv + self.phi_ref

    def update_upwind(self, x) -> None:
        x = ad.device_vector(x)
        k = self._operands()
        q = (k.flux @ self.unknown_layout.parts(x)["pressure"][0]) + k.q_b
        rediscretize_upwind(self.sd, self.data, self.mobility_keyword, q.cpu().numpy(), self.bc_fluid_flux)

    def equations(self, x, x_prev, dt: float) -> list:
        """[mass balance, momentum balance] as ``DeviceAdArray`` at the iterate ``x``."""
        k = self._operands()
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var, prev = self.unknown_layout.variables(x), self.unknown_layout.parts(x_prev)
        (p,), (u,) = var["pressure"], var["displacement"]
        (pn,), (un,) = prev["pressure"], prev["displacement"]
        T = self.data[DISCRETIZATION_MATRICES][self.mobility_keyword]
        mass = self._density(p) * self._porosity(p, u, k) * k.vol
        mass_n = self._density(pn) * self._porosity(pn, un, k) * k.vol
        q = (k.flux @ p) + k.q_b
        w = self._density(p) * (1.0 / self.mu)
        ff = advective_flux(T, q, w, k.bcw, k.bcw)
        mass_eq = (mass - mass_n) * (1.0 / dt) + (k.div @ ff) - k.src
        stress = (k.stress @ u) + (k.grad_p @ (p - self.p_ref)) + k.stress_b
        momentum_eq = -(k.div_nd @ stress) - k.f
        return self.equation_layout.stack({"mass_balance_equation": [mass_eq],
                                           "momentum_balance_equation": [momentum_eq]})

    def linearize(self, x, x_prev, dt: float):
        """(J as ``DeviceCsr``, -R as a CUDA tensor): upwind directions from ``x``, then the AD evaluation."""
        self.update_upwind(x)
        return ad.assemble(self.equations(x, x_prev, dt))

    def time_step(self, x_prev, dt: float, tol: float = 1e-10, max_iterations: int = 15, linear_tol: float = 1e-10,
                  linear_solver=None, verbose: bool = False):
        """One implicit time step by Newton's method.  ``linear_solver(J, rhs) -> dx`` overrides the device Krylov solve
        (the CPU tests pass a direct solve for the scipy stand-in).  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        solver = krylov.bicgstab_solver(linear_tol) if linear_solver is None else linear_solver
        return newton_loop(lambda x: self.linearize(x, x_prev, dt), x_prev, solver, tol, max_iterations, verbose)
