"""TPSA poromechanics on the device: the reference's ``pp.Poromechanics`` with ``TpsaPoromechanicsMixin``
(models/poromechanics.py:92-136, 177-213; constitutive_laws.py:3299-3374, 4536-4610) on one 2-D or 3-D grid without
fractures.

Unknowns and equations per cell, cell by cell: the displacement u (nd), the rotation stress r (nr), the total pressure
p_t and the fluid pressure p, ``[u_c, r_c, p_t_c, p_c]``; the diagonal blocks of the Jacobian are the (nd + nr + 2)^2
cell blocks (5 x 5 in 2-D, 8 x 8 in 3-D).

* momentum, angular momentum     as in ``TpsaElasticity`` (the TPSA stress has no pressure term)
* solid mass                     the TPSA row - vol alpha / lambda p                       poromechanics.py:107-136
* porosity                       phi = phi_ref + N^-1 (p - p_ref) + alpha / lambda (p_t + alpha p),
                                 N^-1 = (alpha - phi_ref)(1 - alpha) / K      constitutive_laws.py:3345-3374, 4582-4610
* fluid mass                     vol rho(p) phi,  rho = rho0 exp(c (p - p_ref))
* fluid mass balance             (mass - mass_n) / dt + div (q (U rho / mu_f) + B_dir (q w_b) + B_neu w_b) - source,
                                 q = flux p + bound_flux p_b (MPFA)

The mechanics rows are linear and constant: ``pb_tpsa_poro_system`` writes them once per ``discretize`` into a row
pattern built on the device.  At every linearization the fluid mass balance is evaluated on the device AD chain with
the variables [p_t | p], and ``pb_tpsa_poro_fluid_rows`` writes its Jacobian rows into the fixed pattern (no
permutation product, nothing copied to the host); -R of the mechanics rows is b0 - A x.  ``pb.Upwind`` is re-discretized
from the iterate's Darcy flux in front of every linearization (models/solution_strategy.py:433-441).
"""
from __future__ import annotations

import time

import numpy as np
import scipy.sparse as sps

from . import ad, krylov
from .advection import advective_flux, rediscretize_upwind
from .params import DISCRETIZATION_MATRICES, PARAMETERS
from .tpsa_elasticity import TpsaNewtonProblem


class TpsaPoromechanics(TpsaNewtonProblem):
    """``data``: PorePy-style dictionary with ``parameters[flow_keyword]`` (``second_order_tensor``, ``bc``) and
    ``parameters[mechanics_keyword]`` (``fourth_order_tensor`` with ``mu`` / ``lmbda``, the ``bc`` of ``pp.Tpsa``).
    ``fluid``: ``compressibility, density, viscosity, reference_pressure``; ``solid``: ``reference_porosity,
    biot_coefficient, bulk_modulus``.  Face data: ``flow_bc_values`` (pressure on Dirichlet faces, flux elsewhere),
    ``mech_bc_values`` (the combined mechanical boundary operator, nd per face, face-major), ``bc_fluid_flux`` +
    ``fluid_flux_values`` (the boundary operator of the advective flux).  Cell data, integrated over the cells (None:
    zero): ``body_force`` (nd per cell), ``angular_source`` (nr), ``mass_source`` (solid mass), ``fluid_source``."""

    mobility_keyword = "mobility"
    scalar_fields = ("total_pressure", "pressure")
    scalar_balances = ("solid_mass_equation", "mass_balance_equation")
    bridge = "tpsa_poromechanics_from_model"
    outside_pattern = "fluid Jacobian entries outside the TPSA poromechanics row pattern"

    def __init__(self, sd, data: dict, fluid: dict, solid: dict, flow_bc_values, mech_bc_values, bc_fluid_flux,
                 fluid_flux_values, body_force=None, angular_source=None, mass_source=None, fluid_source=None,
                 flow_keyword: str = "flow", mechanics_keyword: str = "mechanics") -> None:
        super().__init__(sd, data, mechanics_keyword, mech_bc_values, body_force, angular_source, mass_source,
                         bc_name="mech_bc_values")
        self.fk = flow_keyword
        self.c, self.rho0, self.mu_f = (float(fluid[k]) for k in ("compressibility", "density", "viscosity"))
        self.p_ref = float(fluid.get("reference_pressure", 0.0))
        if not all(np.isfinite(v) and v > 0 for v in (self.c, self.rho0, self.mu_f)):
            raise ValueError("fluid compressibility, density and viscosity must be finite and > 0")
        self.phi_ref = float(solid["reference_porosity"])
        alpha = np.broadcast_to(np.asarray(solid["biot_coefficient"], float), (self.nc,))
        if not np.all(np.isfinite(alpha)):
            raise ValueError("Biot coefficient alpha must be finite")
        self.alpha = np.ascontiguousarray(alpha)
        self.n_inv = (self.alpha - self.phi_ref) * (1.0 - self.alpha) / float(solid["bulk_modulus"])
        nc, nf = self.nc, self.nf
        self.flow_bc = self._vector(flow_bc_values, nf, "flow_bc_values")
        self.bc_fluid_flux = bc_fluid_flux
        self.ff_values = self._vector(fluid_flux_values, nf, "fluid_flux_values")
        self.fluid_source = self._vector(fluid_source, nc, "fluid_source")
        if self.fluid_source is None:
            self.fluid_source = np.zeros(nc)
        self._const = None

    @property
    def mech_bc(self):
        """``mech_bc_values``: the combined mechanical boundary operator."""
        return self.bc_values

    def _system(self, C, codes, robin, flags):
        """MPFA of the flow, then the TPSA face terms and the mechanics rows of the Jacobian (device) with the
        balance-row pattern from div @ flux."""
        t0 = time.perf_counter()
        self._discretize_fluxes()
        self.last_timing["mpfa_s"] = time.perf_counter() - t0
        self._const = None
        self.lmbda = np.asarray(C.lmbda, float)
        return self._mechanics_rows(C.mu, codes, robin, flags, self._balance_pattern(self._operands()))

    def _mechanics_rows(self, mu, codes, robin, flags, pattern):
        return self._fg.tpsa_poro_system(self.nd, mu, self.lmbda, self.alpha, self.sd.cell_volumes, codes, robin,
                                         flags, self.sd.face_areas, pattern)

    def _rhs(self):
        return self._fg.tpsa_poro_rhs(self.num_dofs, self.bc_values, self.body_force, self.angular_source,
                                      self.mass_source)

    def _write_rows(self, jac, neg_res, rhs):
        self._fg.tpsa_poro_fluid_rows(self.A, jac, neg_res, rhs, self._missing)

    def _discretize_fluxes(self) -> None:
        from .fv import Mpfa
        Mpfa(self.fk).discretize(self.sd, self.data)

    def _balance_pattern(self, k):
        """The nc x nc pattern of the couplings of the balance rows to the other cells: div @ flux."""
        return k.div.matmul(k.flux)

    def _operands(self):
        if self._const is None:
            from types import SimpleNamespace
            csr, dev = ad.as_device_csr, ad.device_vector
            F = self.data[DISCRETIZATION_MATRICES][self.fk]
            vol = np.asarray(self.sd.cell_volumes, float)
            lam = np.asarray(self.data[PARAMETERS][self.keyword]["fourth_order_tensor"].lmbda, float)
            k = SimpleNamespace(div=csr(sps.csr_matrix(self.sd.cell_faces.T)), flux=csr(F["flux"]), vol=dev(vol),
                                bcw=dev(self.ff_values), src=dev(self.fluid_source), a_lam=dev(self.alpha / lam),
                                alpha=dev(self.alpha), n_inv=dev(self.n_inv))
            k.q_b = csr(F["bound_flux"]) @ dev(self.flow_bc)   # boundary data: one SpMV, once
            self._const = k
        return self._const

    def _density(self, p):
        return ((p - self.p_ref) * self.c).exp() * self.rho0

    def _porosity(self, pt, p, k):
        """phi(p_t, p) for tensors or ``DeviceAdArray`` operands (constitutive_laws.py:3345-3374, 4552-4610)."""
        return (p - self.p_ref) * k.n_inv + (pt + p * k.alpha) * k.a_lam + self.phi_ref

    def _fields(self, x):
        """The ``scalar_fields`` of a cell-interleaved vector (the unknowns behind r_c), as contiguous device
        vectors."""
        x = ad.device_vector(x).reshape(self.nc, self.block_size)
        return tuple(x[:, j].contiguous() for j in range(self.block_size - len(self.scalar_fields), self.block_size))

    def update_upwind(self, p) -> None:
        k = self._operands()
        q = (k.flux @ ad.device_vector(p)) + k.q_b
        rediscretize_upwind(self.sd, self.data, self.mobility_keyword, q.cpu().numpy(), self.bc_fluid_flux)

    def fluid_equation(self, x, x_prev, dt: float):
        """The fluid mass balance as a ``DeviceAdArray`` in the variables [p_t | p] at the iterate ``x``."""
        k = self._operands()
        pt, p = ad.variables(list(self._fields(x)))
        ptn, pn = self._fields(x_prev)
        T = self.data[DISCRETIZATION_MATRICES][self.mobility_keyword]
        mass = self._density(p) * self._porosity(pt, p, k) * k.vol
        mass_n = self._density(pn) * self._porosity(ptn, pn, k) * k.vol
        q = (k.flux @ p) + k.q_b
        w = self._density(p) * (1.0 / self.mu_f)
        ff = advective_flux(T, q, w, k.bcw, k.bcw)
        return (mass - mass_n) * (1.0 / dt) + (k.div @ ff) - k.src

    def balance_rows(self, x, x_prev, dt: float):
        """(field-ordered Jacobian, -R) of the balance rows at the iterate ``x``: here the fluid mass balance."""
        eq = self.fluid_equation(x, x_prev, dt)
        return eq.jac, -eq.val

    def _iterate_rows(self, x, x_prev, dt: float):
        """The rows ``linearize(x, x_prev, dt)`` writes: upwind directions from ``x``, then ``balance_rows``."""
        self.update_upwind(self._fields(x)[1])
        return self.balance_rows(x, x_prev, dt)

    def time_step(self, x_prev, dt: float, tol: float = 1e-10, max_iterations: int = 15, linear_tol: float = 1e-10,
                  linear_solver=None, verbose: bool = False):
        """One implicit time step by Newton's method.  ``linear_solver(J, rhs) -> dx`` overrides the device
        block-Jacobi BiCGStab (one inverted cell block per cell).  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        if linear_solver is None:
            linear_solver = krylov.bicgstab_solver(linear_tol, block_size=self.block_size)
        return self._newton(lambda x: self.linearize(x, x_prev, dt), x_prev, linear_solver, tol, max_iterations,
                            verbose)
