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

import numpy as np
import scipy.sparse as sps

from . import ad, fv, krylov
from .advection import advective_flux, rediscretize_upwind
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES, PARAMETERS


class TpsaPoromechanics:
    """``data``: PorePy-style dictionary with ``parameters[flow_keyword]`` (``second_order_tensor``, ``bc``) and
    ``parameters[mechanics_keyword]`` (``fourth_order_tensor`` with ``mu`` / ``lmbda``, the ``bc`` of ``pp.Tpsa``).
    ``fluid``: ``compressibility, density, viscosity, reference_pressure``; ``solid``: ``reference_porosity,
    biot_coefficient, bulk_modulus``.  Face data: ``flow_bc_values`` (pressure on Dirichlet faces, flux elsewhere),
    ``mech_bc_values`` (the combined mechanical boundary operator, nd per face, face-major), ``bc_fluid_flux`` +
    ``fluid_flux_values`` (the boundary operator of the advective flux).  Cell data, integrated over the cells (None:
    zero): ``body_force`` (nd per cell), ``angular_source`` (nr), ``mass_source`` (solid mass), ``fluid_source``."""

    mobility_keyword = "mobility"
    # the FaceGrid entry points of this system and what its balance rows are called in errors
    _fg_system, _fg_rhs, _fg_rows = "tpsa_poro_system", "tpsa_poro_rhs", "tpsa_poro_fluid_rows"
    _rows_name = "fluid Jacobian entries outside the TPSA poromechanics row pattern"

    def __init__(self, sd, data: dict, fluid: dict, solid: dict, flow_bc_values, mech_bc_values, bc_fluid_flux,
                 fluid_flux_values, body_force=None, angular_source=None, mass_source=None, fluid_source=None,
                 flow_keyword: str = "flow", mechanics_keyword: str = "mechanics") -> None:
        self.nd = int(sd.dim)
        if self.nd not in (2, 3):
            raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")
        self.sd, self.data = sd, data
        self.fk, self.mk = flow_keyword, mechanics_keyword
        self.nr = 3 if self.nd == 3 else 1
        self.block_size = self.nd + self.nr + 2
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
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
        nc, nf, nd = self.nc, self.nf, self.nd
        self.flow_bc = self._vector(flow_bc_values, nf, "flow_bc_values")
        self.mech_bc = self._vector(mech_bc_values, nd * nf, "mech_bc_values")
        self.bc_fluid_flux = bc_fluid_flux
        self.ff_values = self._vector(fluid_flux_values, nf, "fluid_flux_values")
        self.body_force = self._vector(body_force, nd * nc, "body_force")
        self.angular_source = self._vector(angular_source, self.nr * nc, "angular_source")
        self.mass_source = self._vector(mass_source, nc, "mass_source")
        self.fluid_source = self._vector(fluid_source, nc, "fluid_source")
        if self.fluid_source is None:
            self.fluid_source = np.zeros(nc)
        self.column_map = None
        self.row_map = None
        self.A = None
        self._fg = None
        self._const = None
        self.last_timing: dict = {}

    @staticmethod
    def _vector(v, n: int, name: str):
        if v is None:
            return None
        v = np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
        if v.size != n:
            raise ValueError(f"{name} must have {n} values, got {v.size}")
        return v

    @property
    def num_dofs(self) -> int:
        return self.block_size * self.nc

    def discretize(self) -> None:
        """MPFA of the flow, the TPSA face terms and the mechanics rows of the Jacobian (device), the fluid-row pattern
        from div @ flux, and -R(0) of the mechanics rows."""
        import time
        sd, nd = self.sd, self.nd
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        params = self.data[PARAMETERS][self.mk]
        C = params["fourth_order_tensor"]
        codes, robin = fv.tpsa_bc_arrays(params["bc"], nd, self.nf)
        if nd == 2 and np.any(np.abs(sd.face_normals[2]) > np.maximum(np.abs(sd.face_normals[0]),
                                                                       np.abs(sd.face_normals[1]))):
            raise IndexError("Tpsa: a face normal of a 2d grid points mostly out of the xy-plane")
        flags = np.zeros(self.nf, np.uint8)
        flags[np.asarray(sd.get_all_boundary_faces(), dtype=np.int64)] = 1
        t0 = time.perf_counter()
        self._discretize_fluxes()
        t1 = time.perf_counter()
        self._const = None
        k = self._operands()
        if self._fg is None:
            self._fg = fv.FaceGrid.for_grid(sd)
        self.lmbda = np.asarray(C.lmbda, float)
        self.A, stage_ms = getattr(self._fg, self._fg_system)(nd, C.mu, self.lmbda, self.alpha, sd.cell_volumes, codes,
                                                              robin, flags, sd.face_areas, self._balance_pattern(k))
        self.b0 = getattr(self._fg, self._fg_rhs)(self.num_dofs, self.mech_bc, self.body_force, self.angular_source,
                                                  self.mass_source)
        self.last_timing = dict(mpfa_s=t1 - t0, face_terms_ms=stage_ms[0], rows_ms=stage_ms[1],
                                total_s=time.perf_counter() - t0)

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
            lam = np.asarray(self.data[PARAMETERS][self.mk]["fourth_order_tensor"].lmbda, float)
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
        """(p_t, p) of a cell-interleaved vector, as contiguous device vectors (the scalar fields after r_c)."""
        x = ad.device_vector(x).reshape(self.nc, self.block_size)
        return tuple(x[:, j].contiguous() for j in range(self.nd + self.nr, self.block_size))

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

    def linearize(self, x, x_prev, dt: float):
        """(J as ``DeviceCsr``, -R as a CUDA tensor) in the cell-interleaved order: upwind directions from ``x``, the
        fluid rows from the AD chain written into the fixed pattern, -R of the mechanics rows = b0 - A x.  ``J`` is
        the problem's own matrix, overwritten by the next call."""
        import torch
        if self.A is None:
            self.discretize()
        x = ad.device_vector(x)
        if x.numel() != self.num_dofs:
            raise ValueError(f"x must have {self.num_dofs} values")
        self.update_upwind(self._fields(x)[1])
        jac, neg_res = self.balance_rows(x, x_prev, dt)
        rhs = self.b0 - (self.A @ x)
        if getattr(self, "_missing", None) is None:
            self._missing = torch.zeros(1, dtype=torch.int32, device=rhs.device)
        getattr(self._fg, self._fg_rows)(self.A, jac, neg_res, rhs, self._missing)
        return self.A, rhs

    def time_step(self, x_prev, dt: float, tol: float = 1e-10, max_iterations: int = 15, linear_tol: float = 1e-10,
                  linear_solver=None, verbose: bool = False):
        """One implicit time step by Newton's method.  ``linear_solver(J, rhs) -> dx`` overrides the device
        block-Jacobi BiCGStab (one inverted cell block per cell).  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)

        def linearize(x):
            J, rhs = self.linearize(x, x_prev, dt)
            if int(self._missing.sum()):
                raise RuntimeError(self._rows_name)
            return J, rhs
        if linear_solver is None:
            linear_solver = krylov.bicgstab_solver(linear_tol, block_size=self.block_size)
        return newton_loop(linearize, x_prev, linear_solver, tol, max_iterations, verbose)

    def to_model_order(self, A, b=None):
        """A (scipy) and b permuted to the rows / columns of the model's ``EquationSystem``."""
        if self.column_map is None or self.row_map is None:
            raise ValueError("no dof maps: build the problem with model_bridge.tpsa_poromechanics_from_model")
        n = self.num_dofs
        P = sps.csr_matrix((np.ones(n), (self.row_map, np.arange(n))), shape=(n, n))
        Q = sps.csr_matrix((np.ones(n), (np.arange(n), self.column_map)), shape=(n, n))
        Am = (P @ sps.csr_matrix(A) @ Q).tocsr()
        if b is None:
            return Am
        bm = np.empty(n)
        bm[self.row_map] = np.asarray(b)
        return Am, bm


def interleave(blocks, nd: int, nr: int, nc: int) -> np.ndarray:
    """Cell-interleaved order [u_c, r_c, p_t_c, p_c] (or [u_c, r_c, p_t_c, p_c, T_c]) from the field-wise index arrays."""
    u, r, *scalars = (np.asarray(x, np.int64) for x in blocks)
    out = np.empty((nc, nd + nr + len(scalars)), np.int64)
    out[:, :nd] = u.reshape(nc, nd)
    out[:, nd:nd + nr] = r.reshape(nc, nr)
    for j, v in enumerate(scalars):
        out[:, nd + nr + j] = v
    return out.reshape(-1)
