"""The TPSA three-field elasticity system on the device: the reference's ``pp.MomentumBalance`` with
``TpsaMomentumBalanceMixin`` (models/momentum_balance.py:82-106, 250-280, 344-368) on one grid without fractures,
assembled by ``pb_tpsa_system`` / ``pb_tpsa_rhs`` (csrc/tpsa_system.cuh) and solved by the fused block-Jacobi BiCGStab
of ``krylov``.

Unknowns per cell: the displacement u (nd), the rotation stress r (nr = 3 in 3-D, 1 in 2-D) and the total pressure p.
Unknowns and equations are numbered cell by cell, ``[u_c, r_c, p_c]``, so the diagonal blocks of ``A`` are the
(nd + nr + 1)^2 cell blocks the preconditioner inverts.  ``column_map`` / ``row_map`` (set by
``model_bridge.tpsa_momentum_from_model``) give the model's ``EquationSystem`` dof / row of each unknown / equation.

``TpsaProblem`` and ``TpsaNewtonProblem`` hold what the four TPSA problem classes share: every TPSA system contains
these three-field rows.
"""
from __future__ import annotations

import time

import numpy as np
import scipy.sparse as sps

from . import ad, fv
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import PARAMETERS


class TpsaProblem(LayoutModel):
    """The TPSA three-field rows on grid ``sd``: ``data[PARAMETERS][keyword]`` holds the ``fourth_order_tensor``
    (``mu``, ``lmbda``) and the ``bc`` of ``pp.Tpsa``; ``bc_values`` is the combined mechanical boundary operator (nd
    values per face, face-major, called ``bc_name`` in errors); ``body_force`` (nd per cell), ``angular_source`` (nr per
    cell) and ``mass_source`` (one per cell) are cell-major and already integrated over the cells (None: zero).

    The unknowns and balance equations of a cell are u (nd) and r (nr) with the momentum and angular momentum balances,
    then one of each per name in ``scalar_fields`` / ``scalar_balances``, numbered cell by cell: the first block of
    ``unknown_layout`` / ``equation_layout``.  ``unknowns`` / ``equations`` are the blocks behind it.  A subclass
    assembles its matrix through its own ``FaceGrid`` entry point in ``_system(C, codes, robin, flags)`` -> (A, the
    device times of the two stages in ms)."""

    scalar_fields = ("total_pressure",)
    scalar_balances = ("solid_mass_equation",)
    bridge = "tpsa_momentum_from_model"      # the ``model_bridge`` function that sets ``column_map`` / ``row_map``

    def __init__(self, sd, data: dict, keyword: str, bc_values, body_force, angular_source, mass_source,
                 bc_name: str = "bc_values", unknowns=(), equations=()) -> None:
        self.nd = nd = int(sd.dim)
        if nd not in (2, 3):
            raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")
        self.nr = 3 if nd == 3 else 1
        self.sd, self.data, self.keyword = sd, data, keyword
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        self.fields = [("displacement", nd), ("rotation_stress", self.nr)] + [(f, 1) for f in self.scalar_fields]
        self.balances = ([("momentum_balance_equation", nd), ("angular_momentum_balance_equation", self.nr)]
                         + [(e, 1) for e in self.scalar_balances])
        self.block_size = sum(w for _, w in self.fields)
        cells = [(("matrix",), self.nc, self.block_size)]
        self.unknown_layout = BlockLayout([("cell_fields", cells)] + list(unknowns))
        self.equation_layout = BlockLayout([("cell_balances", cells)] + list(equations))
        self.bc_values = self._vector(bc_values, nd * self.nf, bc_name)
        self.body_force = self._vector(body_force, nd * self.nc, "body_force")
        self.angular_source = self._vector(angular_source, self.nr * self.nc, "angular_source")
        self.mass_source = self._vector(mass_source, self.nc, "mass_source")
        self.column_map = None
        self.row_map = None
        self.A = None
        self._fg = None
        self._missing = None          # entries outside the row pattern, counted on the device (``TpsaNewtonProblem``)
        self.last_timing: dict = {}

    @staticmethod
    def _vector(v, n: int, name: str):
        if v is None:
            return None
        v = np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
        if v.size != n:
            raise ValueError(f"{name} must have {n} values, got {v.size}")
        return v

    def discretize(self) -> None:
        """The face inputs and the grid's device handle (kept for the next call), then ``_system``: the face terms
        (stage 1) and the rows of ``A`` (stage 2) on the device."""
        sd = self.sd
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        params = self.data[PARAMETERS][self.keyword]
        face = fv.tpsa_face_inputs(sd, params["bc"], self.nd)
        t0 = time.perf_counter()
        if self._fg is None:
            self._fg = fv.FaceGrid.for_grid(sd)
        self.last_timing = {}
        self.A, stage_ms = self._system(params["fourth_order_tensor"], *face)
        self.last_timing.update(face_terms_ms=stage_ms[0], rows_ms=stage_ms[1], total_s=time.perf_counter() - t0)

    def to_model_order(self, A, b=None):
        """A (scipy) and b permuted to the rows / columns of the model's ``EquationSystem``."""
        if self.column_map is None or self.row_map is None:
            raise ValueError(f"no dof maps: build the problem with model_bridge.{self.bridge}")
        n = self.num_dofs
        P = sps.csr_matrix((np.ones(n), (self.row_map, np.arange(n))), shape=(n, n))
        Q = sps.csr_matrix((np.ones(n), (np.arange(n), self.column_map)), shape=(n, n))
        Am = (P @ sps.csr_matrix(A) @ Q).tocsr()
        if b is None:
            return Am
        bm = np.empty(n)
        bm[self.row_map] = np.asarray(b)
        return Am, bm


class TpsaNewtonProblem(TpsaProblem):
    """A TPSA problem whose linear rows ``discretize`` writes once, with their -R(0) ``b0`` (``_rhs``), and whose other
    rows ``linearize`` writes into the fixed pattern at every iterate (``_iterate_rows``, ``_write_rows``).  A Newton
    step that counted entries outside that pattern raises ``RuntimeError(outside_pattern)``."""

    def discretize(self) -> None:
        super().discretize()
        self.b0 = self._rhs()

    def linearize(self, x, *state):
        """(J as ``DeviceCsr``, -R as a CUDA tensor) in the problem's order at the iterate ``x``: -R of the linear
        rows is b0 - A x; the rows of ``_iterate_rows(x, *state)`` are written into the fixed pattern.  ``J`` is the
        problem's own matrix, overwritten by the next call."""
        import torch
        if self.A is None:
            self.discretize()
        x = ad.device_vector(x)
        if x.numel() != self.num_dofs:
            raise ValueError(f"x must have {self.num_dofs} values")
        rows = self._iterate_rows(x, *state)
        rhs = self.b0 - (self.A @ x)
        if rows is None:
            return self.A, rhs
        if self._missing is None:
            self._missing = torch.zeros(1, dtype=torch.int32, device=rhs.device)
        self._write_rows(*rows, rhs)
        return self.A, rhs

    def _newton(self, linearize, x0, linear_solver, tol: float, max_iterations: int, verbose: bool):
        """``newton_loop`` from ``x0``; a linearization that counted entries outside the pattern raises
        ``RuntimeError``."""
        def checked(x):
            J, rhs = linearize(x)
            if self._missing is not None and int(self._missing.sum()):
                raise RuntimeError(self.outside_pattern)
            return J, rhs
        return newton_loop(checked, x0, linear_solver, tol, max_iterations, verbose)


class TpsaElasticity(TpsaProblem):
    """``A x = b`` of the TPSA momentum balance on grid ``sd`` (the arguments of ``TpsaProblem``)."""

    def __init__(self, sd, data: dict, keyword: str, bc_values, body_force=None, angular_source=None,
                 mass_source=None) -> None:
        super().__init__(sd, data, keyword, bc_values, body_force, angular_source, mass_source)

    def _system(self, C, codes, robin, flags):
        return self._fg.tpsa_system(self.nd, C.mu, C.lmbda, self.sd.cell_volumes, codes, robin, flags,
                                    self.sd.face_areas)

    def assemble(self):
        """(A, b): the system matrix (``DeviceCsr``) and b = -R(0) (CUDA tensor), both in the cell-interleaved order."""
        if self.A is None:
            self.discretize()
        b = self._fg.tpsa_rhs(self.num_dofs, self.bc_values, self.body_force, self.angular_source, self.mass_source)
        return self.A, b

    def solve(self, tol: float = 1e-10, maxiter: int = 2000):
        """Block-Jacobi BiCGStab (one inverted cell block per cell) on the device: (x as a CUDA tensor, solver info)."""
        from . import krylov
        A, b = self.assemble()
        solver = krylov.bicgstab_solver(tol, maxiter, self.block_size)
        return solver(A, b), solver.last_info


def interleave(parts, nd: int, nr: int, nc: int) -> np.ndarray:
    """Cell-interleaved order [u_c, r_c, s1_c, s2_c, ...] from the field-wise index arrays of a TPSA cell: u (nd per
    cell, cell-major), r (nr per cell), then any number of scalar fields (one per cell)."""
    widths = [nd, nr] + [1] * (len(parts) - 2)
    return np.concatenate([np.asarray(p, np.int64).reshape(nc, w) for p, w in zip(parts, widths)], axis=1).reshape(-1)
