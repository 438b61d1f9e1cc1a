"""The TPSA three-field elasticity system on the device: the reference's ``pp.MomentumBalance`` with
``TpsaMomentumBalanceMixin`` (models/momentum_balance.py:82-106, 250-280, 344-368) on one grid without fractures,
assembled by ``pb_tpsa_system`` / ``pb_tpsa_rhs`` (csrc/tpsa_system.cuh) and solved by the fused block-Jacobi BiCGStab
of ``krylov``.

Unknowns per cell: the displacement u (nd), the rotation stress r (nr = 3 in 3-D, 1 in 2-D) and the total pressure p.
Unknowns and equations are numbered cell by cell, ``[u_c, r_c, p_c]``, so the diagonal blocks of ``A`` are the
(nd + nr + 1)^2 cell blocks the preconditioner inverts.  ``column_map`` / ``row_map`` (set by
``model_bridge.tpsa_momentum_from_model``) give the model's ``EquationSystem`` dof / row of each unknown / equation.
"""
from __future__ import annotations

import time

import numpy as np
import scipy.sparse as sps

from . import fv
from .params import PARAMETERS


class TpsaElasticity:
    """``A x = b`` of the TPSA momentum balance on grid ``sd``.  ``data[PARAMETERS][keyword]`` holds the
    ``fourth_order_tensor`` (``mu``, ``lmbda``) and the ``bc`` of ``pp.Tpsa``; ``bc_values`` is the combined
    mechanical boundary operator (nd values per face, face-major); ``body_force`` (nd per cell), ``angular_source``
    (nr per cell) and ``mass_source`` (one per cell) are cell-major and already integrated over the cells (None:
    zero)."""

    def __init__(self, sd, data: dict, keyword: str, bc_values, body_force=None, angular_source=None,
                 mass_source=None) -> None:
        self.sd, self.data, self.keyword = sd, data, keyword
        self.nd = int(sd.dim)
        if self.nd not in (2, 3):
            raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")
        self.nr = 3 if self.nd == 3 else 1
        self.block_size = self.nd + self.nr + 1
        nc, nf = sd.num_cells, sd.num_faces
        self.bc_values = self._vector(bc_values, self.nd * nf, "bc_values")
        self.body_force = self._vector(body_force, self.nd * nc, "body_force")
        self.angular_source = self._vector(angular_source, self.nr * nc, "angular_source")
        self.mass_source = self._vector(mass_source, nc, "mass_source")
        self.column_map = None
        self.row_map = None
        self.A = None
        self._fg = None
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
        return self.block_size * self.sd.num_cells

    def discretize(self) -> None:
        """Face terms (stage 1) and the rows of ``A`` (stage 2) on the device; the row pattern is built at the first
        call and kept with the grid's device handle."""
        sd, nd = self.sd, self.nd
        params = self.data[PARAMETERS][self.keyword]
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        C = params["fourth_order_tensor"]
        codes, robin = fv.tpsa_bc_arrays(params["bc"], nd, sd.num_faces)
        if nd == 2 and np.any(np.abs(sd.face_normals[2]) > np.maximum(np.abs(sd.face_normals[0]),
                                                                       np.abs(sd.face_normals[1]))):
            raise IndexError("Tpsa: a face normal of a 2d grid points mostly out of the xy-plane")
        flags = np.zeros(sd.num_faces, np.uint8)
        flags[np.asarray(sd.get_all_boundary_faces(), dtype=np.int64)] = 1
        t0 = time.perf_counter()
        if self._fg is None:
            self._fg = fv.FaceGrid.for_grid(sd)
        self.A, stage_ms = self._fg.tpsa_system(nd, C.mu, C.lmbda, sd.cell_volumes, codes, robin, flags,
                                                sd.face_areas)
        self.last_timing = dict(face_terms_ms=stage_ms[0], rows_ms=stage_ms[1], total_s=time.perf_counter() - t0)

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

    def to_model_order(self, A, b=None):
        """A (scipy) and b permuted to the rows / columns of the model's ``EquationSystem``."""
        if self.column_map is None or self.row_map is None:
            raise ValueError("no dof maps: build the problem with model_bridge.tpsa_momentum_from_model")
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
    """Cell-interleaved order [u_c, r_c, p_c] from the three field-wise index arrays (u: nd per cell, cell-major;
    r: nr per cell; p: one per cell)."""
    u, r, p = (np.asarray(x, np.int64) for x in blocks)
    out = np.empty((nc, nd + nr + 1), np.int64)
    out[:, :nd] = u.reshape(nc, nd)
    out[:, nd:nd + nr] = r.reshape(nc, nr)
    out[:, nd + nr] = p
    return out.reshape(-1)
