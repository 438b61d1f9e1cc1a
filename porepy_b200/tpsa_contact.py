"""TPSA elasticity with fractures in frictional contact on the device: the reference's ``pp.MomentumBalance`` with
``TpsaMomentumBalanceMixin`` on a fractured medium (models/momentum_balance.py:127-183, constitutive_laws.py:3064-3248,
contact_mechanics.py:80-245).  The 2-D or 3-D matrix carries the three TPSA fields; its fracture faces are internal
Dirichlet faces whose boundary value is the interface displacement, ``g + Pi^avg u_j``, in the stress, the total rotation
and the solid-mass flux.

Unknowns: [u_c, r_c, p_c per matrix cell (cell by cell, as in ``TpsaElasticity``) | t (contact traction, nd per fracture
cell, local frame, scaled by the characteristic traction) | u_j (nd per mortar cell)]; equations, in the same blocks:

* ``three_field_balance``               momentum, angular momentum and solid mass of ``TpsaElasticity`` per cell, with
                                        the u_j columns of the cell's fracture faces
* ``interface_force_balance_equation``  Pi^int (n_out . sigma) + vol S Pi^int R^T t T_c,
                                        sigma = S_u u + S_r r + S_p p + B_s (g + Pi^avg u_j)
* ``normal_fracture_deformation_equation``, ``tangential_fracture_deformation_equation``: ``contact.contact_laws``

The balance and force rows are linear and constant: ``pb_tpsa_contact_system`` writes them once per ``discretize`` into
a row pattern built on the device.  At every linearization the contact laws are evaluated on the device AD chain in the
variables [t | u_j], and ``pb_tpsa_contact_rows`` writes their Jacobian into the fixed contact rows; -R of the linear
rows is b0 - A x.  The complementarity rows have zeros on the diagonal, so the default solver is the device GMRES with the
grouped block-Jacobi of ``contact.block_groups``.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps

from . import ad, fv, krylov
from .contact import (block_groups, contact_laws, contact_operators, fracture_parts, interface_parts,
                      matrix_dimension)
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import PARAMETERS


def _one_per_row(m, what: str):
    """(column, weight) of every row of a matrix with exactly one entry per row; anything else raises ``ValueError``."""
    m = sps.csr_matrix(m)
    m.sum_duplicates()
    m.eliminate_zeros()
    count = np.diff(m.indptr)
    if (count != 1).any():
        r = int(np.flatnonzero(count != 1)[0])
        raise ValueError(f"{what}: mortar cell {r} maps to {int(count[r])} entries; only matching mortar grids (one "
                         f"face and one fracture cell per mortar cell) are supported")
    return m.indices.astype(np.int64), np.asarray(m.data, float)


class TpsaFracturedMomentumBalance(LayoutModel):
    """``sd``: the 2-D or 3-D matrix grid (faces split along the fractures); ``data``: ``parameters[keyword]`` with the
    ``fourth_order_tensor`` (``mu``, ``lmbda``) and the vectorial ``bc`` of ``pp.Tpsa`` (fracture faces Dirichlet);
    ``bc_values``: the combined mechanical boundary operator, nd per face, face-major; ``fractures``: ``FractureContact``
    per fracture; ``constants``: as for ``FracturedMomentumBalance``; ``body_force`` (nd per cell), ``angular_source``
    (nr per cell), ``mass_source`` (one per cell): cell-major, integrated over the cells (None: zero)."""

    def __init__(self, sd, data: dict, bc_values, fractures, constants: dict, body_force=None, angular_source=None,
                 mass_source=None, keyword: str = "mechanics"):
        self.nd = nd = matrix_dimension(sd)
        self.nr = 3 if nd == 3 else 1
        self.block_size = B = nd + self.nr + 1
        self.sd, self.data, self.kw = sd, data, keyword
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        self.fractures = list(fractures)
        for f in self.fractures:
            if f.nd != nd:
                raise ValueError(f"a fracture with {f.nd}-D local coordinates in a {nd}-D matrix")
        self.k = SimpleNamespace(**{k: float(v) for k, v in constants.items()})
        vec = TpsaFracturedMomentumBalance._vector
        self.bc_values = vec(bc_values, nd * self.nf, "bc_values")
        self.body_force = vec(body_force, nd * self.nc, "body_force")
        self.angular_source = vec(angular_source, self.nr * self.nc, "angular_source")
        self.mass_source = vec(mass_source, self.nc, "mass_source")
        fr, mat = self.fractures, [(("matrix",), self.nc, B)]
        laws = [("contact_traction", fracture_parts(fr, nd)), ("interface_displacement", interface_parts(fr, nd))]
        self.unknown_layout = BlockLayout([("three_field", mat)] + laws)
        eqs = [("normal_fracture_deformation_equation", fracture_parts(fr, 1)),
               ("tangential_fracture_deformation_equation", fracture_parts(fr, nd - 1))]
        self.equation_layout = BlockLayout([("three_field_balance", mat),
                                            ("interface_force_balance_equation", interface_parts(fr, nd))] + eqs)
        self._law_unknowns, self._law_equations = BlockLayout(laws), BlockLayout(eqs)
        self.column_map = None
        self.row_map = None
        self.A = None
        self._fg = None
        self._ops = None
        self._missing = None
        self.last_timing: dict = {}

    @staticmethod
    def _vector(v, n: int, name: str):
        if v is None:
            return None
        v = np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
        if v.size != n:
            raise ValueError(f"{name} must have {n} values, got {v.size}")
        return v

    def interfaces(self):
        """(per mortar cell: ``face``, ``cell``, ``m2p``, ``p2m``, ``sign``, ``volume``; the frames, nd x nd per fracture
        cell) of all fractures, numbered one after the other.  A mortar cell without exactly one face or fracture
        cell, or a face with several mortar cells, raises ``ValueError``."""
        nd = self.nd
        out = {k: [] for k in ("face", "cell", "m2p", "p2m", "sign", "volume")}
        frames, k0 = [], 0
        for fc in self.fractures:
            face, m2p = _one_per_row(fc.m2p[::nd, ::nd].T, "mortar_to_primary_avg")
            p_face, p2m = _one_per_row(fc.p2m[::nd, ::nd], "primary_to_mortar_int")
            cell, s2m = _one_per_row(fc.s2m[::nd, ::nd], "secondary_to_mortar_int")
            if not np.array_equal(face, p_face):
                raise ValueError("mortar_to_primary_avg and primary_to_mortar_int map a mortar cell to different faces")
            if np.unique(face).size != face.size:
                raise ValueError("a face with more than one mortar cell; only matching mortar grids are supported")
            out["face"].append(face)
            out["cell"].append(cell + k0)
            out["m2p"].append(m2p)
            out["p2m"].append(p2m)
            out["sign"].append(fc.sign.diagonal()[::nd])
            out["volume"].append(fc.volumes[::nd] * s2m)
            R = fc.rotation.tocoo()
            if np.any(R.row // nd != R.col // nd):
                raise ValueError("local coordinates must be block diagonal, one nd x nd frame per fracture cell")
            blk = np.zeros((fc.num_cells, nd, nd))
            blk[R.row // nd, R.row % nd, R.col % nd] = R.data
            frames.append(blk.reshape(-1))
            k0 += fc.num_cells
        cat = {k: np.concatenate(v) if v else np.zeros(0) for k, v in out.items()}
        return cat, (np.concatenate(frames) if frames else np.zeros(0))

    def discretize(self) -> None:
        """The TPSA face terms, the balance and force rows of the Jacobian and their -R(0) on the device."""
        import time
        sd, nd = self.sd, self.nd
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        params = self.data[PARAMETERS][self.kw]
        C = params["fourth_order_tensor"]
        codes, robin = fv.tpsa_bc_arrays(params["bc"], nd, self.nf)
        if nd == 2 and np.any(np.abs(sd.face_normals[2]) > np.maximum(np.abs(sd.face_normals[0]),
                                                                       np.abs(sd.face_normals[1]))):
            raise IndexError("Tpsa: a face normal of a 2d grid points mostly out of the xy-plane")
        flags = np.zeros(self.nf, np.uint8)
        flags[np.asarray(sd.get_all_boundary_faces(), dtype=np.int64)] = 1
        mortars, frames = self.interfaces()
        t0 = time.perf_counter()
        if self._fg is None:
            self._fg = fv.FaceGrid.for_grid(sd)
        self.A, stage_ms = self._fg.tpsa_contact_system(nd, C.mu, C.lmbda, sd.cell_volumes, codes, robin, flags,
                                                        sd.face_areas, mortars, frames, self.k.characteristic_traction)
        self.b0 = self._fg.tpsa_contact_rhs(self.num_dofs, self.bc_values, self.body_force, self.angular_source,
                                            self.mass_source)
        self.last_timing = dict(face_terms_ms=stage_ms[0], rows_ms=stage_ms[1], total_s=time.perf_counter() - t0)

    def _operators(self):
        if self._ops is None:
            self._ops = [SimpleNamespace(**contact_operators(fc.rotation, fc.m2s, fc.sign, fc.s2m, fc.volumes,
                                                             self.k.characteristic_traction, self.nd))
                         for fc in self.fractures]
        return self._ops

    def contact_equations(self, x, x_prev) -> list:
        """The [normal | tangential] laws of all fractures as ``DeviceAdArray`` in the variables [t | u_j]."""
        n0 = self.block_size * self.nc
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var = self._law_unknowns.variables(x[n0:])
        ujn = self._law_unknowns.parts(x_prev[n0:])["interface_displacement"]
        normal, tangential = [], []
        for j, q in enumerate(self._operators()):
            nrm, tan = contact_laws(q, var["contact_traction"][j], var["interface_displacement"][j], ujn[j], self.k)
            normal.append(nrm)
            tangential.append(tan)
        return self._law_equations.stack({"normal_fracture_deformation_equation": normal,
                                          "tangential_fracture_deformation_equation": tangential})

    # ``preconditioner_groups()``: the B x B cell block per matrix cell; the laws of fracture cell k and the force
    # balances of its mortar cells m1, m2 <-> t_k, u_j of m1, m2
    matrix_group = ([("three_field_balance", "c")], [("three_field", "c")])
    fracture_group = ([("normal_fracture_deformation_equation", "k"), ("tangential_fracture_deformation_equation", "k"),
                       ("interface_force_balance_equation", "m1"), ("interface_force_balance_equation", "m2")],
                      [("contact_traction", "k"), ("interface_displacement", "m1"), ("interface_displacement", "m2")])
    preconditioner_groups = block_groups

    def linearize(self, x, x_prev):
        """(J as ``DeviceCsr``, -R as a CUDA tensor) at the iterate ``x`` (previous time step ``x_prev``): -R of the
        linear rows is b0 - A x, the contact rows come from the AD chain, written into the fixed pattern.  ``J`` is the
        problem's own matrix, overwritten by the next call."""
        import torch
        if self.A is None:
            self.discretize()
        x = ad.device_vector(x)
        if x.numel() != self.num_dofs:
            raise ValueError(f"x must have {self.num_dofs} values")
        rhs = self.b0 - (self.A @ x)
        if not self.fractures:
            return self.A, rhs
        jac, neg_res = ad.assemble(self.contact_equations(x, x_prev))
        if self._missing is None:
            self._missing = torch.zeros(1, dtype=torch.int32, device=rhs.device)
        self._fg.tpsa_contact_rows(self.A, jac, neg_res, rhs, self._missing)
        return self.A, rhs

    def time_step(self, x_prev, linear_solver=None, x0=None, tol: float = 1e-10, max_iterations: int = 30,
                  verbose: bool = False):
        """Semismooth Newton from ``x0`` (default: the previous state); ``linear_solver(J, rhs) -> dx`` overrides the
        device GMRES with ``preconditioner_groups()``, ``krylov.gmres_solver`` with its defaults (GMRES(30) to 1e-12,
        at most 1,000 iterations), which raises ``RuntimeError`` when a solve does not converge.  Its iteration count
        grows with the grid: up to 600 per update at 16^3 matrix cells, up to 1,850 at 32^3 (DESIGN.md section 8); for
        such grids pass ``krylov.gmres_solver(prob.preconditioner_groups(), maxiter=...)``.  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        x0 = x_prev if x0 is None else ad.device_vector(x0)

        def linearize(x):
            J, rhs = self.linearize(x, x_prev)
            if self._missing is not None and int(self._missing.sum()):
                raise RuntimeError("contact Jacobian entries outside the TPSA contact row pattern")
            return J, rhs
        if linear_solver is None:
            linear_solver = krylov.gmres_solver(self.preconditioner_groups())
        return newton_loop(linearize, x0, linear_solver, tol, max_iterations, verbose)

    def to_model_order(self, A, b=None):
        """A (scipy) and b permuted to the rows / columns of the model's ``EquationSystem``."""
        if self.column_map is None or self.row_map is None:
            raise ValueError("no dof maps: build the problem with model_bridge.tpsa_fractured_momentum_from_model")
        n = self.num_dofs
        P = sps.csr_matrix((np.ones(n), (self.row_map, np.arange(n))), shape=(n, n))
        Q = sps.csr_matrix((np.ones(n), (np.arange(n), self.column_map)), shape=(n, n))
        Am = (P @ sps.csr_matrix(A) @ Q).tocsr()
        if b is None:
            return Am
        bm = np.empty(n)
        bm[self.row_map] = np.asarray(b)
        return Am, bm
