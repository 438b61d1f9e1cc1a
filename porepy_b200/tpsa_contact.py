"""TPSA elasticity with fractures in frictional contact on the device: the reference's ``pp.MomentumBalance`` with
``TpsaMomentumBalanceMixin`` on a fractured medium (models/momentum_balance.py:127-183, constitutive_laws.py:3064-3248,
contact_mechanics.py:80-245).  The 2-D or 3-D matrix carries the three TPSA fields; its fracture faces are internal
Dirichlet faces whose boundary value is the interface displacement, ``g + Pi^avg u_j``, in the stress, the total rotation
and the solid-mass flux.

Unknowns: [u_c, r_c, p_c per matrix cell (cell by cell, as in ``TpsaElasticity``) | t (contact traction, nd per fracture
cell, local frame, scaled by the characteristic traction) | u_j (nd per mortar cell)]; equations, in the same blocks:

* ``cell_balances``                     momentum, angular momentum and solid mass of ``TpsaElasticity`` per cell, with
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

from . import ad, krylov
from .contact import (block_groups, contact_laws, contact_operators, fracture_parts, interface_parts,
                      matrix_dimension)
from .layout import BlockLayout
from .tpsa_elasticity import TpsaNewtonProblem


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


class TpsaFracturedMomentumBalance(TpsaNewtonProblem):
    """``sd``: the 2-D or 3-D matrix grid (faces split along the fractures); ``data``: ``parameters[keyword]`` with the
    ``fourth_order_tensor`` (``mu``, ``lmbda``) and the vectorial ``bc`` of ``pp.Tpsa`` (fracture faces Dirichlet);
    ``bc_values``: the combined mechanical boundary operator, nd per face, face-major; ``fractures``: ``FractureContact``
    per fracture; ``constants``: as for ``FracturedMomentumBalance``; ``body_force`` (nd per cell), ``angular_source``
    (nr per cell), ``mass_source`` (one per cell): cell-major, integrated over the cells (None: zero)."""

    bridge = "tpsa_fractured_momentum_from_model"
    outside_pattern = "contact Jacobian entries outside the TPSA contact row pattern"

    def __init__(self, sd, data: dict, bc_values, fractures, constants: dict, body_force=None, angular_source=None,
                 mass_source=None, keyword: str = "mechanics"):
        nd = matrix_dimension(sd)        # its refusal, ahead of the one of ``TpsaProblem``
        fr = self.fractures = list(fractures)
        laws = [("contact_traction", fracture_parts(fr, nd)), ("interface_displacement", interface_parts(fr, nd))]
        eqs = [("normal_fracture_deformation_equation", fracture_parts(fr, 1)),
               ("tangential_fracture_deformation_equation", fracture_parts(fr, nd - 1))]
        super().__init__(sd, data, keyword, bc_values, body_force, angular_source, mass_source, unknowns=laws,
                         equations=[("interface_force_balance_equation", interface_parts(fr, nd))] + eqs)
        for f in self.fractures:
            if f.nd != nd:
                raise ValueError(f"a fracture with {f.nd}-D local coordinates in a {nd}-D matrix")
        self.k = SimpleNamespace(**{k: float(v) for k, v in constants.items()})
        self._law_unknowns, self._law_equations = BlockLayout(laws), BlockLayout(eqs)
        self._ops = None

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

    def _system(self, C, codes, robin, flags):
        mortars, frames = self.interfaces()
        return self._fg.tpsa_contact_system(self.nd, C.mu, C.lmbda, self.sd.cell_volumes, codes, robin, flags,
                                            self.sd.face_areas, mortars, frames, self.k.characteristic_traction)

    def _rhs(self):
        return self._fg.tpsa_contact_rhs(self.num_dofs, self.bc_values, self.body_force, self.angular_source,
                                         self.mass_source)

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
    matrix_group = ([("cell_balances", "c")], [("cell_fields", "c")])
    fracture_group = ([("normal_fracture_deformation_equation", "k"), ("tangential_fracture_deformation_equation", "k"),
                       ("interface_force_balance_equation", "m1"), ("interface_force_balance_equation", "m2")],
                      [("contact_traction", "k"), ("interface_displacement", "m1"), ("interface_displacement", "m2")])
    preconditioner_groups = block_groups

    def _iterate_rows(self, x, x_prev):
        """The rows ``linearize(x, x_prev)`` writes (``x_prev``: the previous time step): the contact laws from the
        AD chain; none without fractures."""
        if not self.fractures:
            return None
        return ad.assemble(self.contact_equations(x, x_prev))

    def _write_rows(self, jac, neg_res, rhs):
        self._fg.tpsa_contact_rows(self.A, jac, neg_res, rhs, self._missing)

    def time_step(self, x_prev, linear_solver=None, x0=None, tol: float = 1e-10, max_iterations: int = 30,
                  verbose: bool = False):
        """Semismooth Newton from ``x0`` (default: the previous state); ``linear_solver(J, rhs) -> dx`` overrides the
        device GMRES with ``preconditioner_groups()``, ``krylov.gmres_solver`` with its defaults (GMRES(30) to 1e-12,
        at most 1,000 iterations), which raises ``RuntimeError`` when a solve does not converge.  Its iteration count
        grows with the grid: up to 600 per update at 16^3 matrix cells, up to 1,850 at 32^3 (DESIGN.md section 8); for
        such grids pass ``krylov.gmres_solver(prob.preconditioner_groups(), maxiter=...)``.  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        x0 = x_prev if x0 is None else ad.device_vector(x0)
        if linear_solver is None:
            linear_solver = krylov.gmres_solver(self.preconditioner_groups())
        return self._newton(lambda x: self.linearize(x, x_prev), x0, linear_solver, tol, max_iterations, verbose)
