"""Frictional contact on fractures, the reference's ``pp.MomentumBalance`` on the device AD chain -- the contact part of
BASELINE config[4]: MPSA elasticity in the 3-D matrix (``porepy_b200.Mpsa``; the two sides of every fracture are internal
Dirichlet boundaries carrying the interface displacement), force balance on the matrix-fracture interfaces and the
semismooth complementarity laws of the contact traction.  The matrix is 2-D or 3-D (``nd = sd.dim``), the fractures are
lines or planes of dimension ``nd - 1``.

Unknowns: [u (nd per matrix cell) | t (contact traction, nd per fracture cell, in the fracture's local frame: the nd - 1
tangential components, then the normal one; scaled by the characteristic traction) | u_j (nd per mortar cell)];
equations, in the reference's order:

* ``momentum_balance_equation``        -div_nd (stress u + bound_stress (u_b + Pi^avg u_j)) - f          models/momentum_balance.py
* ``interface_force_balance_equation`` Pi^int (n_out . sigma) + vol S Pi^int R^T t T_c                    momentum_balance.py:127-183,
                                                                                               constitutive_laws.py:2956-3001
* ``normal_fracture_deformation_equation``      t_n + max(-t_n - c ([u]_n - g), 0),   g = g0 + tan(psi) ||[u]_t||
                                                                                               contact_mechanics.py:80-129
* ``tangential_fracture_deformation_equation``  (1 - chi) (b_p s - max(b_p, ||s||) t_t) + chi t_t,
                                       s = t_t + c ([u]_t - [u]_t^n),  b_p = max(-mu_f t_n, 0),  chi = 1 where b_p <= tol
                                                                                               contact_mechanics.py:131-245

with the displacement jump ``[u] = R Pi^avg_{mortar -> fracture} S u_j`` (``S``: side signs, ``R``: global -> local
coordinates; constitutive_laws.py ``displacement_jump``).  ``maximum`` / ``l2_norm`` / ``characteristic_function`` are those of
``porepy_b200.ad_functions`` with the reference's tie rules, so the Jacobian of the semismooth laws is the reference's.  The
elastic fracture-deformation laws (Barton-Bandis closure, tangential stiffness) are off in the reference's defaults and not
stated here.  The Jacobian has zeros on the diagonal of the complementarity rows: ``time_step`` takes the linear solver from
the caller.  ``krylov.gmres_solver(prob.preconditioner_groups())`` solves the updates on the device: restarted GMRES with a
block-Jacobi over one group per matrix cell and one per fracture cell with its two mortar cells.
``tests/golden/contact_model.npz`` pins Jacobian, residual, residual history and the converged sliding state.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps

from . import ad, ad_functions as fn
from .fv import Mpsa
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES


class FractureContact:
    """One fracture and its two-sided interface: ``mortar_to_primary_avg``, ``primary_to_mortar_int`` (faces of the matrix
    grid), ``mortar_to_secondary_avg``, ``secondary_to_mortar_int`` (cells of the fracture): the SCALAR projections of the
    reference's ``MortarGrid``; ``mortar_sign`` (+-1 per mortar cell: ``sign_of_mortar_sides``), ``mortar_volumes``,
    ``local_coordinates`` (nd nfc x nd nfc, rows per cell: the nd - 1 tangents, then the normal; ``nd`` follows from its
size)."""

    def __init__(self, mortar_to_primary_avg, primary_to_mortar_int, mortar_to_secondary_avg, secondary_to_mortar_int,
                 mortar_sign, mortar_volumes, local_coordinates):
        self.mortar_to_secondary = sps.csr_matrix(mortar_to_secondary_avg)
        self.rotation = sps.csr_matrix(local_coordinates)
        self.num_mortar = int(np.asarray(mortar_sign).size)
        self.num_cells = int(self.mortar_to_secondary.shape[0])
        self.nd = local_dimension(self.rotation, self.num_cells)
        eye = sps.identity(self.nd, format="csr")
        self.m2p = sps.kron(sps.csr_matrix(mortar_to_primary_avg), eye).tocsr()
        self.p2m = sps.kron(sps.csr_matrix(primary_to_mortar_int), eye).tocsr()
        self.m2s = sps.kron(self.mortar_to_secondary, eye).tocsr()
        self.s2m = sps.kron(sps.csr_matrix(secondary_to_mortar_int), eye).tocsr()
        self.sign = sps.diags(np.repeat(np.asarray(mortar_sign, float), self.nd)).tocsr()
        self.volumes = np.repeat(np.asarray(mortar_volumes, float), self.nd)


def matrix_dimension(sd) -> int:
    """``sd.dim`` of a matrix grid that carries mechanics: 2 or 3, anything else raises ``NotImplementedError``."""
    nd = int(sd.dim)
    if nd not in (2, 3):
        raise NotImplementedError(f"the mechanics equations are stated for a 2-D or 3-D matrix grid, not a {nd}-D one")
    return nd


def local_dimension(local_coordinates, num_cells: int) -> int:
    """``nd`` of the square ``local_coordinates`` (nd num_cells rows) of a fracture with ``num_cells`` cells; anything
    but a 2 x 2 or 3 x 3 frame per cell raises ``ValueError``."""
    rows = int(local_coordinates.shape[0])
    if num_cells < 1 or rows % num_cells or rows // num_cells not in (2, 3) or int(local_coordinates.shape[1]) != rows:
        raise ValueError(f"local coordinates of shape {tuple(local_coordinates.shape)} do not hold a 2 x 2 or 3 x 3 "
                         f"frame per cell of a fracture with {num_cells} cells")
    return rows // num_cells


def mortar_pairs(mortar_to_secondary) -> np.ndarray:
    """(nfc, 2): the two mortar cells of every fracture cell, from the scalar ``mortar_to_secondary_avg``; a fracture cell
    with another number of mortar cells raises ``ValueError``."""
    m = sps.csr_matrix(mortar_to_secondary)
    m.sort_indices()
    count = np.diff(m.indptr)
    if (count != 2).any():
        k = int(np.flatnonzero(count != 2)[0])
        raise ValueError(f"fracture cell {k} has {int(count[k])} mortar cells; the preconditioner groups need two")
    return m.indices.reshape(-1, 2).astype(np.int64)


def fracture_parts(fractures, width: int) -> list:
    """``BlockLayout`` parts of ``width`` entries per cell on every fracture."""
    return [(("fracture", j), f.num_cells, width) for j, f in enumerate(fractures)]


def interface_parts(fractures, width: int) -> list:
    """``BlockLayout`` parts of ``width`` entries per mortar cell on the interface of every fracture."""
    return [(("interface", j), f.num_mortar, width) for j, f in enumerate(fractures)]


def block_groups(prob):
    """``krylov.BlockGroups`` of the grouped block-Jacobi preconditioner of ``krylov.gmres`` for ``prob``: one group per
    matrix cell c and one per fracture cell k with its mortar cells m1, m2, declared by ``prob.matrix_group`` /
    ``prob.fracture_group`` as (rows, cols) lists of (equation block, cell) / (unknown block, cell)."""
    from .krylov import BlockGroups

    def group(decl, cells):
        rows, cols = decl
        return (np.hstack([prob.equation_layout.span(b, *cells[c]) for b, c in rows]),
                np.hstack([prob.unknown_layout.span(b, *cells[c]) for b, c in cols]))
    blocks = [group(prob.matrix_group, {"c": (("matrix",), np.arange(prob.nc))})]
    for j, fc in enumerate(prob.fractures):
        m = mortar_pairs(fc.mortar_to_secondary)
        blocks.append(group(prob.fracture_group, {"k": (("fracture", j), np.arange(fc.num_cells)),
                                                  "m1": (("interface", j), m[:, 0]), "m2": (("interface", j), m[:, 1])}))
    sizes = np.concatenate([np.full(r.shape[0], r.shape[1], np.int64) for r, _ in blocks])
    return BlockGroups(np.concatenate(([0], np.cumsum(sizes))), np.concatenate([r.ravel() for r, _ in blocks]),
                       np.concatenate([c.ravel() for _, c in blocks]))


def contact_operators(rotation, mortar_to_secondary, sign, secondary_to_mortar, volumes, characteristic_traction: float,
                      nd: int = 3):
    """Device operators of the contact laws of one fracture with n cells in an ``nd``-D matrix: ``sel_n`` / ``sel_t``
    (normal / tangential components of a local nd-vector per cell: the last one / the nd - 1 first ones), ``s2t`` (one
    value per cell to its nd - 1 tangential components), ``jump`` (u_j -> local displacement jump) and ``traction``
    (contact traction -> force on the mortar cells), and ``nd`` itself.  ``rotation``: ``local_coordinates``;
    ``mortar_to_secondary``, ``sign``, ``secondary_to_mortar``: the nd-component projections and side signs;
    ``volumes``: mortar volumes, nd per mortar cell."""
    csr = ad.as_device_csr
    nt = nd - 1
    n = rotation.shape[0] // nd
    sel_n = sps.csr_matrix((np.ones(n), (np.arange(n), nd * np.arange(n) + nt)), shape=(n, nd * n))
    sel_t = sps.csr_matrix((np.ones(nt * n), (np.arange(nt * n), nd * np.repeat(np.arange(n), nt)
                                              + np.tile(np.arange(nt), n))), shape=(nt * n, nd * n))
    s2t = sps.csr_matrix((np.ones(nt * n), (np.arange(nt * n), np.repeat(np.arange(n), nt))), shape=(nt * n, n))
    jump = rotation @ mortar_to_secondary @ sign
    traction = sps.diags(volumes * characteristic_traction) @ sign @ secondary_to_mortar @ rotation.T
    return dict(sel_n=csr(sel_n), sel_t=csr(sel_t), s2t=csr(s2t), jump=csr(jump), traction=csr(traction), nd=nd)


def contact_laws(q, t, u_j, u_j_prev, c):
    """(normal, tangential) complementarity laws of one fracture: ``q`` holds the ``contact_operators``, ``t`` and
    ``u_j`` are the contact traction and the mortar displacement of the iterate, ``u_j_prev`` that of the previous time
    step, ``c`` the contact constants.  Tangential norms are over the ``q.nd - 1`` tangential components, as in
    models/contact_mechanics.py:177-201 (for a line fracture: the absolute value)."""
    nt = q.nd - 1
    jump, jump_n = q.jump @ u_j, q.jump @ u_j_prev
    t_n, u_n = q.sel_n @ t, q.sel_n @ jump
    t_t, u_t, u_t_prev = q.sel_t @ t, q.sel_t @ jump, q.sel_t @ jump_n
    gap = fn.l2_norm(nt, u_t) * float(np.tan(c.dilation_angle)) + c.reference_gap
    normal = t_n + fn.maximum(-t_n - (u_n - gap) * c.numerical_constant, 0.0)
    s = t_t + (u_t - u_t_prev) * c.numerical_constant
    b_p = fn.maximum(t_n * (-c.friction_coefficient), 0.0)
    chi = q.s2t @ fn.characteristic_function(c.open_state_tolerance, b_p).val
    tangential = ((q.s2t @ b_p) * s - (q.s2t @ fn.maximum(b_p, fn.l2_norm(nt, s))) * t_t) * (1.0 - chi) + t_t * chi
    return normal, tangential


class FracturedMomentumBalance(LayoutModel):
    """``sd``: the 2-D or 3-D matrix grid (faces split along the fractures, ``fracture_faces`` tag), ``data``:
    ``parameters[keyword]`` with ``fourth_order_tensor`` and the vectorial ``bc`` (fracture faces Dirichlet,
    ``internal_to_dirichlet``); ``bc_values``: nd nf face-major (displacement / traction); ``fractures``: list of
    ``FractureContact`` (dimension nd - 1); ``constants``: ``numerical_constant, characteristic_traction,
    friction_coefficient, dilation_angle, reference_gap, open_state_tolerance``."""

    def __init__(self, sd, data: dict, bc_values, fractures, constants: dict, body_force=None, keyword: str = "mechanics"):
        self.nd = nd = matrix_dimension(sd)
        self.sd, self.data, self.kw = sd, data, keyword
        self.bc_values = np.asarray(bc_values, float)
        self.fractures = list(fractures)
        for f in self.fractures:
            if f.nd != nd:
                raise ValueError(f"a fracture with {f.nd}-D local coordinates in a {nd}-D matrix")
        self.k = SimpleNamespace(**{k: float(v) for k, v in constants.items()})
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        self.body_force = np.zeros(nd * self.nc) if body_force is None else np.asarray(body_force, float)
        fr, mat = self.fractures, [(("matrix",), self.nc, nd)]
        self.unknown_layout = BlockLayout([("displacement", mat), ("contact_traction", fracture_parts(fr, nd)),
                                           ("interface_displacement", interface_parts(fr, nd))])
        self.equation_layout = BlockLayout([
            ("momentum_balance_equation", mat), ("interface_force_balance_equation", interface_parts(fr, nd)),
            ("normal_fracture_deformation_equation", fracture_parts(fr, 1)),
            ("tangential_fracture_deformation_equation", fracture_parts(fr, nd - 1))])
        self._const = None

    def discretize(self) -> None:
        Mpsa(self.kw).discretize(self.sd, self.data)
        self._const = None

    def _operands(self):
        if self._const is None:
            csr, dev = ad.as_device_csr, ad.device_vector
            M = self.data[DISCRETIZATION_MATRICES][self.kw]
            cf = sps.csr_matrix(self.sd.cell_faces)
            frac = np.asarray(self.sd.tags["fracture_faces"], bool)
            out = np.where(frac, np.asarray(cf.sum(axis=1)).ravel(), 0.0)      # +-1 on fracture faces: outward normal
            k = SimpleNamespace(
                div_nd=csr(sps.kron(sps.csr_matrix(self.sd.cell_faces.T), sps.identity(self.nd)).tocsr()),
                stress=csr(M["stress"]), bound=csr(M["bound_stress"]),
                outward=dev(np.repeat(out, self.nd)), f=dev(self.body_force), fr=[])
            k.stress_b = k.bound @ dev(self.bc_values)
            for fc in self.fractures:
                k.fr.append(SimpleNamespace(m2p=csr(fc.m2p), p2m=csr(fc.p2m), **contact_operators(
                    fc.rotation, fc.m2s, fc.sign, fc.s2m, fc.volumes, self.k.characteristic_traction, self.nd)))
            self._const = k
        return self._const

    def equations(self, x, x_prev) -> list:
        k, c = self._operands(), self.k
        nfr = len(self.fractures)
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var = self.unknown_layout.variables(x)
        u, t, uj = var["displacement"][0], var["contact_traction"], var["interface_displacement"]
        ujn = self.unknown_layout.parts(x_prev)["interface_displacement"]
        boundary = None
        for j in range(nfr):
            term = k.fr[j].m2p @ uj[j]
            boundary = term if boundary is None else boundary + term
        stress = (k.stress @ u) + k.stress_b
        if boundary is not None:
            stress = stress + (k.bound @ boundary)
        momentum = -(k.div_nd @ stress) - k.f
        force, normal, tangential = [], [], []
        for j in range(nfr):
            q = k.fr[j]
            force.append((q.p2m @ (stress * k.outward)) + (q.traction @ t[j]))
            nrm, tan = contact_laws(q, t[j], uj[j], ujn[j], c)
            normal.append(nrm)
            tangential.append(tan)
        return self.equation_layout.stack({
            "momentum_balance_equation": [momentum], "interface_force_balance_equation": force,
            "normal_fracture_deformation_equation": normal, "tangential_fracture_deformation_equation": tangential})

    # ``preconditioner_groups()``: momentum_c <-> u_c (nd) per matrix cell c; the normal and tangential laws of fracture
    # cell k and the force balances of its mortar cells m1, m2 <-> t_k, u_j of m1, m2 (3 nd: 9 in 3-D, 6 in 2-D)
    matrix_group = ([("momentum_balance_equation", "c")], [("displacement", "c")])
    fracture_group = ([("normal_fracture_deformation_equation", "k"), ("tangential_fracture_deformation_equation", "k"),
                       ("interface_force_balance_equation", "m1"), ("interface_force_balance_equation", "m2")],
                      [("contact_traction", "k"), ("interface_displacement", "m1"), ("interface_displacement", "m2")])
    preconditioner_groups = block_groups

    def linearize(self, x, x_prev):
        """(J as ``DeviceCsr``, -R as a CUDA tensor) at the iterate ``x`` (previous time step ``x_prev``)."""
        return ad.assemble(self.equations(x, x_prev))

    def time_step(self, x_prev, linear_solver, x0=None, tol: float = 1e-10, max_iterations: int = 30, verbose: bool = False):
        """Semismooth Newton from ``x0`` (default: the previous state); ``linear_solver(J, rhs) -> dx``."""
        x_prev = ad.device_vector(x_prev)
        x0 = x_prev if x0 is None else ad.device_vector(x0)
        return newton_loop(lambda x: self.linearize(x, x_prev), x0, linear_solver, tol, max_iterations, verbose)
