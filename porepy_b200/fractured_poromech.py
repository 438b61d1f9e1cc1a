"""Poromechanics of a fractured medium with frictional contact -- the reference's ``pp.Poromechanics`` on a matrix cut by
fractures, BASELINE configs[3] + [4] in one model: Biot poromechanics in the 2-D or 3-D matrix (``nd = sd.dim``;
``porepy_b200.Mpfa`` + ``Biot``), compressible flow in the fractures of dimension nd - 1 (planes in 3-D; lines in 2-D,
whose fluxes run through the TPFA delegation of ``Mpfa``) with an aperture that follows the displacement jump, the
interface Darcy law with that aperture, the fluid pressure acting on the fracture walls, and the semismooth contact laws --
every term and its Jacobian by ``DeviceAdArray`` on device-resident matrices.

Couplings on top of ``porepy_b200.poromech`` (matrix), ``mdflow_nl`` (fracture flow, interface law) and ``contact``
(interface force balance, complementarity laws):

* aperture               a = max([u]_n + a_res, a_res)                       constitutive_laws.py:307-365
* fracture fluid mass    vol a rho(p_f)      (specific volume a, porosity 1)  constitutive_laws.py:203-282, 4509-4534
* interface Darcy law    lambda - vol kappa (2 Pi (1 / a)) (Pi tr p - Pi p_f): the normal gradient follows a
* matrix porosity        displacement_divergence u + boundary_displacement_divergence (u_b + Pi u_j)
* matrix stress          stress u + bound_stress (u_b + Pi u_j) + scalar_gradient (p - p0)
* force balance          ... + vol n_out Pi p_f         (``fracture_pressure_stress``, constitutive_laws.py:3470-3492)

As in the reference's Newton loop (``Poromechanics.add_nonlinear_darcy_flux_discretization``, models/poromechanics.py), the
fracture flux is RE-DISCRETIZED in front of every linearization with the tangential permeability times the current
aperture (``operator_to_SecondOrderTensor``: the specific volume of the iterate; not differentiated), next to the
upwinding.  Unknowns and equations: ``unknown_layout``, ``equation_layout`` (the fixtures carry the maps to the
reference's numbering).  One matrix subdomain, fractures without intersections; saddle-point Jacobian: the
linear solver of ``time_step`` is the caller's; ``krylov.gmres_solver(prob.preconditioner_groups())`` is the device one.  ``tests/golden/contact_poromech*.npz`` pin Jacobian, residual, the residual
history of the semismooth Newton loop and the converged state, ``contact_poromech_2d.npz`` the same on a line fracture.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps

from . import ad, ad_functions as fn
from .advection import advective_flux, rediscretize_upwind, rediscretize_upwind_coupling
from .contact import (block_groups, contact_laws, contact_operators, fracture_parts, interface_parts, local_dimension,
                      matrix_dimension)
from .fv import Biot, Mpfa
from .layout import BlockLayout, LayoutModel
from .newton import newton_loop
from .params import DISCRETIZATION_MATRICES, PARAMETERS


class FractureCoupling:
    """One fracture: its grid and data dictionary (``parameters[flow_keyword]``: ``bc``, ``ambient_dimension``; the
    ``second_order_tensor`` entry is written at every linearization: ``intrinsic_permeability`` (3, 3, nfc) times the
    aperture), the eight scalar mortar projections of its two-sided interface (``*_int`` / ``*_avg`` of the
    reference's ``MortarGrid``), ``mortar_sign``, ``mortar_volumes``, ``local_coordinates`` (nd nfc x nd nfc: nd - 1
    tangents, then the normal, per cell) and the normal permeability per mortar cell; ``bc``: boundary data of a fracture
    that reaches the domain boundary."""

    def __init__(self, sd, data, projections: dict, mortar_sign, mortar_volumes, local_coordinates, normal_permeability,
                 intrinsic_permeability, bc: dict | None = None):
        self.sd, self.data = sd, data
        # boundary data of a fracture that reaches the domain boundary: face arrays ``flow``, ``fluid_flux`` (and
        # ``fourier``, ``enthalpy_flux``) plus the objects ``fluid_flux_type`` (``enthalpy_flux_type``); None: closed tips
        self.bc = bc
        self.k_intrinsic = np.asarray(intrinsic_permeability, float)
        self.p = {k: sps.csr_matrix(v) for k, v in projections.items()}
        self.mortar_to_secondary = self.p["mortar_to_secondary_avg"]
        self.sign = np.asarray(mortar_sign, float)
        self.volumes = np.asarray(mortar_volumes, float)
        self.rotation = sps.csr_matrix(local_coordinates)
        self.kappa = np.asarray(normal_permeability, float)
        self.num_cells, self.num_mortar = int(sd.num_cells), int(self.sign.size)
        self.nd = local_dimension(self.rotation, self.num_cells)


class FracturedPoromechanics(LayoutModel):
    """``sd`` / ``data``: the 2-D or 3-D matrix grid (fracture faces split) with ``parameters[flow_keyword]`` and
    ``parameters[mechanics_keyword]`` (``scalar_vector_mappings`` = {flow_keyword: Biot coefficient}).  ``bc``: dict of face
    arrays ``flow``, ``mechanics`` (nd nf), ``fluid_flux`` and the object ``fluid_flux_type``.  ``fluid``: ``compressibility,
    density, viscosity, reference_pressure``; ``solid``: ``reference_porosity, n_inv, residual_aperture``; ``contact``: the
    constants of ``porepy_b200.contact``."""

    mobility_keyword = "mobility"

    def __init__(self, sd, data: dict, fractures, fluid: dict, solid: dict, contact: dict, bc: dict,
                 flow_keyword: str = "flow", mechanics_keyword: str = "mechanics"):
        self.nd = nd = matrix_dimension(sd)
        self.sd, self.data = sd, data
        self.fractures = list(fractures)
        for f in self.fractures:
            if f.nd != nd or int(f.sd.dim) != nd - 1:
                raise ValueError(f"a {int(f.sd.dim)}-D fracture with {f.nd}-D local coordinates in a {nd}-D matrix")
        self.fk, self.mk = flow_keyword, mechanics_keyword
        self.fl = SimpleNamespace(**{k: float(v) for k, v in fluid.items()})
        self.so = SimpleNamespace(**{k: float(v) for k, v in solid.items()})
        self.ct = SimpleNamespace(**{k: float(v) for k, v in contact.items()})
        self.bc = bc
        self.nc, self.nf = int(sd.num_cells), int(sd.num_faces)
        fr = self.fractures
        scalar, vector = [(("matrix",), self.nc, 1)] + fracture_parts(fr, 1), [(("matrix",), self.nc, nd)]
        flux, mortar = interface_parts(fr, 1), interface_parts(fr, nd)
        self.unknown_layout = BlockLayout([
            ("pressure", scalar), ("displacement", vector), ("contact_traction", fracture_parts(fr, nd)),
            ("interface_darcy_flux", flux), ("interface_displacement", mortar)])
        self.equation_layout = BlockLayout([
            ("mass_balance_equation", scalar), ("momentum_balance_equation", vector),
            ("interface_darcy_flux_equation", flux), ("interface_force_balance_equation", mortar),
            ("normal_fracture_deformation_equation", fracture_parts(fr, 1)),
            ("tangential_fracture_deformation_equation", fracture_parts(fr, nd - 1))])
        self._intf_data = [{} for _ in self.fractures]
        self._const = None

    def _discretize_fracture(self, fc, aperture) -> None:
        from .params import SecondOrderTensor
        fc.data[PARAMETERS][self.fk]["second_order_tensor"] = SecondOrderTensor.from_values(
            fc.k_intrinsic * np.asarray(aperture, float)[None, None, :])
        Mpfa(self.fk).discretize(fc.sd, fc.data)

    def discretize(self) -> None:
        """Matrix: Darcy flux and the Biot terms (once).  Fractures: Darcy flux at the residual aperture (re-discretized
        by ``update_discretizations`` at every iterate)."""
        Mpfa(self.fk).discretize(self.sd, self.data)
        Biot(self.mk).discretize(self.sd, self.data)
        for f in self.fractures:
            self._discretize_fracture(f, np.full(f.num_cells, self.so.residual_aperture))
        self._const = None

    def _operands(self):
        if self._const is None:
            csr, dev = ad.as_device_csr, ad.device_vector
            nd = self.nd
            eye = sps.identity(nd, format="csr")
            F = self.data[DISCRETIZATION_MATRICES][self.fk]
            M = self.data[DISCRETIZATION_MATRICES][self.mk]
            cf = sps.csr_matrix(self.sd.cell_faces)
            frac_faces = np.asarray(self.sd.tags["fracture_faces"], bool)
            out = np.where(frac_faces, np.asarray(cf.sum(axis=1)).ravel(), 0.0)
            vol = np.asarray(self.sd.cell_volumes, float)
            k = SimpleNamespace(
                div=csr(sps.csr_matrix(self.sd.cell_faces.T)), div_nd=csr(sps.kron(sps.csr_matrix(self.sd.cell_faces.T), eye).tocsr()),
                trace=csr(abs(cf)), vol=dev(vol), inv_vol=dev(1.0 / vol),
                F={key: csr(F[key]) for key in ("flux", "bound_flux", "bound_pressure_cell", "bound_pressure_face")},
                stress=csr(M["stress"]), bound=csr(M["bound_stress"]), grad_p=csr(M["scalar_gradient"][self.fk]),
                div_u=csr(M["displacement_divergence"][self.fk]), div_u_b=csr(M["boundary_displacement_divergence"][self.fk]),
                cons=csr(M["mpsa_consistency"][self.fk]), outward=dev(np.repeat(out, nd)),
                bcq=dev(self.bc["flow"]), ubc=dev(self.bc["mechanics"]), bcw=dev(self.bc["fluid_flux"]), fr=[])
            for fc in self.fractures:
                p = fc.p
                # unit normal of the primary face of every mortar cell, pointing out of the matrix, times the mortar volume
                pf = p["primary_to_mortar_avg"].tocsr().indices
                n_out = np.asarray(self.sd.face_normals)[:nd, pf] / np.asarray(self.sd.face_areas)[pf] * out[pf]
                rows = np.arange(nd * fc.num_mortar)
                pressure_load = sps.csr_matrix(((n_out * fc.volumes).ravel("F"), (rows, np.repeat(np.arange(fc.num_mortar), nd))),
                                               shape=(nd * fc.num_mortar, fc.num_mortar)) @ p["secondary_to_mortar_avg"]
                k.fr.append(SimpleNamespace(
                    m2p=csr(p["mortar_to_primary_int"]), p2m=csr(p["primary_to_mortar_avg"]),
                    m2s=csr(p["mortar_to_secondary_int"]), s2m=csr(p["secondary_to_mortar_avg"]),
                    m2p_nd=csr(sps.kron(p["mortar_to_primary_avg"], eye).tocsr()),
                    p2m_nd=csr(sps.kron(p["primary_to_mortar_int"], eye).tocsr()),
                    pressure_load=csr(pressure_load), coef=dev(fc.volumes * fc.kappa * 2.0),
                    div=csr(sps.csr_matrix(fc.sd.cell_faces.T)), vol=dev(np.asarray(fc.sd.cell_volumes, float)),
                    bc=None if fc.bc is None else {key: dev(v) for key, v in fc.bc.items() if not key.endswith("_type")},
                    **contact_operators(fc.rotation, sps.kron(p["mortar_to_secondary_avg"], eye),
                                        sps.diags(np.repeat(fc.sign, nd)), sps.kron(p["secondary_to_mortar_int"], eye),
                                        np.repeat(fc.volumes, nd), self.ct.characteristic_traction, nd)))
            self._const = k
        return self._const

    def _density(self, p):
        return ((p - self.fl.reference_pressure) * self.fl.compressibility).exp() * self.fl.density

    def _porosity(self, p, u, uj, k):
        dp = p - self.fl.reference_pressure
        b = k.ubc
        for j in range(len(self.fractures)):
            b = (k.fr[j].m2p_nd @ uj[j]) + b
        return ((k.div_u @ u) + (k.div_u_b @ b) + (k.cons @ dp)) * k.inv_vol + dp * self.so.n_inv + self.so.reference_porosity

    def _fracture_flux(self, fc, q, p, keyword=None, bc_key="flow"):
        """Diffusive flux of a fracture (Darcy by default): flux p (+ bound_flux p_b when the fracture carries boundary
        data)."""
        F = fc.data[DISCRETIZATION_MATRICES][keyword or self.fk]
        flux = ad.as_device_csr(F["flux"]) @ p
        if q.bc is not None:
            flux = flux + (ad.as_device_csr(F["bound_flux"]) @ q.bc[bc_key])
        return flux

    @staticmethod
    def _fracture_bc(q, key):
        """Boundary values ``key`` of a fracture, None for a fracture without boundary data."""
        return None if q.bc is None else q.bc[key]

    def _upwind_keywords(self):
        """(upwind keyword, key of its boundary-condition object in ``bc``) of every advected quantity."""
        return [(self.mobility_keyword, "fluid_flux_type")]

    def _aperture(self, uj_j, q):
        return fn.maximum((q.sel_n @ (q.jump @ uj_j)) + self.so.residual_aperture, self.so.residual_aperture)

    def update_discretizations(self, x) -> None:
        """What follows the iterate: the fracture flux discretization (aperture) and every upwind direction."""
        x = ad.device_vector(x)
        k = self._operands()
        parts = self.unknown_layout.parts(x)
        (p3, *pf), lam, uj = parts["pressure"], parts["interface_darcy_flux"], parts["interface_displacement"]
        for j, fc in enumerate(self.fractures):
            self._discretize_fracture(fc, self._aperture(uj[j], k.fr[j]).cpu().numpy())
        b = k.bcq
        for j in range(len(self.fractures)):
            b = (k.fr[j].m2p @ lam[j]) + b
        q3 = ((k.F["flux"] @ p3) + (k.F["bound_flux"] @ b)).cpu().numpy()
        for kw, key in self._upwind_keywords():
            rediscretize_upwind(self.sd, self.data, kw, q3, self.bc[key])
        for j, fc in enumerate(self.fractures):
            qf = self._fracture_flux(fc, k.fr[j], pf[j]).cpu().numpy()
            for kw, key in self._upwind_keywords():
                bc = fc.data[PARAMETERS][self.fk]["bc"] if fc.bc is None else fc.bc[key]
                rediscretize_upwind(fc.sd, fc.data, kw, qf, bc)
            rediscretize_upwind_coupling(self.sd, fc.sd, fc.num_mortar, self.data, fc.data, self._intf_data[j],
                                         self.mobility_keyword, lam[j].cpu().numpy())

    def equations(self, x, x_prev, dt: float) -> list:
        k, ct, fl = self._operands(), self.ct, self.fl
        csr = ad.as_device_csr
        nfr = len(self.fractures)
        mk = self.mobility_keyword
        x, x_prev = ad.device_vector(x), ad.device_vector(x_prev)
        var, prev = self.unknown_layout.variables(x), self.unknown_layout.parts(x_prev)
        (p3, *pf), (u,), t = var["pressure"], var["displacement"], var["contact_traction"]
        lam, uj = var["interface_darcy_flux"], var["interface_displacement"]
        (p3n, *pfn), (un,), ujn = prev["pressure"], prev["displacement"], prev["interface_displacement"]
        w3 = self._density(p3) * (1.0 / fl.viscosity)
        wf = [self._density(pf[j]) * (1.0 / fl.viscosity) for j in range(nfr)]
        # interface mass fluxes, boundary operators of the matrix
        ifl, b_flow, b_mech = [], k.bcq, k.ubc
        for j in range(nfr):
            q = k.fr[j]
            U = self._intf_data[j][DISCRETIZATION_MATRICES][mk]
            ifl.append(lam[j] * ((csr(U["upwind_primary"]) @ (q.p2m @ (k.trace @ w3)))
                                 + (csr(U["upwind_secondary"]) @ (q.s2m @ wf[j]))))
            b_flow = (q.m2p @ lam[j]) + b_flow
            b_mech = (q.m2p_nd @ uj[j]) + b_mech
        # ---- matrix: mass and momentum balance
        Tm = self.data[DISCRETIZATION_MATRICES][mk]
        q3 = (k.F["flux"] @ p3) + (k.F["bound_flux"] @ b_flow)
        neu = k.bcw
        for j in range(nfr):
            neu = (k.fr[j].m2p @ ifl[j]) + neu
        ff3 = advective_flux(Tm, q3, w3, k.bcw, neu)
        mass3 = (self._density(p3) * self._porosity(p3, u, uj, k) - self._density(p3n) * self._porosity(p3n, un, ujn, k)) \
            * (k.vol * (1.0 / dt)) + (k.div @ ff3)
        stress = (k.stress @ u) + (k.bound @ b_mech) + (k.grad_p @ (p3 - fl.reference_pressure))
        momentum = -(k.div_nd @ stress)
        trace_p = (k.F["bound_pressure_cell"] @ p3) + (k.F["bound_pressure_face"] @ b_flow)
        mass_f, darcy, force, normal, tangential = [], [], [], [], []
        for j, fc in enumerate(self.fractures):
            q = k.fr[j]
            a, a_n = self._aperture(uj[j], q), self._aperture(ujn[j], q)
            # ---- fracture: mass balance
            Tf = fc.data[DISCRETIZATION_MATRICES][mk]
            qf = self._fracture_flux(fc, q, pf[j])
            bw = self._fracture_bc(q, "fluid_flux")
            mass_f.append((a * self._density(pf[j]) - a_n * self._density(pfn[j])) * (q.vol * (1.0 / dt))
                          + (q.div @ advective_flux(Tf, qf, wf[j], bw, bw)) - (q.m2s @ ifl[j]))
            # ---- interface: Darcy law with the current aperture; force balance with the fluid pressure on the walls
            darcy.append(lam[j] - ((q.p2m @ trace_p) - (q.s2m @ pf[j])) * (q.s2m @ a.reciprocal()) * q.coef)
            force.append((q.p2m_nd @ (stress * k.outward)) + (q.traction @ t[j]) + (q.pressure_load @ pf[j]))
            nrm, tan = contact_laws(q, t[j], uj[j], ujn[j], ct)
            normal.append(nrm)
            tangential.append(tan)
        return self.equation_layout.stack({
            "mass_balance_equation": [mass3] + mass_f, "momentum_balance_equation": [momentum],
            "interface_darcy_flux_equation": darcy, "interface_force_balance_equation": force,
            "normal_fracture_deformation_equation": normal, "tangential_fracture_deformation_equation": tangential})

    # ``preconditioner_groups()``: nd + 1 unknowns per matrix cell c; per fracture cell k, those of ``contact`` plus the
    # fracture mass balance of k and the Darcy laws of its mortar cells (3 nd + 3: 12 in 3-D, 9 in 2-D)
    matrix_group = ([("mass_balance_equation", "c"), ("momentum_balance_equation", "c")],
                    [("pressure", "c"), ("displacement", "c")])
    fracture_group = ([("normal_fracture_deformation_equation", "k"), ("tangential_fracture_deformation_equation", "k"),
                       ("interface_force_balance_equation", "m1"), ("interface_force_balance_equation", "m2"),
                       ("mass_balance_equation", "k"), ("interface_darcy_flux_equation", "m1"),
                       ("interface_darcy_flux_equation", "m2")],
                      [("contact_traction", "k"), ("interface_displacement", "m1"), ("interface_displacement", "m2"),
                       ("pressure", "k"), ("interface_darcy_flux", "m1"), ("interface_darcy_flux", "m2")])
    preconditioner_groups = block_groups

    def linearize(self, x, x_prev, dt: float):
        self.update_discretizations(x)
        return ad.assemble(self.equations(x, x_prev, dt))

    def time_step(self, x_prev, dt: float, linear_solver, tol: float = 1e-10, max_iterations: int = 30, verbose: bool = False):
        """Semismooth Newton; ``linear_solver(J, rhs) -> dx``.  Returns (x, history)."""
        x_prev = ad.device_vector(x_prev)
        return newton_loop(lambda x: self.linearize(x, x_prev, dt), x_prev, linear_solver, tol, max_iterations, verbose)
