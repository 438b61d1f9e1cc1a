"""Generate tests/golden/tpsa_model_*.npz from the unmodified reference's TPSA momentum-balance model
(``pp.MomentumBalance`` with ``TpsaMomentumBalanceMixin``), run in the build container where the reference is
importable.

Every model has heterogeneous mu and lambda, a non-zero body force and Dirichlet, roller, Neumann and Robin faces.  Each
fixture holds
  * the grid (``make_golden.grid_arrays``), mu, lambda, the boundary condition and the 14 TPSA matrices of the model's
    discretization in the layout of the ``tpsa_*`` fixtures (so the discretization tests read them too);
  * the system inputs: bc_values (the evaluated ``combine_boundary_operators_mechanical_stress``), body_force,
    angular_source, mass_source;
  * ``J`` / ``rhs``: the model's ``equation_system.assemble()`` at the zero state, and ``solution``: the state after
    one Newton step of the model's own linear solver from there (the system is linear);
  * ``column_map`` / ``row_map``: the model dof / row of each unknown / equation in the cell-interleaved order
    [u_c, r_c, p_c], from ``dofs_of`` and ``assembled_equation_indices``.

    python tools/make_tpsa_model_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import OUT, grid_arrays, perturb, pp, put_matrix  # noqa: E402
from make_mdflow_golden import put_csr  # noqa: E402
from make_tpsa_golden import KEYS  # noqa: E402


class Geometry:
    def set_domain(self):
        box = {"xmin": 0, "xmax": 1.25, "ymin": 0, "ymax": 1}
        if self.params["tpsa_nd"] == 3:
            box.update(zmin=0, zmax=1)
        self._domain = pp.Domain(box)

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": self.params["cell_size"]}

    def create_mdg(self):
        super().create_mdg()
        if self.params.get("perturb"):
            perturb(self.mdg.subdomains()[0], np.random.default_rng(self.params["seed"]))


class Physics:
    def stiffness_tensor(self, sd):
        rng = np.random.default_rng(self.params["seed"])
        mu = 1.5 * np.exp(0.5 * rng.standard_normal(sd.num_cells))
        mu[sd.cell_centers[0] < 0.5] *= 1e2
        lmbda = 2.0 * np.exp(0.5 * rng.standard_normal(sd.num_cells))
        return pp.FourthOrderTensor(mu, lmbda)

    def body_force(self, subdomains):
        vals = []
        for sd in subdomains:
            f = np.zeros((self.nd, sd.num_cells))
            f[0] = 0.1 * np.sin(3 * sd.cell_centers[1])
            f[self.nd - 1] = -0.2 * (1 + sd.cell_centers[0])
            vals.append(f.ravel("F"))
        return self.volume_integral(pp.wrap_as_dense_ad_array(np.hstack(vals), name="body_force_density"),
                                    subdomains, dim=self.nd)

    def bc_type_mechanics(self, sd):
        """Dirichlet west, a roller south (Dirichlet in y), Robin east (diagonal weights 0.5 .. 3), Neumann elsewhere."""
        s = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, s.west, "dir")
        south = s.south & ~s.west
        bc.is_dir[1, south] = True
        bc.is_neu[1, south] = False
        east = s.east & ~s.south
        bc.is_rob[:, east] = True
        bc.is_neu[:, east] = False
        w = np.zeros((self.nd, self.nd, sd.num_faces))
        rng = np.random.default_rng(self.params["seed"] + 1)
        for i in range(self.nd):
            w[i, i] = rng.uniform(0.5, 3.0, sd.num_faces)
        bc.robin_weight = w
        return bc

    def bc_values_displacement(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[0, s.west] = 0.01 * bg.cell_centers[1, s.west]
        v[self.nd - 1, s.west] = -0.005
        return v.ravel("F")

    def bc_values_stress(self, bg):
        s = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[1, s.north] = -1e-2 * bg.cell_volumes[s.north]
        v[0, s.east] = 5e-3 * bg.cell_volumes[s.east]
        return v.ravel("F")


class Model(Geometry, Physics, pp.models.momentum_balance.TpsaMomentumBalanceMixin, pp.MomentumBalance):
    pass


def interleave(blocks, nd, nr, nc):
    u, r, p = blocks
    out = np.empty((nc, nd + nr + 1), np.int64)
    out[:, :nd] = np.asarray(u).reshape(nc, nd)
    out[:, nd:nd + nr] = np.asarray(r).reshape(nc, nr)
    out[:, nd + nr] = p
    return out.reshape(-1)


def case(name, nd, cell_size, seed, perturbed=False):
    m = Model({"times_to_export": [], "tpsa_nd": nd, "cell_size": cell_size, "seed": seed, "perturb": perturbed})
    m.prepare_simulation()
    es = m.equation_system
    sd = m.mdg.subdomains()[0]
    nc, nf = sd.num_cells, sd.num_faces
    nr = m.rotation_dimension()
    assert np.all(es.get_variable_values(iterate_index=0) == 0)
    J, rhs = es.assemble()
    idx = es.assembled_equation_indices
    data = m.mdg.subdomain_data(sd)
    prm = data[pp.PARAMETERS][m.stress_keyword]
    bc, C = prm["bc"], prm["fourth_order_tensor"]
    mats = data[pp.DISCRETIZATION_MATRICES][m.stress_keyword]

    def ev(op):
        v = es.evaluate(op)
        return np.asarray(getattr(v, "val", v), float)

    def dofs(var):
        return es.dofs_of([v for v in es.variables if v.name == var])
    cols = interleave([dofs(m.displacement_variable), dofs(m.rotation_stress_variable),
                       dofs(m.total_pressure_variable)], nd, nr, nc)
    rows = interleave([idx["momentum_balance_equation"], idx["angular_momentum_balance_equation"],
                       idx["solid_mass_equation"]], nd, nr, nc)
    d = grid_arrays(sd)
    bmask = np.zeros(nf, bool)
    bmask[sd.get_all_boundary_faces()] = True
    d.update(kind=np.array("tpsa"), mu=C.mu, lmbda=C.lmbda, boundary_faces=bmask,
             bc_is_dir=bc.is_dir, bc_is_neu=bc.is_neu, bc_is_rob=bc.is_rob,
             bc_is_internal=np.asarray(bc.is_internal, bool), bc_robin_weight=np.asarray(bc.robin_weight, float),
             bc_basis=np.asarray(bc.basis, float),
             bc_values=ev(m.combine_boundary_operators_mechanical_stress([sd])), body_force=ev(m.body_force([sd])),
             angular_source=np.broadcast_to(ev(m.source_angular_momentum([sd])), (nr * nc,)).copy(),
             mass_source=np.broadcast_to(ev(m.solid_mass_source([sd])), (nc,)).copy(),
             rhs=np.asarray(rhs, float), column_map=cols, row_map=rows)
    for key in KEYS:
        put_matrix(d, key, mats[key])
    put_csr(d, "J", J)
    m.before_nonlinear_loop()
    m.before_nonlinear_iteration()
    m.assemble_linear_system()
    m.after_nonlinear_iteration(m.solve_linear_system())   # linear: one Newton step from zero is the solution
    d["solution"] = es.get_variable_values(iterate_index=0)
    assert np.linalg.norm(d["body_force"]) > 0 and np.linalg.norm(d["bc_values"]) > 0
    assert bc.is_rob.any() and bc.is_dir.any() and bc.is_neu.any()
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print(name, "nc", nc, "dofs", es.num_dofs(), "nnz(J)", J.nnz, f"{os.path.getsize(path) / 1e3:.0f} kB")


CASES = [
    ("tpsa_model_cart2d", 2, 0.125, 201, False),
    ("tpsa_model_cart3d", 3, 0.25, 202, False),
    ("tpsa_model_cart3d_pert", 3, 0.25, 203, True),
]


def main():
    os.makedirs(OUT, exist_ok=True)
    for name, nd, h, seed, pert in CASES:
        case(name, nd, h, seed, pert)


if __name__ == "__main__":
    main()
