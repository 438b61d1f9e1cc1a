"""The TPSA three-field elasticity system (``pb_tpsa_system`` / ``pb_tpsa_rhs``, csrc/tpsa_system.cuh,
``porepy_b200.TpsaElasticity``): the host build and the GPU against a scipy restatement of the model equations and
against the unmodified reference model's Jacobian and right-hand side (fixtures of tools/make_tpsa_model_golden.py),
the block-Jacobi BiCGStab solve, the refusals and the bench-size mesh; the block-diagonal inverses of every TPSA block
size (4 to 9), and the register use of every TPSA kernel of face.cu and of the 6 x 6 and 9 x 9 Krylov kernels."""
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.tpsa_elasticity import TpsaElasticity
from golden_io import case_names, load_case
from tpsa_checks import (check_model_order, check_single_grid_refusals, compare_with_host_build, csr, field_order,
                         field_ordered_reference, full_size_problem, host, ptxas_properties, to_model, use_host_build)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsa_")
MODEL_CASES = case_names("tpsa_model_")


@pytest.fixture()
def host_build(monkeypatch):
    use_host_build(monkeypatch, plan=False, sparse=False)


def _divergences(prob):
    div = sps.csr_matrix(prob.sd.cell_faces).T.tocsr()
    return div, sps.kron(div, sps.eye(prob.nd)).tocsr(), sps.kron(div, sps.eye(prob.nr)).tocsr()


def _restated_rhs(prob, mats):
    """b of the three equations of ``prob`` from its inputs and the TPSA boundary matrices with scipy, in the
    cell-interleaved order."""
    div, dn, dr = _divergences(prob)
    M = {k: sps.csr_matrix(mats[k]) for k in ("bound_stress", "bound_rotation_displacement", "bound_mass_displacement")}
    bcv = prob.bc_values
    b = np.concatenate([dn @ (M["bound_stress"] @ bcv) + prob.body_force,
                        -(dr @ (M["bound_rotation_displacement"] @ bcv)) + prob.angular_source,
                        -(div @ (M["bound_mass_displacement"] @ bcv)) + prob.mass_source])
    return b[field_order(prob)]


def _restated(prob, mats):
    """A and b of the three equations of ``prob`` from its inputs and the 14 TPSA matrices with scipy, in the
    cell-interleaved order."""
    div, dn, dr = _divergences(prob)
    vol = prob.sd.cell_volumes
    C = prob.data[pb.PARAMETERS][prob.keyword]["fourth_order_tensor"]
    M = {k: sps.csr_matrix(v) for k, v in mats.items()}
    A = sps.bmat([[-dn @ M["stress"], -dn @ M["stress_rotation"], -dn @ M["stress_total_pressure"]],
                  [dr @ M["rotation_displacement"],
                   dr @ M["rotation_rotation"] - sps.diags(np.repeat(vol / C.mu, prob.nr)), None],
                  [div @ M["solid_mass_displacement"], None,
                   div @ M["solid_mass_total_pressure"] - sps.diags(vol / C.lmbda)]]).tocsr()
    perm = field_order(prob)
    return A[perm][:, perm].tocsr(), _restated_rhs(prob, mats)


def _seeded_inputs(g, seed):
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.standard_normal(nc))
    return (lam, rng.standard_normal(nd * nf), rng.standard_normal(nd * nc), rng.standard_normal((3 if nd == 3 else 1) * nc),
            rng.standard_normal(nc))


def _problem(c, lam=None, bcv=None, f=None, sr=None, sp=None):
    """TpsaElasticity on a fixture's grid, mu and boundary condition (the model's inputs by default)."""
    d = c.raw
    c.g.tags["fracture_faces"] = np.asarray(d["fracture_faces"], bool)
    lam = d["lmbda"] if lam is None else lam
    C = pb.FourthOrderTensor(d["mu"], lam)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": c.bc})
    if bcv is None:
        bcv, f, sr, sp = d["bc_values"], d["body_force"], d["angular_source"], d["mass_source"]
    return TpsaElasticity(c.g, data, "mech", bcv, f, sr, sp)


def _scipy(A):
    return A.to_scipy() if hasattr(A, "to_scipy") else sps.csr_matrix(A)


def _check_restatement(name, tol):
    """A and b of the assembly against the scipy restatement built from the matrices pb.Tpsa computes on the same
    face-grid implementation."""
    c = load_case(name)
    lam, bcv, f, sr, sp = _seeded_inputs(c.g, 11)
    prob = _problem(c, lam, bcv, f, sr, sp)
    A, b = prob.assemble()
    A, b = _scipy(A), host(b)
    C = pb.FourthOrderTensor(c.raw["mu"], lam)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": c.bc})
    pb.Tpsa("mech").discretize(c.g, data)
    Ar, br = _restated(prob, data[pb.DISCRETIZATION_MATRICES]["mech"])
    assert A.shape == Ar.shape
    nd = c.g.dim
    assert A.nnz == (37 if nd == 3 else 12) * (c.g.num_cells + 2 * int((np.diff(sps.csr_matrix(c.g.cell_faces).indptr)
                                                                      == 2).sum()))
    assert abs(A - Ar).max() <= tol * abs(Ar).max(), name
    assert np.abs(b - br).max() <= tol * np.abs(br).max(), name


def _check_model(name, tol):
    c = load_case(name)
    d = c.raw
    prob = _problem(c)
    prob.column_map, prob.row_map = d["column_map"], d["row_map"]
    A, b = prob.assemble()
    Am, bm = prob.to_model_order(_scipy(A), host(b))
    J = csr(d, "J")
    assert abs(Am - J).max() <= tol * abs(J).max(), name
    assert np.abs(bm - d["rhs"]).max() <= tol * np.abs(d["rhs"]).max(), name


def test_model_fixtures_present():
    assert len(MODEL_CASES) >= 3, MODEL_CASES
    dims = {int(load_case(n).raw["dim"]) for n in MODEL_CASES}
    assert dims == {2, 3}


@pytest.mark.parametrize("name", CASES)
def test_host_build_matches_restatement(name, host_build):
    _check_restatement(name, 1e-14)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_host_build_matches_reference_model(name, host_build):
    _check_model(name, 1e-12)


def test_refusals_host():
    g1 = SimpleNamespace(dim=1, num_cells=2, num_faces=3)
    with pytest.raises(NotImplementedError, match="only implemented for 2d and 3d"):
        TpsaElasticity(g1, {}, "mech", np.zeros(3))
    g = pb.cart_grid_2d([3, 2])
    with pytest.raises(ValueError, match="bc_values must have"):
        TpsaElasticity(g, {}, "mech", np.zeros(g.num_faces))
    with pytest.raises(ValueError, match="body_force must have"):
        TpsaElasticity(g, {}, "mech", np.zeros(2 * g.num_faces), body_force=np.zeros(3))
    with pytest.raises(ValueError, match="no dof maps"):
        TpsaElasticity(g, {}, "mech", np.zeros(2 * g.num_faces)).to_model_order(sps.eye(4 * g.num_cells))
    from porepy_b200 import model_bridge
    check_single_grid_refusals(model_bridge.tpsa_momentum_from_model, model_bridge.tpsa_momentum_from_model,
                               ["mass_balance_equation"], "poromechanics")


# ---- the stock model through the plugin's bridge -----------------------------------------------------------------


class _Square:
    def set_domain(self):
        import porepy as pp
        box = {"xmin": 0, "xmax": 1, "ymin": 0, "ymax": 1}
        if self.params.get("tpsa_nd", 2) == 3:
            box.update(zmin=0, zmax=1)
        self._domain = pp.Domain(box)

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": 0.25}

    def stiffness_tensor(self, sd):
        import porepy as pp
        rng = np.random.default_rng(5)
        return pp.FourthOrderTensor(np.exp(rng.standard_normal(sd.num_cells)),
                                    np.exp(rng.standard_normal(sd.num_cells)))

    def bc_type_mechanics(self, sd):
        import porepy as pp
        sides = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, sides.west, "dir")
        bc.is_dir[1, sides.south] = True
        bc.is_neu[1, sides.south] = False
        return bc

    def bc_values_stress(self, bg):
        sides = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[1, sides.north] = -1e-3 * bg.cell_volumes[sides.north]
        return v.ravel("F")


def _stock_model(pp, nd):
    class Stock(_Square, pp.models.momentum_balance.TpsaMomentumBalanceMixin, pp.MomentumBalance):
        pass
    m = Stock({"times_to_export": [], "tpsa_nd": nd})
    m.prepare_simulation()
    return m


def _check_bridge(nd):
    """The stock model through ``tpsa_momentum_from_model``: A and b equal the model's own Jacobian and right-hand
    side.  Returns the problem, the model's Jacobian and right-hand side."""
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    prob, cols, rows = plugin(pp).tpsa_momentum_from_model(m)
    J, rhs = m.equation_system.assemble()
    check_model_order(prob, *prob.assemble(), J, rhs, cols, rows)
    return prob, J, rhs


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("nd", [2, 3])
def test_bridge_host_build(nd, host_build):
    _check_bridge(nd)


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
def test_bridge_refuses_tpsa_poromechanics():
    from test_porepy_plugin import _FlowBC
    from porepy_b200 import model_bridge
    pp = load_porepy()

    class Poro(_Square, _FlowBC, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Poromechanics):
        pass
    m = Poro({"times_to_export": []})
    m.prepare_simulation()
    with pytest.raises(NotImplementedError, match="poromechanics"):
        model_bridge.tpsa_momentum_from_model(m)


# ---- register use (compile only) ----------------------------------------------------------------------------------

_ND = ["<2>", "<3>"]
_ND_NS = [f"<{nd}, {ns}>" for nd in (2, 3) for ns in (1, 2)]
TPSA_KERNELS = {
    "tpsa_kernel": _ND, "tpsa_nb_count_kernel": [""], "tpsa_nb_list_kernel": [""], "tpsa_pattern_kernel": _ND,
    "tpsa_system_kernel": _ND, "tpsa_rhs_kernel": [f"<{nd}, {ns}>" for nd in (2, 3) for ns in (0, 1, 2)],
    "tpsa_poro_count_kernel": _ND_NS, "tpsa_poro_pattern_kernel": _ND_NS, "tpsa_poro_system_kernel": _ND_NS,
    "tpsa_poro_fluid_kernel": _ND_NS, "tpsa_contact_count_kernel": _ND, "tpsa_contact_pattern_kernel": _ND,
    "tpsa_contact_iface_pattern_kernel": _ND, "tpsa_contact_block_kernel": _ND, "tpsa_contact_iface_kernel": _ND,
    "tpsa_contact_law_kernel": _ND,
}
# the kernels that enumerate the face neighbours of a cell hold them in a kTpsaMaxNb = 32 int32 array on the stack
NB_STACK = {"tpsa_nb_count_kernel": 128, "tpsa_nb_list_kernel": 128}
# the block sizes of the thermo-poromechanics systems (6 in 2-D, 9 in 3-D)
KRYLOV_KERNELS = re.compile(r"(block_diag_inv_inplace|kry_[ps])_kernel<[69]>")


def test_tpsa_kernels_do_not_spill(tmp_path):
    seen = set()
    for name, props in ptxas_properties("face.cu", tmp_path).items():
        if "tpsa" not in name:
            continue
        seen.add(name)
        stack = NB_STACK.get(name, 0)
        assert props.startswith(f"{stack} bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"), (name, props)
    want = {stem + args for stem, all_args in TPSA_KERNELS.items() for args in all_args}
    assert want <= seen, sorted(want - seen)


def test_krylov_kernels_do_not_spill(tmp_path):
    seen = []
    for name, props in ptxas_properties("krylov.cu", tmp_path).items():
        if KRYLOV_KERNELS.fullmatch(name):
            seen.append(name)
            assert props.startswith("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"), (name, props)
    assert len(seen) == 6, seen


# ---- GPU ----------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_restatement_and_host_build(name):
    _check_restatement(name, 1e-13)
    c = load_case(name)
    inputs = _seeded_inputs(c.g, 11)
    A, b = _problem(c, *inputs).assemble()
    compare_with_host_build(lambda: [_problem(load_case(name), *inputs).assemble()], [(A.to_scipy(), host(b))],
                            same_pattern=True, plan=False, sparse=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODEL_CASES)
def test_gpu_matches_reference_model(name):
    _check_model(name, 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODEL_CASES)
def test_gpu_solve_matches_reference_solution(name):
    c = load_case(name)
    d = c.raw
    prob = _problem(c)
    prob.column_map, prob.row_map = d["column_map"], d["row_map"]
    x, info = prob.solve(tol=1e-12, maxiter=5000)
    assert info["converged"] and info.get("fused"), info
    A, b = prob.assemble()
    A, b = A.to_scipy(), b.cpu().numpy()
    assert np.linalg.norm(b - A @ host(x)) <= 1e-11 * np.linalg.norm(b)
    assert np.linalg.norm(to_model(prob, x) - d["solution"]) <= 1e-8 * np.linalg.norm(d["solution"])


@pytest.mark.gpu
def test_gpu_refusals():
    c = load_case(MODEL_CASES[0])
    lam = c.raw["lmbda"].copy()
    for bad in (0.0, -1.0, np.nan, np.inf):
        lam[3] = bad
        with pytest.raises(ValueError, match="first Lame parameter"):
            _problem(c, lam).discretize()
    mu = c.raw["mu"].copy()
    mu[0] = 0.0
    c.raw["mu"] = mu
    with pytest.raises(ValueError, match="shear modulus"):
        _problem(c).discretize()
    c = load_case(MODEL_CASES[0])
    g = c.g
    fg = fv.FaceGrid(g)
    with pytest.raises(ValueError, match="has not been called"):
        fg.tpsa_rhs(4 * g.num_cells, np.zeros(2 * g.num_faces))
    codes, rob = fv.tpsa_bc_arrays(c.bc, 2, g.num_faces)
    flags = np.zeros(g.num_faces, np.uint8)
    flags[g.get_all_boundary_faces()] = 1
    args = (c.raw["mu"], c.raw["lmbda"], g.cell_volumes, codes, rob, flags, g.face_areas)
    with pytest.raises(ValueError, match="only implemented for 2d and 3d"):
        fg.tpsa_system(1, *args)
    with pytest.raises(ValueError, match="Robin faces need robin_diag"):
        fg.tpsa_system(2, *args[:4], None, *args[5:])
    inner = np.flatnonzero(np.diff(sps.csr_matrix(g.cell_faces).indptr) == 2)[0]
    bad_flags = flags.copy()
    bad_flags[inner] = 1
    with pytest.raises(ValueError, match="sign of internal faces"):
        fg.tpsa_system(2, *args[:5], bad_flags, args[6])


def _blocks_csr(blocks, noise, rng):
    """Block-diagonal matrix of the given blocks plus off-block entries (which the inverse must ignore)."""
    nb, bs = blocks.shape[0], blocks.shape[1]
    A = sps.block_diag(list(blocks), format="csr")
    off = sps.random(nb * bs, nb * bs, density=min(1.0, 4.0 / bs / nb), random_state=rng.integers(1 << 30)).tocsr()
    mask = (off.nonzero()[0] // bs) != (off.nonzero()[1] // bs)
    r, c = off.nonzero()
    return (A + noise * sps.csr_matrix((np.ones(mask.sum()), (r[mask], c[mask])), shape=A.shape)).tocsr()


@pytest.mark.gpu
@pytest.mark.parametrize("bs", [4, 5, 6, 7, 8, 9])
def test_gpu_block_inverse(bs):
    """The block-diagonal inverse of every TPSA block size (elasticity 4 / 7, poromechanics 5 / 8, thermo-poromechanics
    6 / 9) against numpy, with blocks that need a pivot swap at some or every step and a singular block."""
    rng = np.random.default_rng(bs)
    nb = 300
    blocks = rng.standard_normal((nb, bs, bs)) + 3 * bs * np.eye(bs)
    blocks[5, 0, 0] = 0.0                                    # pivoting needed, still regular
    blocks[6] = blocks[6][rng.permutation(bs)]                # every row swapped
    blocks[8] = blocks[8][::-1]                               # anti-diagonal dominant: a swap at every step
    A = pb.DeviceCsr(_blocks_csr(blocks, 0.7, rng))
    got = A.block_diagonal_inverse(bs).cpu().numpy().reshape(nb, bs, bs)
    want = np.linalg.inv(blocks)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    sing = blocks.copy()
    sing[7, 1, :] = 0.0                                      # singular block: inverse of its diagonal, 1 where it is 0
    sing[7, 2, :] = sing[7, 3, :]
    got = pb.DeviceCsr(_blocks_csr(sing, 0.7, rng)).block_diagonal_inverse(bs).cpu().numpy().reshape(nb, bs, bs)
    dg = np.diagonal(sing[7])
    assert np.array_equal(got[7], np.diag(np.where(dg != 0, 1.0 / np.where(dg != 0, dg, 1.0), 1.0)))
    assert np.abs(np.delete(got, 7, 0) - np.linalg.inv(np.delete(sing, 7, 0))).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.gpu
def test_gpu_full_size_matches_device_ad_assembly():
    """998,250 tetrahedra with Dirichlet, roller, Robin and Neumann faces and a seeded lambda field: A of the new kernels
    against the field-ordered porepy_b200.ad bmat assembly (device SpGEMM) of the same pb.Tpsa face matrices, b against
    their scipy restatement, and two assemblies bit-identical."""
    import torch
    prob, _ = full_size_problem("elasticity", 23)
    g = prob.sd
    assert g.num_cells == 998_250
    A1, b1 = prob.assemble()
    a1 = A1.to_scipy()
    del A1
    prob.discretize()
    A2, b2 = prob.assemble()
    a2 = A2.to_scipy()
    assert np.array_equal(a1.indptr, a2.indptr) and np.array_equal(a1.indices, a2.indices)
    assert np.array_equal(a1.data, a2.data) and torch.equal(b1, b2)
    del a2, A2
    pb.Tpsa("mech").discretize(g, prob.data)
    mats = prob.data[pb.DISCRETIZATION_MATRICES]["mech"]
    diff = field_ordered_reference(prob, mats, []).axpby(1.0, prob.A, -1.0).to_scipy()
    assert np.abs(diff.data).max() <= 1e-13 * np.abs(a1.data).max()
    assert a1.nnz == 37 * (g.num_cells + 2 * int((np.diff(sps.csr_matrix(g.cell_faces).indptr) == 2).sum()))
    bref = _restated_rhs(prob, mats)
    assert np.abs(host(b1) - bref).max() <= 1e-13 * np.abs(bref).max()


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("nd", [2, 3])
def test_gpu_bridge_solves_stock_model(nd):
    """The stock TPSA model through ``tpsa_momentum_from_model``: A, b equal the model's own Jacobian and right-hand
    side, and the device solve gives the model's solution."""
    import scipy.sparse.linalg as spla
    prob, J, rhs = _check_bridge(nd)
    x, info = prob.solve(tol=1e-12, maxiter=5000)
    assert info["converged"], info
    ref = spla.spsolve(sps.csc_matrix(J), rhs)
    assert np.linalg.norm(to_model(prob, x) - ref) <= 1e-8 * np.linalg.norm(ref)
