"""The TPSA three-field elasticity system (``pb_tpsa_system`` / ``pb_tpsa_rhs``, csrc/tpsa_system.cuh,
``porepy_b200.TpsaElasticity``): the host build and the GPU against a scipy restatement of the model equations and
against the unmodified reference model's Jacobian and right-hand side (fixtures of tools/make_tpsa_model_golden.py),
the block-Jacobi BiCGStab solve, the 4 x 4 and 7 x 7 block inverses, the refusals, and the bench-size mesh."""
import os
import re
import shutil
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.tpsa_elasticity import TpsaElasticity, interleave
from golden_io import case_names, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsa_")
MODEL_CASES = case_names("tpsa_model_")


@pytest.fixture()
def host_build(monkeypatch):
    from emu_tpsa import EmuTpsaFaceGrid
    monkeypatch.setattr(fv, "FaceGrid", EmuTpsaFaceGrid)


def _nr(nd):
    return 3 if nd == 3 else 1


def _field_order(nd, nc):
    """For each cell-interleaved index, the index in the field-wise order [u | r | p]."""
    nr = _nr(nd)
    return interleave([np.arange(nd * nc), nd * nc + np.arange(nr * nc), (nd + nr) * nc + np.arange(nc)], nd, nr, nc)


def _restated(g, mats, mu, lam, bcv, f, sr, sp):
    """A and b of the three equations from the 14 TPSA matrices with scipy, in the cell-interleaved order."""
    nd, nc = g.dim, g.num_cells
    nr = _nr(nd)
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr = sps.kron(div, sps.eye(nd)).tocsr(), sps.kron(div, sps.eye(nr)).tocsr()
    vol = g.cell_volumes
    M = {k: sps.csr_matrix(v) for k, v in mats.items()}
    A = sps.bmat([[-dn @ M["stress"], -dn @ M["stress_rotation"], -dn @ M["stress_total_pressure"]],
                  [dr @ M["rotation_displacement"], dr @ M["rotation_rotation"] - sps.diags(np.repeat(vol / mu, nr)),
                   None],
                  [div @ M["solid_mass_displacement"], None,
                   div @ M["solid_mass_total_pressure"] - sps.diags(vol / lam)]]).tocsr()
    b = np.concatenate([dn @ (M["bound_stress"] @ bcv) + f, -(dr @ (M["bound_rotation_displacement"] @ bcv)) + sr,
                        -(div @ (M["bound_mass_displacement"] @ bcv)) + sp])
    perm = _field_order(nd, nc)
    return A[perm][:, perm].tocsr(), b[perm]


def _seeded_inputs(g, seed):
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.standard_normal(nc))
    return (lam, rng.standard_normal(nd * nf), rng.standard_normal(nd * nc), rng.standard_normal(_nr(nd) * nc),
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


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _scipy(A):
    return A.to_scipy() if hasattr(A, "to_scipy") else sps.csr_matrix(A)


def _check_restatement(name, tol):
    """A and b of the assembly against the scipy restatement built from the matrices pb.Tpsa computes on the same
    face-grid implementation."""
    c = load_case(name)
    lam, bcv, f, sr, sp = _seeded_inputs(c.g, 11)
    prob = _problem(c, lam, bcv, f, sr, sp)
    A, b = prob.assemble()
    A, b = _scipy(A), _host(b)
    C = pb.FourthOrderTensor(c.raw["mu"], lam)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": c.bc})
    pb.Tpsa("mech").discretize(c.g, data)
    Ar, br = _restated(c.g, data[pb.DISCRETIZATION_MATRICES]["mech"], c.raw["mu"], lam, bcv, f, sr, sp)
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
    Am, bm = prob.to_model_order(_scipy(A), _host(b))
    J = sps.csr_matrix((d["J__data"], d["J__indices"], d["J__indptr"]), shape=tuple(d["J__shape"]))
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
    sd = SimpleNamespace(dim=2)
    fake = SimpleNamespace(nd=2, mdg=SimpleNamespace(subdomains=lambda: [sd, sd], interfaces=lambda: []),
                           equation_system=SimpleNamespace(equations={}))
    with pytest.raises(NotImplementedError, match="one subdomain"):
        model_bridge.tpsa_momentum_from_model(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd, SimpleNamespace(dim=1)], interfaces=lambda: [])
    with pytest.raises(NotImplementedError, match="fractures"):
        model_bridge.tpsa_momentum_from_model(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd], interfaces=lambda: [])
    fake.equation_system = SimpleNamespace(equations={"mass_balance_equation": None})
    with pytest.raises(NotImplementedError, match="poromechanics"):
        model_bridge.tpsa_momentum_from_model(fake)


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


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("nd", [2, 3])
def test_bridge_host_build(nd, host_build):
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    prob, cols, rows = plugin(pp).tpsa_momentum_from_model(m)
    J, rhs = m.equation_system.assemble()
    A, b = prob.assemble()
    Am, bm = prob.to_model_order(A, b)
    assert abs(Am - J).max() <= 1e-12 * abs(J).max()
    assert np.abs(bm - rhs).max() <= 1e-12 * np.abs(rhs).max()
    assert np.array_equal(np.sort(cols), np.arange(J.shape[1])) and np.array_equal(np.sort(rows), np.arange(J.shape[0]))


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


# ---- register use of every TPSA kernel of face.cu (compile only) --------------------------------------------------

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


def _kernel_name(mangled):
    """'stem<a, b>' of an Itanium-mangled kernel whose template arguments are ints ('_Z<len><stem>ILi2ELi1EE...')."""
    m = re.match(r"_Z(\d+)", mangled)
    n = int(m.group(1))
    stem, rest = mangled[m.end():m.end() + n], mangled[m.end() + n:]
    args = re.match(r"I((?:Li-?\d+E)+)E", rest)
    return stem + (f"<{', '.join(re.findall(r'Li(-?\d+)E', args.group(1)))}>" if args else "")


def test_tpsa_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-c", os.path.join(ROOT, "porepy_b200", "csrc", "face.cu"),
                          "-o", str(tmp_path / "face.o")], capture_output=True, text=True, check=True)
    seen = set()
    for fn, props in re.findall(r"Function properties for (\S+)\n\s*(.*)", out.stderr):
        if "tpsa" not in fn:
            continue
        name = _kernel_name(fn)
        seen.add(name)
        stack = NB_STACK.get(name, 0)
        assert props.startswith(f"{stack} bytes stack frame, 0 bytes spill stores, 0 bytes spill loads"), (name, props)
    want = {stem + args for stem, all_args in TPSA_KERNELS.items() for args in all_args}
    assert want <= seen, sorted(want - seen)


# ---- GPU ----------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_restatement_and_host_build(name, monkeypatch):
    from emu_tpsa import EmuTpsaFaceGrid
    _check_restatement(name, 1e-13)
    c = load_case(name)
    lam, bcv, f, sr, sp = _seeded_inputs(c.g, 11)
    A, b = _problem(c, lam, bcv, f, sr, sp).assemble()
    A, b = A.to_scipy(), b.cpu().numpy()
    with monkeypatch.context() as mp:
        mp.setattr(fv, "FaceGrid", EmuTpsaFaceGrid)
        Ah, bh = _problem(load_case(name), lam, bcv, f, sr, sp).assemble()
    assert np.array_equal(A.indptr, Ah.indptr) and np.array_equal(A.indices, Ah.indices)
    assert np.abs(A.data - Ah.data).max() <= 1e-13 * np.abs(Ah.data).max()
    assert np.abs(b - bh).max() <= 1e-13 * np.abs(bh).max()


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
    A, b, x = A.to_scipy(), b.cpu().numpy(), x.cpu().numpy()
    assert np.linalg.norm(b - A @ x) <= 1e-11 * np.linalg.norm(b)
    xm = np.empty_like(x)
    xm[prob.column_map] = x
    assert np.linalg.norm(xm - d["solution"]) <= 1e-8 * np.linalg.norm(d["solution"])


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
@pytest.mark.parametrize("bs", [4, 7])
def test_gpu_block_inverse_4_and_7(bs):
    rng = np.random.default_rng(bs)
    nb = 200
    blocks = rng.standard_normal((nb, bs, bs)) + 3 * bs * np.eye(bs)
    blocks[5, 0, 0] = 0.0                                   # pivoting needed, still regular
    A = pb.DeviceCsr(_blocks_csr(blocks, 0.7, rng))
    got = A.block_diagonal_inverse(bs).cpu().numpy().reshape(nb, bs, bs)
    want = np.linalg.inv(blocks)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    sing = blocks.copy()
    sing[7, 1, :] = 0.0                                     # singular block: inverse of its diagonal, 1 where it is 0
    sing[7, 2, :] = sing[7, 3, :]
    got = pb.DeviceCsr(_blocks_csr(sing, 0.7, rng)).block_diagonal_inverse(bs).cpu().numpy().reshape(nb, bs, bs)
    dg = np.diagonal(sing[7])
    assert np.array_equal(got[7], np.diag(np.where(dg != 0, 1.0 / np.where(dg != 0, dg, 1.0), 1.0)))
    assert np.abs(np.delete(got, 7, 0) - np.linalg.inv(np.delete(sing, 7, 0))).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.gpu
def test_gpu_full_size_matches_device_ad_assembly():
    """998,250 tetrahedra with Dirichlet, roller, Robin and Neumann faces and a seeded lambda field: A and b of the new
    kernels against the porepy_b200.ad assembly (device SpGEMM / bmat) of the same pb.Tpsa face matrices, and two
    assemblies bit-identical."""
    import torch
    from porepy_b200 import ad
    from porepy_b200.sparse import DeviceCsr
    from test_tpsa import _full_size_problem
    g, bc, mu = _full_size_problem()
    assert g.num_cells == 998_250
    nd, nc, nf, nr = 3, g.num_cells, g.num_faces, 3
    B, n = 7, 7 * g.num_cells
    lam, bcv, f, sr, sp = _seeded_inputs(g, 23)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
    prob = TpsaElasticity(g, data, "mech", bcv, f, sr, sp)
    A1, b1 = prob.assemble()
    a1 = A1.to_scipy()
    del A1
    prob.discretize()
    A2, b2 = prob.assemble()
    a2 = A2.to_scipy()
    assert np.array_equal(a1.indptr, a2.indptr) and np.array_equal(a1.indices, a2.indices)
    assert np.array_equal(a1.data, a2.data) and torch.equal(b1, b2)
    del a2, A2
    # the same equations on the device AD chain, unknowns numbered cell by cell through the variables' Jacobians
    pb.Tpsa("mech").discretize(g, data)
    M = {k: ad.as_device_csr(v) for k, v in data[pb.DISCRETIZATION_MATRICES]["mech"].items()}
    pos = np.empty(n, np.int64)
    pos[_field_order(nd, nc)] = np.arange(n)             # field-wise dof -> cell-interleaved column
    sizes = [nd * nc, nr * nc, nc]
    starts = np.cumsum([0] + sizes)
    u, r, p = (ad.DeviceAdArray(np.zeros(m), DeviceCsr(sps.csr_matrix(
        (np.ones(m), (np.arange(m), pos[s:s + m])), shape=(m, n)))) for m, s in zip(sizes, starts))
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr, d1 = (DeviceCsr(sps.kron(div, sps.eye(k)).tocsr()) for k in (nd, nr, 1))
    vol = g.cell_volumes
    mom = -(dn @ (M["stress"] @ u + M["stress_rotation"] @ r + M["stress_total_pressure"] @ p
                  + torch.as_tensor(M["bound_stress"] @ bcv, device="cuda"))) - f
    ang = (dr @ (M["rotation_displacement"] @ u + M["rotation_rotation"] @ r
                 + torch.as_tensor(M["bound_rotation_displacement"] @ bcv, device="cuda"))
           + r * (-np.repeat(vol / mu, nr)) - sr)
    mass = (d1 @ (M["solid_mass_displacement"] @ u + M["solid_mass_total_pressure"] @ p
                  + torch.as_tensor(M["bound_mass_displacement"] @ bcv, device="cuda"))
            + p * (-vol / lam) - sp)
    jac, rhs = ad.assemble([mom, ang, mass])
    order = _field_order(nd, nc)
    P = DeviceCsr(sps.csr_matrix((np.ones(n), (np.arange(n), order)), shape=(n, n)))
    ref = P @ jac
    del jac, mom, ang, mass
    diff = ref.axpby(1.0, prob.A, -1.0).to_scipy()
    scale = np.abs(a1.data).max()
    assert np.abs(diff.data).max() <= 1e-13 * scale
    assert a1.nnz == 37 * (nc + 2 * int((np.diff(sps.csr_matrix(g.cell_faces).indptr) == 2).sum()))
    bref = rhs[torch.as_tensor(order, device=rhs.device)]
    assert float((b1 - bref).abs().max()) <= 1e-13 * float(bref.abs().max())


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("nd", [2, 3])
def test_gpu_bridge_solves_stock_model(nd):
    """The stock TPSA model through ``tpsa_momentum_from_model``: A, b equal the model's own Jacobian and right-hand
    side, and the device solve gives the model's solution."""
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    prob, cols, rows = plugin(pp).tpsa_momentum_from_model(m)
    J, rhs = m.equation_system.assemble()
    A, b = prob.assemble()
    Am, bm = prob.to_model_order(A.to_scipy(), b.cpu().numpy())
    assert abs(Am - J).max() <= 1e-12 * abs(J).max()
    assert np.abs(bm - rhs).max() <= 1e-12 * np.abs(rhs).max()
    x, info = prob.solve(tol=1e-12, maxiter=5000)
    assert info["converged"], info
    xm = np.empty(x.numel())
    xm[cols] = x.cpu().numpy()
    import scipy.sparse.linalg as spla
    ref = spla.spsolve(sps.csc_matrix(J), rhs)
    assert np.linalg.norm(xm - ref) <= 1e-8 * np.linalg.norm(ref)
