"""TPSA poromechanics (``porepy_b200.TpsaPoromechanics``, ``pb_tpsa_poro_system`` / ``pb_tpsa_poro_fluid_rows``,
csrc/tpsa_system.cuh) against the unmodified reference's ``pp.Poromechanics`` + ``TpsaPoromechanicsMixin``: Jacobian and
-R at the zero state and at an intermediate Newton iterate of two time steps, the residual histories and converged
states (fixtures of tools/make_tpsa_poromech_golden.py), a live stock model through the bridge, the refusals, the 5 x 5
and 8 x 8 block inverses and the bench-size mesh.
CPU: host build of tpsa_system.cuh + the scipy stand-in for the device sparse algebra."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.tpsa_poromech import TpsaPoromechanics
from golden_io import case_names, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsaporo_")


def _csr(d, key):
    return sps.csr_matrix((d[key + "__data"], d[key + "__indices"], d[key + "__indptr"]), shape=tuple(d[key + "__shape"]))


def _scalar_bc(d, prefix, nf):
    return SimpleNamespace(is_dir=d[prefix + "_is_dir"], is_neu=d[prefix + "_is_neu"], is_rob=np.zeros(nf, bool),
                           is_internal=np.zeros(nf, bool), robin_weight=np.ones(nf), bc_type="scalar", num_faces=nf)


def _problem(name):
    c = load_case(name)
    d, g = c.raw, c.g
    nf = g.num_faces
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(d["K"]),
                                           "bc": _scalar_bc(d, "flow", nf)})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(d["mu"], d["lmbda"]),
                                           "bc": c.bc})
    fluid = {k: float(d[k]) for k in ("compressibility", "density", "viscosity", "reference_pressure")}
    solid = {k: float(d[k]) for k in ("reference_porosity", "biot_coefficient", "bulk_modulus")}
    prob = TpsaPoromechanics(g, data, fluid, solid, d["flow_bc_values"], d["bc_values"], _scalar_bc(d, "ff", nf),
                             d["ff_values"], body_force=d["body_force"], angular_source=d["angular_source"],
                             mass_source=d["mass_source"], fluid_source=d["fluid_source"])
    prob.column_map, prob.row_map = d["column_map"], d["row_map"]
    return prob, d


def _to_solver(prob, xm):
    """A state of the model's dof order in the problem's cell-interleaved order."""
    return np.asarray(xm)[prob.column_map]


def _states(d):
    """(label, x, x_prev, J key, rhs key) of the stored linearizations."""
    out = [("zero", d["s0_previous"], d["s0_previous"], "J0", "rhs0")]
    for s in range(2):
        out.append((f"step {s}", d[f"s{s}_iterate"], d[f"s{s}_previous"], f"s{s}_J", f"s{s}_rhs"))
    return out


def _host(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def check_linearizations(prob, d, tol):
    prob.discretize()
    got = []
    for label, x, xp, jk, rk in _states(d):
        J, rhs = prob.linearize(_to_solver(prob, x), _to_solver(prob, xp), float(d["dt"]))
        Jm, bm = prob.to_model_order(J.to_scipy(), _host(rhs))
        Jr, br = _csr(d, jk), d[rk]
        assert abs(Jm - Jr).max() <= tol * abs(Jr).max(), label
        assert np.abs(bm - br).max() <= tol * np.abs(br).max(), label
        got.append((J.to_scipy(), _host(rhs).copy()))
    assert int(prob._missing.sum()) == 0
    return got


def check_time_steps(prob, d, tol, linear_solver=None, linear_tol=1e-13):
    for s in range(2):
        x, hist = prob.time_step(_to_solver(prob, d[f"s{s}_previous"]), float(d["dt"]), tol=1e-13,
                                 linear_solver=linear_solver, linear_tol=linear_tol)
        ref = d[f"s{s}_residual_norms"]
        mine = np.array([h["residual"] for h in hist])
        assert len(mine) == len(ref), (mine, ref)
        assert np.abs(mine - ref).max() <= tol * ref[0], (mine, ref)
        xm = np.empty(prob.num_dofs)
        xm[prob.column_map] = _host(x)
        sol = d[f"s{s}_solution"]
        assert np.linalg.norm(xm - sol) <= tol * np.linalg.norm(sol), s


@pytest.fixture()
def host_build(monkeypatch):
    import emu_sparse
    from emu_binding import EmuBackedPlan
    from emu_tpsa import EmuTpsaFaceGrid
    monkeypatch.setattr(fv, "DevicePlan", EmuBackedPlan)
    monkeypatch.setattr(fv, "FaceGrid", EmuTpsaFaceGrid)
    emu_sparse.install(monkeypatch)


def _direct(J, rhs):
    import torch
    return torch.as_tensor(spla.spsolve(J.to_scipy().tocsc(), _host(rhs)))


def test_fixtures_present():
    assert {int(load_case(n).raw["dim"]) for n in CASES} == {2, 3}


@pytest.mark.parametrize("name", CASES)
def test_host_build_matches_reference(name, host_build):
    prob, d = _problem(name)
    check_linearizations(prob, d, 1e-12)
    check_time_steps(prob, d, 1e-10, linear_solver=_direct)


def test_refusals_host():
    g1 = SimpleNamespace(dim=1, num_cells=2, num_faces=3)
    fluid = dict(compressibility=0.1, density=1.0, viscosity=1.0)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.5, bulk_modulus=2.0)
    with pytest.raises(NotImplementedError, match="only implemented for 2d and 3d"):
        TpsaPoromechanics(g1, {}, fluid, solid, np.zeros(3), np.zeros(3), None, np.zeros(3))
    g = pb.cart_grid_2d([3, 2])
    nf = g.num_faces
    args = (np.zeros(nf), np.zeros(2 * nf), None, np.zeros(nf))
    for k in ("compressibility", "density", "viscosity"):
        for bad in (0.0, -1.0, np.nan):
            with pytest.raises(ValueError, match="must be finite and > 0"):
                TpsaPoromechanics(g, {}, dict(fluid, **{k: bad}), solid, *args)
    for bad in (np.nan, np.inf):
        with pytest.raises(ValueError, match="Biot coefficient"):
            TpsaPoromechanics(g, {}, fluid, dict(solid, biot_coefficient=bad), *args)
    with pytest.raises(ValueError, match="mech_bc_values must have"):
        TpsaPoromechanics(g, {}, fluid, solid, np.zeros(nf), np.zeros(nf), None, np.zeros(nf))
    with pytest.raises(ValueError, match="no dof maps"):
        TpsaPoromechanics(g, {}, fluid, solid, *args).to_model_order(sps.eye(5 * g.num_cells))
    from porepy_b200 import model_bridge
    sd = SimpleNamespace(dim=2)
    fake = SimpleNamespace(nd=2, mdg=SimpleNamespace(subdomains=lambda: [sd, sd], interfaces=lambda: []),
                           equation_system=SimpleNamespace(equations={}))
    with pytest.raises(NotImplementedError, match="one subdomain"):
        model_bridge.tpsa_poromechanics_from_model(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd, SimpleNamespace(dim=1)], interfaces=lambda: [])
    with pytest.raises(NotImplementedError, match="fractures"):
        model_bridge.tpsa_poromechanics_from_model(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd], interfaces=lambda: [])
    fake.equation_system = SimpleNamespace(equations={"mass_balance_equation": None})
    with pytest.raises(NotImplementedError, match="tpsa_poromechanics_from_model"):
        model_bridge.tpsa_momentum_from_model(fake)


# ---- the stock model through the plugin's bridge -----------------------------------------------------------------


def _stock_model(pp, nd):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_tpsa_poromech_golden import Setup

    class Stock(Setup, pp.models.poromechanics.TpsaPoromechanicsMixin, pp.Poromechanics):
        pass
    fluid = pp.FluidComponent(compressibility=0.02, viscosity=0.7, density=1.1)
    solid = pp.SolidConstants(porosity=0.15, biot_coefficient=0.6, lame_lambda=1.5, shear_modulus=1.0, permeability=2.0)
    m = Stock({"times_to_export": [], "tpsa_nd": nd, "cell_size": 0.25, "seed": 9,
               "material_constants": {"fluid": fluid, "solid": solid},
               "reference_variable_values": pp.ReferenceVariableValues(pressure=0.1)})
    m.prepare_simulation()
    rng = np.random.default_rng(nd)
    x = 0.1 * rng.standard_normal(m.equation_system.num_dofs())
    m.equation_system.set_variable_values(x, iterate_index=0)
    m.equation_system.set_variable_values(0.5 * x, time_step_index=0)
    m.update_derived_quantities()         # upwind directions of the iterate, as after a Newton update
    return m


def _check_bridge(nd, to_host):
    from porepy_b200.porepy_plugin import plugin
    pp = load_porepy()
    m = _stock_model(pp, nd)
    es = m.equation_system
    prob, cols, rows = plugin(pp).tpsa_poromechanics_from_model(m)
    J, rhs = es.assemble()
    x, xp = es.get_variable_values(iterate_index=0), es.get_variable_values(time_step_index=0)
    A, b = prob.linearize(x[cols], xp[cols], float(m.time_manager.dt))
    Am, bm = prob.to_model_order(A.to_scipy(), to_host(b))
    assert abs(Am - J).max() <= 1e-12 * abs(J).max()
    assert np.abs(bm - rhs).max() <= 1e-12 * np.abs(rhs).max()
    assert np.array_equal(np.sort(cols), np.arange(J.shape[1])) and np.array_equal(np.sort(rows), np.arange(J.shape[0]))


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("nd", [2, 3])
def test_bridge_host_build(nd, host_build):
    _check_bridge(nd, _host)


# ---- GPU ----------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_reference_and_host_build(name, monkeypatch):
    prob, d = _problem(name)
    dev = check_linearizations(prob, d, 1e-12)
    check_time_steps(prob, d, 1e-10, linear_solver=lambda J, rhs: _direct(J, rhs).to(rhs.device))
    with monkeypatch.context() as mp:
        import emu_sparse
        from emu_binding import EmuBackedPlan
        from emu_tpsa import EmuTpsaFaceGrid
        mp.setattr(fv, "DevicePlan", EmuBackedPlan)
        mp.setattr(fv, "FaceGrid", EmuTpsaFaceGrid)
        emu_sparse.install(mp)
        ph, _ = _problem(name)
        host = check_linearizations(ph, d, 1e-12)
    # -R near convergence is b0 - A x with cancellation: its round-off is measured on the scale of -R at the zero state
    rscale = np.abs(host[0][1]).max()
    for (A, b), (Ah, bh) in zip(dev, host):
        # the device SpGEMM keeps exact cancellations of div @ flux in the fluid-row pattern, scipy drops them
        assert abs(A - Ah).max() <= 1e-13 * abs(Ah).max()
        assert np.abs(b - bh).max() <= 1e-13 * rscale


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_newton_with_block_jacobi(name):
    """The Newton loop with the device block-Jacobi BiCGStab reproduces the reference's converged states."""
    prob, d = _problem(name)
    prob.discretize()
    for s in range(2):
        x, hist = prob.time_step(_to_solver(prob, d[f"s{s}_previous"]), float(d["dt"]), tol=1e-12, linear_tol=1e-13)
        assert all(h.get("linear_converged", True) for h in hist), hist
        xm = np.empty(prob.num_dofs)
        xm[prob.column_map] = _host(x)
        sol = d[f"s{s}_solution"]
        assert np.linalg.norm(xm - sol) <= 1e-8 * np.linalg.norm(sol), (s, hist)


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("nd", [2, 3])
def test_gpu_bridge(nd):
    _check_bridge(nd, _host)


@pytest.mark.gpu
def test_gpu_refusals():
    import torch
    prob, d = _problem(CASES[0])
    prob.discretize()
    g, fg = prob.sd, prob._fg
    nc = g.num_cells
    codes, rob = fv.tpsa_bc_arrays(prob.data[pb.PARAMETERS]["mechanics"]["bc"], 2, g.num_faces)
    flags = np.zeros(g.num_faces, np.uint8)
    flags[g.get_all_boundary_faces()] = 1
    fp = prob._operands().div.matmul(prob._operands().flux)
    args = [d["mu"], d["lmbda"], np.full(nc, 0.5), g.cell_volumes, codes, rob, flags, g.face_areas, fp]
    for i, what in ((1, "first Lame parameter"), (2, "Biot coefficient")):
        bad = np.array(args[i], float)
        bad[3] = np.nan
        with pytest.raises(ValueError, match=what):
            fg.tpsa_poro_system(2, *args[:i], bad, *args[i + 1:])
    with pytest.raises(ValueError, match="only implemented for 2d and 3d"):
        fg.tpsa_poro_system(1, *args)
    with pytest.raises(ValueError, match="flux pattern"):
        fg.tpsa_poro_system(2, *args[:-1], pb.DeviceCsr(sps.eye(nc + 1, format="csr")))
    b = torch.zeros(prob.num_dofs, dtype=torch.float64, device="cuda")
    r = torch.zeros(nc, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="num_cells x 2 num_cells"):
        fg.tpsa_poro_fluid_rows(prob.A, pb.DeviceCsr(sps.eye(nc, format="csr")), r, b)
    with pytest.raises(ValueError, match="not the TPSA poromechanics system"):
        fg.tpsa_poro_fluid_rows(pb.DeviceCsr(sps.eye(prob.num_dofs, format="csr")),
                                pb.DeviceCsr(sps.csr_matrix((nc, 2 * nc))), r, b)


def _blocks_csr(blocks, noise, rng):
    nb, bs = blocks.shape[0], blocks.shape[1]
    A = sps.block_diag(list(blocks), format="csr")
    off = sps.random(nb * bs, nb * bs, density=min(1.0, 4.0 / bs / nb), random_state=rng.integers(1 << 30)).tocsr()
    r, c = off.nonzero()
    mask = (r // bs) != (c // bs)
    return (A + noise * sps.csr_matrix((np.ones(mask.sum()), (r[mask], c[mask])), shape=A.shape)).tocsr()


@pytest.mark.gpu
@pytest.mark.parametrize("bs", [5, 8])
def test_gpu_block_inverse_5_and_8(bs):
    rng = np.random.default_rng(bs)
    nb = 300
    blocks = rng.standard_normal((nb, bs, bs)) + 3 * bs * np.eye(bs)
    blocks[5, 0, 0] = 0.0                                    # pivoting needed, still regular
    blocks[6] = blocks[6][rng.permutation(bs)]                # every row swapped
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


def full_size_problem(seed=29):
    """998,250 tetrahedra (the TPSA bench mesh) with seeded coefficients and boundary data: Dirichlet, roller, Robin and
    Neumann mechanical faces, Dirichlet pressure on two sides."""
    from test_tpsa import _full_size_problem
    g, bc, mu = _full_size_problem()
    nc, nf = g.num_cells, g.num_faces
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.standard_normal(nc))
    K = pb.SecondOrderTensor(np.exp(0.5 * rng.standard_normal(nc)))
    bf = np.asarray(g.get_all_boundary_faces(), np.int64)
    x = g.face_centers[0, bf]
    dirf = bf[(x < x.min() + 1e-9) | (x > x.max() - 1e-9)]
    is_dir = np.zeros(nf, bool)
    is_dir[dirf] = True
    is_neu = np.zeros(nf, bool)
    is_neu[bf] = True
    is_neu[dirf] = False
    fbc = SimpleNamespace(is_dir=is_dir, is_neu=is_neu, is_rob=np.zeros(nf, bool), is_internal=np.zeros(nf, bool),
                          robin_weight=np.ones(nf), bc_type="scalar", num_faces=nf)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": K, "bc": fbc})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
    flow_bc = np.where(is_dir, rng.random(nf), 0.0)
    fluid = dict(compressibility=0.05, density=1.7, viscosity=1.3, reference_pressure=0.3)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.7, bulk_modulus=3.0)
    prob = TpsaPoromechanics(g, data, fluid, solid, flow_bc, rng.standard_normal(3 * nf), fbc,
                             np.where(is_dir, 1.7 / 1.3, 0.0), body_force=rng.standard_normal(3 * nc),
                             fluid_source=rng.standard_normal(nc) * g.cell_volumes)
    return prob, rng


@pytest.mark.gpu
def test_gpu_full_size_matches_device_ad_assembly():
    """998,250 tetrahedra, seeded inputs: J of the second linearization of a time step against the field-ordered
    porepy_b200.ad bmat assembly of the same matrices (mechanics rows from pb.Tpsa, fluid rows from the AD chain) permuted
    to the cell-interleaved order; two linearizations bit-identical."""
    import torch
    from porepy_b200 import ad
    from porepy_b200.sparse import DeviceCsr
    prob, rng = full_size_problem()
    g = prob.sd
    nc, nd, nr, B = g.num_cells, 3, 3, 8
    n = B * nc
    assert nc == 998_250
    prob.discretize()
    x_prev = torch.as_tensor(0.1 * rng.standard_normal(n), device="cuda")
    x = x_prev + torch.as_tensor(0.01 * rng.standard_normal(n), device="cuda")
    prob.linearize(x_prev, x_prev, 0.25)
    J1, r1 = prob.linearize(x, x_prev, 0.25)
    a1, r1 = J1.to_scipy(), r1.clone()
    J2, r2 = prob.linearize(x, x_prev, 0.25)
    a2 = J2.to_scipy()
    assert np.array_equal(a1.indptr, a2.indptr) and np.array_equal(a1.indices, a2.indices)
    assert np.array_equal(a1.data, a2.data) and torch.equal(r1, r2)
    assert int(prob._missing.sum()) == 0
    del a2
    # field-ordered reference: blocks [u | r | p_t | p] x [u | r | p_t | p]
    data = prob.data
    pb.Tpsa("mechanics").discretize(g, data)
    M = {k: ad.as_device_csr(v) for k, v in data[pb.DISCRETIZATION_MATRICES]["mechanics"].items()}
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr, d1 = (DeviceCsr(sps.kron(div, sps.eye(k)).tocsr()) for k in (nd, nr, 1))
    vol = g.cell_volumes
    lam = np.asarray(data[pb.PARAMETERS]["mechanics"]["fourth_order_tensor"].lmbda)
    mu = np.asarray(data[pb.PARAMETERS]["mechanics"]["fourth_order_tensor"].mu)

    def diag(v):
        return DeviceCsr(sps.diags(v).tocsr())
    eq = prob.fluid_equation(x, x_prev, 0.25)
    jf = eq.jac
    Jpt = DeviceCsr(jf.to_scipy()[:, :nc])
    Jp = DeviceCsr(jf.to_scipy()[:, nc:])
    ref = DeviceCsr.bmat([
        [-(dn @ M["stress"]), -(dn @ M["stress_rotation"]), -(dn @ M["stress_total_pressure"]), None],
        [dr @ M["rotation_displacement"], (dr @ M["rotation_rotation"]) - diag(np.repeat(vol / mu, nr)), None, None],
        [d1 @ M["solid_mass_displacement"], None, (d1 @ M["solid_mass_total_pressure"]) - diag(vol / lam),
         diag(-vol * prob.alpha / lam)],
        [None, None, Jpt, Jp]])
    order = np.empty((nc, B), np.int64)
    order[:, :nd] = np.arange(nd * nc).reshape(nc, nd)
    order[:, nd:nd + nr] = nd * nc + np.arange(nr * nc).reshape(nc, nr)
    order[:, 6] = (nd + nr) * nc + np.arange(nc)
    order[:, 7] = (nd + nr + 1) * nc + np.arange(nc)
    order = order.reshape(-1)
    P = DeviceCsr(sps.csr_matrix((np.ones(n), (np.arange(n), order)), shape=(n, n)))
    refp = (P @ ref) @ DeviceCsr(sps.csr_matrix((np.ones(n), (order, np.arange(n))), shape=(n, n)))
    diff = refp.axpby(1.0, J1, -1.0).to_scipy()
    assert np.abs(diff.data).max() <= 1e-13 * np.abs(a1.data).max()
