"""Restarted GMRES with the grouped block-Jacobi preconditioner (porepy_b200/csrc/gmres.cu, ``krylov.gmres``): the device
solve of the Newton updates of the fractured contact models (``preconditioner_groups()`` of ``FracturedMomentumBalance``,
``FracturedPoromechanics`` and ``FracturedThermoporomechanics``).
CPU: the model groups on the stored Jacobians of the eight contact fixtures, scipy's GMRES with the same preconditioner,
the host build of the group gather and Gauss-Jordan routines (tests/emu/emu_group.cpp) and the refusals of
``BlockGroups``.  GPU: the device inverses, ``gmres`` against ``spsolve``, its edge cases, and the Newton loops of the eight
fixtures with no matrix leaving the device."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import test_contact_model as tcm
import test_contact_poromech as tcp
import test_contact_thm as tct
from porepy_b200 import krylov
from porepy_b200.contact import mortar_pairs

MODULES = {**{n: tcm for n in tcm.CASES}, **{n: tcp for n in tcp.CASES}, **{n: tct for n in tct.CASES}}
FIXTURES = sorted(MODULES)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def stored_jacobians(name):
    """The problem and its stored Jacobians (initial and iterate, where present) in the problem's own ordering."""
    mod = MODULES[name]
    prob, d = mod.load_problem(name)
    cm = d["column_map"]
    rm = d["row_map"] if "row_map" in d else np.arange(prob.num_dofs)
    jacs = {key: mod._csr(d, key)[rm][:, cm].tocsr() for key in ("initial_jacobian", "iterate_jacobian")
            if key + "__data" in d}
    return prob, d, jacs


def host_preconditioner(J, groups):
    blocks = []
    for g in range(groups.num_groups):
        r, c = groups.rows[groups.ptr[g]:groups.ptr[g + 1]], groups.cols[groups.ptr[g]:groups.ptr[g + 1]]
        blocks.append((r, c, np.linalg.inv(J[r][:, c].toarray())))

    def apply(y):
        z = np.zeros_like(y)
        for r, c, binv in blocks:
            z[c] = binv @ y[r]
        return z
    return apply


def random_group_case(seed=0, singular=None, max_size=32):
    """A random sparse matrix with groups of every size 1 .. max_size over shuffled rows and columns.  Every row has entries
    outside its group, some blocks have structural zeros, group 3 has a zero leading diagonal that forces a row swap and
    ``singular`` (if given) is an exactly singular group (two equal rows)."""
    rng = np.random.default_rng(seed)
    sizes = np.arange(1, max_size + 1)
    n = int(sizes.sum())
    ptr = np.concatenate(([0], np.cumsum(sizes)))
    rows, cols = rng.permutation(n), rng.permutation(n)
    A = sps.random(n, n, density=0.05, random_state=seed, format="lil") * 0.1      # entries outside the groups
    for g, s in enumerate(sizes):
        r, c = rows[ptr[g]:ptr[g + 1]], cols[ptr[g]:ptr[g + 1]]
        B = rng.standard_normal((s, s)) + s * np.eye(s)
        if s >= 4:
            B[rng.random((s, s)) < 0.3] = 0.0                                           # structural zeros in the block
            B += s * np.eye(s)
        if g == 3:
            B[0, 0] = 0.0                                                               # zero leading pivot: a swap
        if g == singular:
            B[-1] = B[0]
        for i in range(s):
            for j in range(s):
                A[r[i], c[j]] = B[i, j] if B[i, j] != 0.0 else 0.0
    A = A.tocsr()
    A.eliminate_zeros()
    groups = krylov.BlockGroups(ptr, rows, cols)
    return A, groups


def numpy_inverses(A, groups):
    out = []
    for g in range(groups.num_groups):
        r, c = groups.rows[groups.ptr[g]:groups.ptr[g + 1]], groups.cols[groups.ptr[g]:groups.ptr[g + 1]]
        out.append(np.linalg.inv(A[r][:, c].toarray()))
    return out


# ---------------------------------------------------------------- CPU


@pytest.mark.parametrize("name", FIXTURES)
def test_model_groups_partition_and_blocks_are_nonsingular(name):
    prob, _, jacs = stored_jacobians(name)
    groups = prob.preconditioner_groups()              # BlockGroups validates the partition
    assert groups.n == prob.num_dofs
    assert np.array_equal(np.sort(groups.rows), np.arange(prob.num_dofs))
    assert np.array_equal(np.sort(groups.cols), np.arange(prob.num_dofs))
    assert set(groups.sizes.tolist()) == {tcm: {3, 9}, tcp: {4, 12}, tct: {5, 17}}[MODULES[name]]
    assert jacs
    for key, J in jacs.items():
        for g in range(groups.num_groups):
            r, c = groups.rows[groups.ptr[g]:groups.ptr[g + 1]], groups.cols[groups.ptr[g]:groups.ptr[g + 1]]
            assert np.linalg.cond(J[r][:, c].toarray()) < 1e4, (key, g)


@pytest.mark.parametrize("name", FIXTURES)
def test_scipy_gmres_with_model_groups_converges(name):
    prob, _, jacs = stored_jacobians(name)
    groups = prob.preconditioner_groups()
    b = np.random.default_rng(1).standard_normal(prob.num_dofs)
    for key, J in jacs.items():
        minv = host_preconditioner(J, groups)
        n = J.shape[0]
        op = spla.LinearOperator((n, n), matvec=lambda v: J @ minv(v))
        y, info = spla.gmres(op, b, rtol=1e-12, atol=0.0, restart=30, maxiter=20)
        x = minv(y)
        assert info == 0, key
        assert np.linalg.norm(J @ x - b) <= 1e-11 * np.linalg.norm(b), key
        xd = spla.spsolve(J.tocsc(), b)
        assert np.linalg.norm(x - xd) <= 1e-9 * np.linalg.norm(xd), key


def test_host_group_inverse_matches_numpy():
    from emu_group import group_inverses
    A, groups = random_group_case()
    assert set(groups.sizes.tolist()) == set(range(1, 33))
    # every row also has entries outside its group
    inv, bad = group_inverses(A, groups)
    assert bad == -1
    for g, ref in enumerate(numpy_inverses(A, groups)):
        s = int(groups.sizes[g])
        mine = inv[groups.inv_offsets[g]:groups.inv_offsets[g + 1]].reshape(s, s)
        assert np.abs(mine - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()) * s, g
    A2, groups2 = random_group_case(singular=20)
    _, bad = group_inverses(A2, groups2)
    assert bad == 20


def test_random_group_case_has_the_intended_structure():
    A, groups = random_group_case()
    r, c = groups.rows[groups.ptr[3]:groups.ptr[4]], groups.cols[groups.ptr[3]:groups.ptr[4]]
    assert A[r[0], c[0]] == 0.0                                  # the zero pivot that forces a swap
    in_group = np.zeros(A.shape, bool)
    for g in range(groups.num_groups):
        sl = slice(groups.ptr[g], groups.ptr[g + 1])
        in_group[np.ix_(groups.rows[sl], groups.cols[sl])] = True
    outside = (A != 0).toarray() & ~in_group
    assert outside.sum() > A.shape[0] // 2
    r, c = groups.rows[groups.ptr[20]:groups.ptr[21]], groups.cols[groups.ptr[20]:groups.ptr[21]]
    assert (A[r][:, c].toarray() == 0).any()                     # structural zeros inside a block


def test_block_groups_refusals():
    ok = krylov.BlockGroups([0, 2, 3], [0, 1, 2], [2, 0, 1])
    assert ok.num_groups == 2 and ok.inv_offsets.tolist() == [0, 4, 5]
    with pytest.raises(ValueError, match="more than one group"):
        krylov.BlockGroups([0, 2, 3], [0, 0, 2], [0, 1, 2])       # duplicate row
    with pytest.raises(ValueError, match="more than one group"):
        krylov.BlockGroups([0, 2, 3], [0, 1, 2], [1, 1, 2])       # duplicate column
    with pytest.raises(ValueError, match="out of range"):
        krylov.BlockGroups([0, 2, 3], [0, 1, 3], [0, 1, 2])       # not a partition of 0 .. n-1
    with pytest.raises(ValueError, match="columns"):
        krylov.BlockGroups([0, 2, 3], [0, 1, 2], [0, 1])          # sizes do not match
    with pytest.raises(ValueError, match="ptr"):
        krylov.BlockGroups([0, 2, 4], [0, 1, 2], [0, 1, 2])
    with pytest.raises(ValueError, match="empty"):
        krylov.BlockGroups([0, 2, 2, 3], [0, 1, 2], [0, 1, 2])
    n = 33
    with pytest.raises(ValueError, match="more than 32"):
        krylov.BlockGroups([0, n], np.arange(n), np.arange(n))
    krylov.BlockGroups([0, 32, 33], np.arange(n), np.arange(n))


def test_mortar_pairs_need_two_mortar_cells():
    m = sps.csr_matrix(np.array([[0.5, 0.5, 0, 0], [0, 0, 0.5, 0.5]]))
    assert mortar_pairs(m).tolist() == [[0, 1], [2, 3]]
    with pytest.raises(ValueError, match="fracture cell 1 has 3"):
        mortar_pairs(sps.csr_matrix(np.array([[0.5, 0.5, 0, 0, 0], [0, 0, 0.3, 0.3, 0.4]])))


def test_gmres_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "porepy_b200", "csrc", "gmres.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                          src, "-o", str(tmp_path / "gmres.o")], capture_output=True, text=True, check=True)
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out.stderr)
    assert len(spills) == 12, out.stderr
    assert all(v == ("0", "0", "0") for v in spills), out.stderr


# ---------------------------------------------------------------- GPU


def _cuda(a):
    import torch
    return torch.as_tensor(np.asarray(a, float), device="cuda")


@pytest.mark.gpu
def test_group_inverse_and_apply_gpu():
    import torch
    from porepy_b200.sparse import DeviceCsr
    A, groups = random_group_case()
    M = krylov.GroupedBlockJacobi(DeviceCsr(A), groups)
    for g, ref in enumerate(numpy_inverses(A, groups)):
        s = int(groups.sizes[g])
        assert np.abs(M.block(g).cpu().numpy() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()) * s, g
    y = np.random.default_rng(2).standard_normal(A.shape[0])
    z = M.apply(_cuda(y)).cpu().numpy()
    zr = np.zeros_like(y)
    for g, ref in enumerate(numpy_inverses(A, groups)):
        sl = slice(groups.ptr[g], groups.ptr[g + 1])
        zr[groups.cols[sl]] = ref @ y[groups.rows[sl]]
    assert np.abs(z - zr).max() <= 1e-12 * np.abs(zr).max()
    A2, groups2 = random_group_case(singular=20)
    with pytest.raises(ValueError, match="group 20 "):
        krylov.GroupedBlockJacobi(DeviceCsr(A2), groups2)
    assert torch.isfinite(M.inv).all()


def _check_solution(A, b, x, tol=1e-9):
    xd = spla.spsolve(sps.csc_matrix(A), b)
    assert np.linalg.norm(x - xd) <= tol * np.linalg.norm(xd)


@pytest.mark.gpu
def test_gmres_random_nonsymmetric_gpu():
    from porepy_b200.sparse import DeviceCsr
    rng = np.random.default_rng(3)
    n = 3000
    A = (sps.random(n, n, density=4.0 / n, random_state=3) + sps.diags(4.0 + rng.random(n))).tocsr()
    b = rng.standard_normal(n)
    groups = krylov.BlockGroups(np.arange(0, n + 1, 3), np.arange(n), np.arange(n))
    Ad = DeviceCsr(A)
    x, info = krylov.gmres(Ad, _cuda(b), krylov.GroupedBlockJacobi(Ad, groups), tol=1e-12)
    assert info["converged"] and info["relres"] <= 1e-12 and info["cuda_graph"], info
    assert info["host_syncs"] == info["restarts"] + 1
    _check_solution(A, b, x.cpu().numpy())
    x0, info0 = krylov.gmres(Ad, _cuda(b), None, tol=1e-12, restart=50)              # no preconditioner
    assert info0["converged"], info0
    _check_solution(A, b, x0.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_gmres_on_contact_jacobians_gpu(name):
    from porepy_b200.sparse import DeviceCsr
    prob, _, jacs = stored_jacobians(name)
    groups = prob.preconditioner_groups()
    b = np.random.default_rng(4).standard_normal(prob.num_dofs)
    for key, J in jacs.items():
        Jd = DeviceCsr(J)
        x, info = krylov.gmres(Jd, _cuda(b), krylov.GroupedBlockJacobi(Jd, groups), tol=1e-12, restart=30)
        assert info["converged"] and not info["breakdown"] and info["iterations"] < 200, (key, info)
        assert np.linalg.norm(J @ x.cpu().numpy() - b) <= 1e-11 * np.linalg.norm(b), key
        _check_solution(J, b, x.cpu().numpy())


@pytest.mark.gpu
def test_gmres_edge_cases_gpu():
    import torch
    from porepy_b200.sparse import DeviceCsr
    A, groups = random_group_case()
    n = A.shape[0]
    # exactly block-diagonal: the preconditioner is the inverse, one step and an invariant subspace
    mask = np.zeros(A.shape, bool)
    for g in range(groups.num_groups):
        sl = slice(groups.ptr[g], groups.ptr[g + 1])
        mask[np.ix_(groups.rows[sl], groups.cols[sl])] = True
    D = sps.csr_matrix(np.where(mask, A.toarray(), 0.0))
    b = np.random.default_rng(5).standard_normal(n)
    Dd = DeviceCsr(D)
    x, info = krylov.gmres(Dd, _cuda(b), krylov.GroupedBlockJacobi(Dd, groups), tol=1e-12)
    assert info["converged"] and info["iterations"] == 1 and info["lucky_breakdown"] and not info["breakdown"], info
    assert torch.isfinite(x).all()
    _check_solution(D, b, x.cpu().numpy())
    # restart >= n (55 unknowns)
    As, gs = random_group_case(seed=1, max_size=10)
    bs = np.random.default_rng(7).standard_normal(As.shape[0])
    Asd = DeviceCsr(As)
    x, info = krylov.gmres(Asd, _cuda(bs), krylov.GroupedBlockJacobi(Asd, gs), tol=1e-12, restart=As.shape[0] + 5)
    assert info["converged"] and info["restarts"] <= 2 and torch.isfinite(x).all(), info
    _check_solution(As, bs, x.cpu().numpy())
    # a general system: maxiter not a multiple of restart, too small a maxiter
    Ad = DeviceCsr(A)
    M = krylov.GroupedBlockJacobi(Ad, groups)
    x, info = krylov.gmres(Ad, _cuda(b), M, tol=1e-12, restart=4, maxiter=4 * 50 + 3)
    assert info["converged"], info
    _check_solution(A, b, x.cpu().numpy())
    x, info = krylov.gmres(Ad, _cuda(b), M, tol=1e-12, restart=4, maxiter=7)
    assert not info["converged"] and info["iterations"] == 7 and info["restarts"] == 2 and info["relres"] > 1e-12, info
    solver = krylov.gmres_solver(groups, tol=1e-12, restart=4, maxiter=7)
    with pytest.raises(RuntimeError, match="did not converge"):
        solver(Ad, _cuda(b))
    x, info = krylov.gmres(Ad, torch.zeros(n, dtype=torch.float64, device="cuda"), M)
    assert info["converged"] and info["iterations"] == 0 and not x.any()


@pytest.mark.gpu
def test_gmres_is_bit_identical_on_repeat_gpu():
    from porepy_b200.sparse import DeviceCsr
    prob, _, jacs = stored_jacobians("contact_thm")
    J = jacs["iterate_jacobian"]
    Jd = DeviceCsr(J)
    b = _cuda(np.random.default_rng(6).standard_normal(J.shape[0]))
    groups = prob.preconditioner_groups()
    x1, i1 = krylov.gmres(Jd, b, krylov.GroupedBlockJacobi(Jd, groups), tol=1e-12, restart=20)
    x2, i2 = krylov.gmres(Jd, b, krylov.GroupedBlockJacobi(Jd, groups), tol=1e-12, restart=20)
    assert i1["restarts"] > 1 and i1 == i2
    assert np.array_equal(x1.cpu().numpy(), x2.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_time_step_with_device_gmres_gpu(name, monkeypatch):
    """The Newton loops of the eight fixtures with the device solver: the assertions of the host-solve tests, and no matrix
    is downloaded."""
    from porepy_b200.sparse import DeviceCsr
    mod = MODULES[name]
    prob, d = mod.load_problem(name)
    prob.discretize()
    solver = krylov.gmres_solver(prob.preconditioner_groups())

    def refuse(self):
        raise AssertionError("a matrix left the device")
    monkeypatch.setattr(DeviceCsr, "to_scipy", refuse)
    cm = d["column_map"]
    if mod is tcm:
        x, hist = prob.time_step(d["previous"], solver, tol=1e-11)
        nref = 4
    else:
        x, hist = prob.time_step(d["previous"][cm], float(d["dt"]), solver, tol=1e-11)
        nref = 5
    monkeypatch.undo()
    ref = d["residual_norms"]
    assert hist[-1]["residual"] <= 1e-10 * hist[0]["residual"] and len(hist) <= len(ref) + 1, hist
    for mine, theirs in zip(hist[:nref], ref[:nref]):
        if theirs > 1e-9 * ref[0]:
            assert abs(mine["residual"] - theirs) <= 0.05 * theirs, (hist, ref)
    xh = x.cpu().numpy()
    assert np.linalg.norm(xh - d["solution"][cm]) <= 1e-8 * np.linalg.norm(d["solution"])
    assert solver.last_info["converged"] and solver.last_info["cuda_graph"]
    if mod is tcm:                                 # the contact state of the pure-contact cases
        t = prob.unknown_layout.parts(xh)["contact_traction"][0].reshape(-1, 3)
        mu = float(d["friction_coefficient"])
        is_open = np.abs(t[:, 2]) < 1e-12
        assert np.all(np.abs(t[is_open]) < 1e-12) and np.all(t[~is_open, 2] < 0)
        assert np.all(np.linalg.norm(t[~is_open, :2], axis=1) <= mu * np.abs(t[~is_open, 2]) * (1 + 1e-8))
        ratio = np.linalg.norm(t[:, :2], axis=1) / np.maximum(mu * np.abs(t[:, 2]), 1e-300)
        expect = {"contact_model": lambda: np.allclose(ratio, 1.0, rtol=1e-8),
                  "contact_sticking": lambda: np.all(ratio < 0.2),
                  "contact_open": lambda: np.all(t == 0.0),
                  "contact_mixed": lambda: np.sum(np.abs(t[:, 2]) < 1e-12) == 2
                  and np.allclose(ratio[np.abs(t[:, 2]) > 1e-12], 1.0)}
        assert expect[name](), (name, t)


def _live_two_fracture_problems():
    """(problem, previous state, dt) of ``pp.MomentumBalance``, ``pp.Poromechanics`` and ``pp.Thermoporomechanics`` on a
    cube with two parallel fractures, through the model bridges (the geometry of test_porepy_plugin's two-fracture
    test)."""
    import make_contact_golden as gc
    from make_mdflow_golden import rect
    from test_porepy_plugin import load_porepy
    pp = load_porepy()
    from porepy_b200.porepy_plugin import plugin
    b = plugin(pp)

    class Geometry:
        set_domain, grid_type, stiffness_tensor = gc.Model.set_domain, gc.Model.grid_type, gc.Model.stiffness_tensor
        bc_type_mechanics = gc.Model.bc_type_mechanics

        def meshing_arguments(self):
            return {"cell_size": 0.25}

        def set_fractures(self):
            self._fractures = [pp.PlaneFracture(rect(0, 0.25, 0.25, 0.75)), pp.PlaneFracture(rect(0, 0.75, 0.0, 0.5))]

        def bc_values_displacement(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros((3, bg.num_cells))
            v[0, s.east] = 0.02 * (bg.cell_centers[2, s.east] - 0.4)
            v[1, s.east] = 0.01
            return v.ravel("F")

        def bc_type_darcy_flux(self, sd):
            s = self.domain_boundary_sides(sd)
            return pp.BoundaryCondition(sd, s.south + s.north, "dir")
        bc_type_fluid_flux = bc_type_fourier_flux = bc_type_enthalpy_flux = bc_type_darcy_flux

        def bc_values_pressure(self, bg):
            s = self.domain_boundary_sides(bg)
            v = np.zeros(bg.num_cells)
            v[s.south] = 0.02 * (1 + bg.cell_centers[0, s.south])
            return v
    fluid = pp.FluidComponent(compressibility=0.05, viscosity=1.3, density=1.7, thermal_expansion=0.03,
                              specific_heat_capacity=2.0, thermal_conductivity=0.7)
    solid = pp.SolidConstants(porosity=0.2, biot_coefficient=0.8, lame_lambda=2.0, shear_modulus=1.5, permeability=1.0,
                              normal_permeability=2.0, residual_aperture=0.05, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1, thermal_expansion=0.02, specific_heat_capacity=1.5,
                              thermal_conductivity=1.1, density=2.5)
    params = {"times_to_export": [], "material_constants": {"fluid": fluid, "solid": solid}}
    for ref_cls, build, dt in ((pp.MomentumBalance, b.fractured_momentum_from_model, None),
                               (pp.Poromechanics, b.fractured_poromechanics_from_model, 0.25),
                               (pp.Thermoporomechanics, b.fractured_thermoporomechanics_from_model, 0.25)):
        model = type("Live2", (Geometry, ref_cls), {})(dict(
            params, time_manager=pp.TimeManager([0, 1.0], dt or 1.0, constant_dt=True)))
        model.prepare_simulation()
        model.time_manager.increase_time()
        model.time_manager.increase_time_index()
        assert len(model.mdg.subdomains(dim=2)) == 2
        out = build(model)
        yield out[0], model.equation_system.get_variable_values(time_step_index=0)[out[1]], dt


@pytest.mark.gpu
def test_live_two_fracture_models_with_device_gmres_gpu():
    """Where the reference is present: the two-fracture live models through the bridges take one time step with the device
    solver and reach the state of the host-solve path."""
    from test_porepy_plugin import reference_available
    if not reference_available():
        pytest.skip("oracle/_ref not present")
    for prob, x_prev, dt in _live_two_fracture_problems():
        prob.discretize()
        solver = krylov.gmres_solver(prob.preconditioner_groups())

        def direct(J, r):
            return _cuda(spla.spsolve(J.to_scipy().tocsc(), r.cpu().numpy()))
        step = (lambda s: prob.time_step(x_prev, s, tol=1e-11)) if dt is None else \
            (lambda s: prob.time_step(x_prev, dt, s, tol=1e-11))
        xh, _ = step(direct)
        xg, hg = step(solver)
        assert hg[-1]["residual"] <= 1e-10 * hg[0]["residual"], (type(prob), hg)
        xh, xg = xh.cpu().numpy(), xg.cpu().numpy()
        assert np.linalg.norm(xg - xh) <= 1e-8 * np.linalg.norm(xh), type(prob)
