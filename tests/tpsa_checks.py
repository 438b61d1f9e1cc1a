"""Checks shared by the tests of the four TPSA systems (three-field elasticity, poromechanics, thermo-poromechanics and
frictional contact): the host build, the linearizations and Newton loops against the reference's stored states, the
device assembly against the host build, the stock models through the bridges, the 998,250-tetrahedron problems with
their field-ordered references, and the ptxas report of a CUDA source."""
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.tpsa_elasticity import TpsaElasticity, interleave
from porepy_b200.tpsa_poromech import TpsaPoromechanics
from porepy_b200.tpsa_thermoporomech import TpsaThermoporomechanics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- small helpers ------------------------------------------------------------------------------------------------


def csr(d, key):
    return sps.csr_matrix((d[key + "__data"], d[key + "__indices"], d[key + "__indptr"]), shape=tuple(d[key + "__shape"]))


def host(t):
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def scalar_bc(d, prefix, nf):
    return SimpleNamespace(is_dir=d[prefix + "_is_dir"], is_neu=d[prefix + "_is_neu"], is_rob=np.zeros(nf, bool),
                           is_internal=np.zeros(nf, bool), robin_weight=np.ones(nf), bc_type="scalar", num_faces=nf)


def direct(J, rhs):
    """The Newton update J dx = rhs by scipy's direct solver, as a tensor on rhs's device."""
    import torch
    return torch.as_tensor(spla.spsolve(J.to_scipy().tocsc(), host(rhs)), device=rhs.device)


def to_solver(prob, x):
    """A state of the model's dof order in the problem's cell-interleaved order."""
    return np.asarray(x)[prob.column_map]


def to_model(prob, x):
    """A state of the problem's order in the model's dof order."""
    xm = np.empty(prob.num_dofs)
    xm[prob.column_map] = host(x)
    return xm


def use_host_build(mp, plan=True, sparse=True):
    """Run the TPSA problems on the host build of tpsa_system.cuh on the monkeypatch ``mp``; ``plan`` / ``sparse``
    also install the host ``DevicePlan`` and the scipy stand-in for the device sparse algebra."""
    from emu_tpsa import EmuTpsaFaceGrid
    mp.setattr(fv, "FaceGrid", EmuTpsaFaceGrid)
    if plan:
        from emu_binding import EmuBackedPlan
        mp.setattr(fv, "DevicePlan", EmuBackedPlan)
    if sparse:
        import emu_sparse
        emu_sparse.install(mp)


# ---- against the reference's stored states ------------------------------------------------------------------------


def newton_states(d):
    """(label, x, x_prev, J key, rhs key) of the zero state and of an intermediate iterate of each of two time steps."""
    return [("zero", d["s0_previous"], d["s0_previous"], "J0", "rhs0")] + [
        (f"step {s}", d[f"s{s}_iterate"], d[f"s{s}_previous"], f"s{s}_J", f"s{s}_rhs") for s in range(2)]


OWN, ZERO = "own", "zero"          # the scale of -R in check_linearizations: each state's own, or the zero state's


def check_linearizations(prob, d, states, tol, rhs_scale, *args):
    """J and -R of ``prob.linearize(x, x_prev, *args)`` at each stored state after the dof maps: J to ``tol`` of
    max |J|, -R to ``tol`` of max |-R| of the same state (``OWN``) or of the zero state (``ZERO``, for a stored iterate
    that is converged).  Returns the (J, -R) pairs."""
    prob.discretize()
    got = []
    for label, x, xp, jk, rk in states:
        J, rhs = prob.linearize(to_solver(prob, x), to_solver(prob, xp), *args)
        Jm, bm = prob.to_model_order(J.to_scipy(), host(rhs))
        Jr, br = csr(d, jk), d[rk]
        assert abs(Jm - Jr).max() <= tol * abs(Jr).max(), label
        assert np.abs(bm - br).max() <= tol * np.abs(br if rhs_scale == OWN else d["rhs0"]).max(), label
        got.append((J.to_scipy(), host(rhs).copy()))
    assert int(prob._missing.sum()) == 0
    return got


def check_time_steps(prob, d, tol):
    """Two time steps from the stored previous states with a direct solver: residual histories to ``tol`` of the first
    residual, with as many iterations, and converged states to ``tol``."""
    for s in range(2):
        x, hist = prob.time_step(to_solver(prob, d[f"s{s}_previous"]), float(d["dt"]), tol=1e-13,
                                 linear_solver=direct, linear_tol=1e-13)
        ref = d[f"s{s}_residual_norms"]
        mine = np.array([h["residual"] for h in hist])
        assert len(mine) == len(ref), (mine, ref)
        assert np.abs(mine - ref).max() <= tol * ref[0], (mine, ref)
        sol = d[f"s{s}_solution"]
        assert np.linalg.norm(to_model(prob, x) - sol) <= tol * np.linalg.norm(sol), s


def newton_reaches_reference(prob, d, tol):
    """The Newton loop with the device block-Jacobi BiCGStab reaches the reference's converged states to ``tol``."""
    prob.discretize()
    for s in range(2):
        x, hist = prob.time_step(to_solver(prob, d[f"s{s}_previous"]), float(d["dt"]), tol=1e-12, linear_tol=1e-13)
        assert all(h.get("linear_converged", True) for h in hist), hist
        sol = d[f"s{s}_solution"]
        assert np.linalg.norm(to_model(prob, x) - sol) <= tol * np.linalg.norm(sol), (s, hist)


def compare_with_host_build(host_pairs, dev, tol=1e-13, same_pattern=False, **build):
    """The device's (A, b) pairs ``dev`` against ``host_pairs()`` run on the host build (``use_host_build(**build)``):
    A to ``tol`` of max |A|, b to ``tol`` of max |b| of the first pair (-R near convergence is b0 - A x with
    cancellation: its round-off is measured on the scale of -R at the zero state); ``same_pattern``: equal patterns."""
    with pytest.MonkeyPatch.context() as mp:
        use_host_build(mp, **build)
        hst = host_pairs()
    rscale = np.abs(hst[0][1]).max()
    for (A, b), (Ah, bh) in zip(dev, hst):
        if same_pattern:
            assert np.array_equal(A.indptr, Ah.indptr) and np.array_equal(A.indices, Ah.indices)
        assert abs(A - Ah).max() <= tol * abs(Ah).max()
        assert np.abs(b - bh).max() <= tol * rscale


# ---- the stock models through the bridges --------------------------------------------------------------------------


def check_model_order(prob, A, b, J, rhs, cols, rows):
    """A and b after the dof maps equal the model's J and -R to 1e-12, and the two maps are permutations."""
    Am, bm = prob.to_model_order(A.to_scipy() if hasattr(A, "to_scipy") else A, host(b))
    assert abs(Am - J).max() <= 1e-12 * abs(J).max()
    assert np.abs(bm - rhs).max() <= 1e-12 * np.abs(rhs).max()
    assert np.array_equal(np.sort(cols), np.arange(J.shape[1])) and np.array_equal(np.sort(rows), np.arange(J.shape[0]))


def check_bridge_linearization(m, prob, cols, rows, *args):
    """The linearization at the model's iterate and previous state (``linearize(x, x_prev, *args)``) against the
    model's own."""
    es = m.equation_system
    J, rhs = es.assemble()
    x, xp = es.get_variable_values(iterate_index=0), es.get_variable_values(time_step_index=0)
    A, b = prob.linearize(x[cols], xp[cols], *args)
    check_model_order(prob, A, b, J, rhs, cols, rows)


def check_single_grid_refusals(bridge, other_bridge, equations, match):
    """``bridge`` refuses a fake model on two subdomains and one with a fracture; ``other_bridge`` refuses one grid with
    the balance ``equations``, naming ``match``."""
    sd = SimpleNamespace(dim=2)
    fake = SimpleNamespace(nd=2, mdg=SimpleNamespace(subdomains=lambda: [sd, sd], interfaces=lambda: []),
                           equation_system=SimpleNamespace(equations={}))
    with pytest.raises(NotImplementedError, match="one subdomain"):
        bridge(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd, SimpleNamespace(dim=1)], interfaces=lambda: [])
    with pytest.raises(NotImplementedError, match="fractures"):
        bridge(fake)
    fake.mdg = SimpleNamespace(subdomains=lambda: [sd], interfaces=lambda: [])
    fake.equation_system = SimpleNamespace(equations=dict.fromkeys(equations))
    with pytest.raises(NotImplementedError, match=match):
        other_bridge(fake)


# ---- 998,250 tetrahedra (the TPSA bench mesh) ---------------------------------------------------------------------


def full_size_mechanics():
    """The bench mesh with Dirichlet, roller, Robin and Neumann mechanical faces and a seeded shear modulus, 10^6 times
    larger where x < 0.3: (grid, bc, mu)."""
    g = pb.structured_tet_grid((55, 55, 55))
    nf, nd = g.num_faces, 3
    bf = g.get_all_boundary_faces()
    xf = g.face_centers[:, bf]
    bc = pb.BoundaryConditionVectorial(g)
    west = bf[xf[0] < 1e-10]
    south = bf[(xf[1] < 1e-10) & (xf[0] > 1e-10)]
    top = bf[(xf[2] > 1 - 1e-10) & (xf[0] > 1e-10) & (xf[1] > 1e-10)]
    bc.is_dir[:, west] = True
    bc.is_neu[:, west] = False
    bc.is_dir[1, south] = True          # roller
    bc.is_neu[1, south] = False
    bc.is_rob[:, top] = True
    bc.is_neu[:, top] = False
    rng = np.random.default_rng(7)
    w = np.zeros((nd, nd, nf))
    for i in range(nd):
        w[i, i] = 0.2 + 5 * rng.random(nf)
    bc.robin_weight = w
    mu = np.exp(rng.standard_normal(g.num_cells))
    mu[g.cell_centers[0] < 0.3] *= 1e6
    return g, bc, mu


def full_size_problem(physics, seed):
    """The bench mesh of ``full_size_mechanics`` with seeded lambda and seeded data for ``physics`` ("elasticity",
    "poromechanics" or "thermoporomechanics"): (problem, the generator for further draws).  The scalar fields have
    Dirichlet faces on the two x-sides and Neumann faces elsewhere."""
    g, bc, mu = full_size_mechanics()
    nc, nf = g.num_cells, g.num_faces
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.standard_normal(nc))
    if physics == "elasticity":
        data = pb.initialize_data({}, "mech", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
        return TpsaElasticity(g, data, "mech", rng.standard_normal(3 * nf), rng.standard_normal(3 * nc),
                              rng.standard_normal(3 * nc), rng.standard_normal(nc)), rng
    thermal = physics == "thermoporomechanics"
    K = pb.SecondOrderTensor(np.exp(0.5 * rng.standard_normal(nc)))
    bf = np.asarray(g.get_all_boundary_faces(), np.int64)
    x = g.face_centers[0, bf]
    is_dir = np.isin(np.arange(nf), bf[(x < x.min() + 1e-9) | (x > x.max() - 1e-9)])
    is_neu = np.isin(np.arange(nf), bf) & ~is_dir
    fbc = SimpleNamespace(is_dir=is_dir, is_neu=is_neu, is_rob=np.zeros(nf, bool), is_internal=np.zeros(nf, bool),
                          robin_weight=np.ones(nf), bc_type="scalar", num_faces=nf)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": K, "bc": fbc})
    if thermal:
        pb.initialize_data(data, "fourier", {"bc": fbc})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
    fluid = dict(compressibility=0.05, density=1.7, viscosity=1.3, reference_pressure=0.3)
    if thermal:
        cls = TpsaThermoporomechanics
        fluid.update(thermal_expansion=0.2, heat_capacity=2.0, conductivity=0.7, reference_temperature=0.4)
        solid = dict(reference_porosity=0.2, biot_coefficient=0.8, bulk_modulus=3.0, thermal_expansion=0.1,
                     heat_capacity=1.5, conductivity=1.1, density=2.5)
    else:
        cls = TpsaPoromechanics
        solid = dict(reference_porosity=0.2, biot_coefficient=0.7, bulk_modulus=3.0)
    # the boundary values of the scalar fields (pressure, then temperature) and of the mechanics, then the Neumann
    # flux boundary operators with their values
    args = [np.where(is_dir, rng.random(nf), 0.0) for _ in range(1 + thermal)] + [rng.standard_normal(3 * nf)]
    args += [fbc, np.where(is_dir, 1.7 / 1.3, 0.0)] + ([fbc, np.where(is_dir, 0.5, 0.0)] if thermal else [])
    return cls(g, data, fluid, solid, *args, body_force=rng.standard_normal(3 * nc),
               fluid_source=rng.standard_normal(nc) * g.cell_volumes), rng


def field_order(prob):
    """For each cell-interleaved index of ``prob``, its index in the field-wise order [u | r | scalar fields]."""
    starts = np.cumsum([0] + [w * prob.nc for _, w in prob.fields])
    return interleave([np.arange(s, e) for s, e in zip(starts[:-1], starts[1:])], prob.nd, prob.nr, prob.nc)


def field_ordered_reference(prob, mech_matrices, scalar_rows):
    """J of ``prob`` in its cell-interleaved order, assembled field-wise with the device ``bmat`` and permuted: the
    momentum, angular momentum and solid mass rows from the ``pb.Tpsa`` matrices ``mech_matrices``, then the caller's
    scalar balance rows (``scalar_rows``: their device blocks from the p_t column on)."""
    from porepy_b200 import ad
    from porepy_b200.sparse import DeviceCsr
    M = {k: ad.as_device_csr(v) for k, v in mech_matrices.items()}
    g, nd, nr, nc = prob.sd, prob.nd, prob.nr, prob.nc
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr, d1 = (DeviceCsr(sps.kron(div, sps.eye(k)).tocsr()) for k in (nd, nr, 1))
    vol = g.cell_volumes
    C = prob.data[pb.PARAMETERS][prob.keyword]["fourth_order_tensor"]
    lam, mu = np.asarray(C.lmbda), np.asarray(C.mu)

    def diag(v):
        return DeviceCsr(sps.diags(v).tocsr())
    pad = [None] * len(scalar_rows)
    pressure = [diag(-vol * prob.alpha / lam)] + pad[1:] if scalar_rows else []     # p in the solid mass balance
    ref = DeviceCsr.bmat([
        [-(dn @ M["stress"]), -(dn @ M["stress_rotation"]), -(dn @ M["stress_total_pressure"]), *pad],
        [dr @ M["rotation_displacement"], (dr @ M["rotation_rotation"]) - diag(np.repeat(vol / mu, nr)), None, *pad],
        [d1 @ M["solid_mass_displacement"], None, (d1 @ M["solid_mass_total_pressure"]) - diag(vol / lam), *pressure]]
        + [[None, None, *row] for row in scalar_rows])
    order = field_order(prob)
    n = order.size
    P = DeviceCsr(sps.csr_matrix((np.ones(n), (np.arange(n), order)), shape=(n, n)))
    return (P @ ref) @ DeviceCsr(sps.csr_matrix((np.ones(n), (order, np.arange(n))), shape=(n, n)))


def check_full_size_linearization(physics, seed, scalar_rows):
    """``full_size_problem(physics, seed)`` at a seeded iterate of a time step: two linearizations bit-identical with no
    entry outside the pattern, and J to 1e-13 of max |J| against ``field_ordered_reference`` with the scalar balance
    rows ``scalar_rows(prob, x, x_prev, dt)``."""
    import torch
    prob, rng = full_size_problem(physics, seed)
    assert prob.nc == 998_250
    n = prob.num_dofs
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
    pb.Tpsa("mechanics").discretize(prob.sd, prob.data)
    ref = field_ordered_reference(prob, prob.data[pb.DISCRETIZATION_MATRICES]["mechanics"],
                                  scalar_rows(prob, x, x_prev, 0.25))
    diff = ref.axpby(1.0, J1, -1.0).to_scipy()
    assert np.abs(diff.data).max() <= 1e-13 * np.abs(a1.data).max()


# ---- register use (compile only) ------------------------------------------------------------------------------------


def _kernel_name(mangled):
    """'stem<a, b>' of an Itanium-mangled kernel whose template arguments are ints ('_Z<len><stem>ILi2ELi1EE...');
    any other name as it is."""
    m = re.match(r"_Z(\d+)", mangled)
    if m is None:
        return mangled
    n = int(m.group(1))
    stem, rest = mangled[m.end():m.end() + n], mangled[m.end() + n:]
    args = re.match(r"I((?:Li-?\d+E)+)E", rest)
    return stem + (f"<{', '.join(re.findall(r'Li(-?\d+)E', args.group(1)))}>" if args else "")


def ptxas_properties(src, tmp_path):
    """{kernel name: ptxas properties line ('<n> bytes stack frame, ...')} of ``porepy_b200/csrc/<src>`` compiled for
    sm_90a; skips the test when nvcc is not available."""
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-c", os.path.join(ROOT, "porepy_b200", "csrc", src),
                          "-o", str(tmp_path / (os.path.splitext(src)[0] + ".o"))],
                         capture_output=True, text=True, check=True)
    return {_kernel_name(fn): props for fn, props in re.findall(r"Function properties for (\S+)\n\s*(.*)", out.stderr)}
