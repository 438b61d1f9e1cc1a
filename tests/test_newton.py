"""The device-resident Newton loop (porepy_b200/newton.py): nonlinear single-phase flow with k = k0 exp(beta p) on the
differentiable two-point flux (reference constitutive_laws.py:1500-1583).  CPU: the host restatement of the residual and
its Jacobian (finite differences, Newton convergence, T against the reference's golden AD values).  GPU: the
``DeviceAdArray`` chain against the host restatement entry by entry, the one-kernel ``pb_tpfa_diff`` against the chain,
and the whole loop (device Jacobian chain + fused BiCGStab) against a scipy Newton iteration."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200 import newton


def _problem(dims=(6, 5, 4), beta=0.7, seed=3):
    g = pb.cart_grid_3d(list(dims), perturb=0.25, seed=seed)
    rng = np.random.default_rng(seed)
    nc = g.num_cells
    q = rng.standard_normal((nc, 3, 3))
    k0 = (np.einsum("cij,ckj->cik", 0.2 * q, 0.2 * q) + np.eye(3)).reshape(-1)
    bf = g.get_all_boundary_faces()
    x = g.face_centers[0, bf]
    dirf = bf[(x < 1e-10) | (x > 1 - 1e-10)]
    dirv = np.where(g.face_centers[0, dirf] < 0.5, 1.0, 0.0)
    src = 0.5 * g.cell_volumes * rng.random(nc)
    return newton.NonlinearTpfaFlow(g, k0, beta, dirf, dirv, src)


def _host_newton(prob, tol=1e-12, maxit=25):
    p = np.zeros(prob.g.num_cells)
    hist = []
    for _ in range(maxit):
        R, J = prob.residual_host(p)
        hist.append(float(np.linalg.norm(R)))
        if hist[-1] <= tol * hist[0]:
            break
        p = p - spla.spsolve(J.tocsc(), R)
    return p, hist


def test_host_restatement_jacobian_and_convergence():
    prob = _problem()
    rng = np.random.default_rng(0)
    p = 0.3 * rng.standard_normal(prob.g.num_cells)
    R, J = prob.residual_host(p)
    v = rng.standard_normal(p.size)
    eps = 1e-6
    fd = (prob.residual_host(p + eps * v)[0] - prob.residual_host(p - eps * v)[0]) / (2 * eps)
    assert np.abs(J @ v - fd).max() <= 1e-7 * np.abs(fd).max()
    sol, hist = _host_newton(prob)
    assert hist[-1] <= 1e-12 * hist[0] and len(hist) <= 10
    # beta = 0: the linear TPFA problem, one step
    lin = _problem(beta=0.0)
    _, h0 = _host_newton(lin)
    assert len(h0) <= 3


@pytest.mark.gpu
def test_device_chain_matches_host_and_fused_kernel():
    import torch
    prob = _problem()
    rng = np.random.default_rng(1)
    p = 0.3 * rng.standard_normal(prob.g.num_cells)
    R_dev = prob.residual(torch.as_tensor(p, device="cuda"))
    val, jac = R_dev.host()
    R, J = prob.residual_host(p)
    assert np.abs(val - R).max() <= 1e-12 * np.abs(R).max()
    assert abs(J - jac).max() <= 1e-11 * abs(J).max()
    # the one-kernel transmissibility + Jacobian equals the AD chain's
    from porepy_b200 import ad
    T_ad, _ = prob.transmissibility(ad.variables([torch.as_tensor(p, device="cuda")])[0])
    Tv, Tj = T_ad.host()
    Tf, Jf = prob.fused_transmissibility(p)
    assert np.abs(Tv - Tf).max() <= 1e-12 * np.abs(Tf).max()
    assert abs(Tj - Jf).max() <= 1e-11 * abs(Jf).max()


@pytest.mark.gpu
def test_device_newton_loop_matches_scipy_newton():
    prob = _problem((10, 9, 8))
    sol, hist = _host_newton(prob)
    p, h = newton.solve(prob, tol=1e-11, linear_tol=1e-12)
    assert h[-1]["residual"] <= 1e-11 * h[0]["residual"] and len(h) <= len(hist) + 2
    assert all(r.get("linear_converged", True) for r in h)
    assert np.linalg.norm(p.cpu().numpy() - sol) <= 1e-8 * np.linalg.norm(sol)


class _Dense:
    """A dense Jacobian with an ``nnz``, as ``DeviceCsr`` has."""

    def __init__(self, a):
        self.a, self.nnz = a, int((a != 0).sum())


def _cubic(with_nnz=True):
    """R(x) = x^3 + x - b on CPU tensors: (linearize, linear solver, b, the list of solved right-hand sides)."""
    import torch
    b = torch.tensor([1.0, 2.0, -3.0], dtype=torch.float64)
    solved = []

    def linearize(x):
        J = torch.diag(3 * x * x + 1)
        return (_Dense(J) if with_nnz else J), -(x ** 3 + x - b)

    def solver(J, rhs):
        solved.append(rhs.clone())
        return torch.linalg.solve(J.a if with_nnz else J, rhs)
    return linearize, solver, b, solved


def test_newton_loop_stops_at_the_relative_tolerance_and_keeps_x0():
    import torch
    linearize, solver, b, solved = _cubic()
    x0 = torch.zeros(3, dtype=torch.float64)
    x, hist = newton.newton_loop(linearize, x0, solver, tol=1e-12, max_iterations=30)
    assert torch.equal(x0, torch.zeros(3, dtype=torch.float64))
    assert hist[-1]["residual"] <= 1e-12 * hist[0]["residual"] < hist[-2]["residual"]
    assert [h["iteration"] for h in hist] == list(range(len(hist))) and len(solved) == len(hist) - 1
    assert float(torch.linalg.vector_norm(x ** 3 + x - b)) <= 1e-12 * float(torch.linalg.vector_norm(b))
    assert all(h["jacobian_nnz"] == 3 for h in hist) and "linear_iterations" not in hist[0]


def test_newton_loop_zero_initial_residual_and_iteration_limit():
    import torch
    linearize, solver, _, solved = _cubic()
    x, hist = newton.newton_loop(linearize, torch.zeros(3, dtype=torch.float64), solver, tol=0.0, max_iterations=2)
    assert len(hist) == 3 and len(solved) == 2                         # max_iterations + 1 records, no last solve
    # r0 = 0: the stopping test is against 1e-300, met at once, nothing solved
    linearize, solver, _, solved = _cubic()
    x0 = torch.ones(3, dtype=torch.float64)
    x, hist = newton.newton_loop(lambda x: (linearize(x)[0], torch.zeros(3, dtype=torch.float64)), x0, solver, 1e-10, 4)
    assert [h["residual"] for h in hist] == [0.0] and not solved and torch.equal(x, x0) and x is not x0


def test_newton_loop_records_linear_solver_info_and_nnz_only_when_present():
    import torch
    linearize, solver, _, _ = _cubic(with_nnz=False)
    infos = iter([{"iterations": 7, "converged": True}, {"iterations": 5, "converged": False, "true_relres": 1e-3}])

    def with_info(J, rhs):
        with_info.last_info = next(infos)
        return solver(J, rhs)
    with_info.last_info = None
    _, hist = newton.newton_loop(linearize, torch.zeros(3, dtype=torch.float64), with_info, tol=0.0, max_iterations=2)
    assert all("jacobian_nnz" not in h for h in hist)
    assert hist[0]["linear_iterations"] == 7 and hist[0]["linear_converged"] is True
    assert "linear_true_relres" not in hist[0]
    assert hist[1]["linear_iterations"] == 5 and hist[1]["linear_converged"] is False
    assert hist[1]["linear_true_relres"] == 1e-3
    assert "linear_iterations" not in hist[2]                          # the last record: no solve
