"""Time the device Jacobian of the TPSA poromechanics model (``porepy_b200.TpsaPoromechanics``, ``pb_tpsa_poro_system`` /
``pb_tpsa_poro_fluid_rows``) on one GPU.

    python tools/bench_tpsa_poromech.py [--launches 10] [--warmup 2] [--tol 1e-8] [--maxiter 2000] [--small]

Meshes: the bench mesh (``structured_tet_grid((55, 55, 55))``, 998,250 tetrahedra) and a Cartesian 100^3 grid with the
mechanical faces of tools/bench_tpsa.py, a seeded lambda field exp(N(0, 1)), a seeded permeability exp(N(0, 0.25)),
Dirichlet pressure on the two x-sides, a seeded fluid source and the fluid constants of the poromechanics fixtures.
Per mesh one JSON line with

* the device, its power limit and SM clock limit (read in the same run),
* ``discretize`` (MPFA, TPSA face terms, the mechanics rows, the fluid-row pattern on the first call): wall clock to
  the end of the call, first call and median of later calls,
* one ``linearize`` end to end (upwinding from the iterate, the AD fluid mass balance, b0 - A x, the fluid rows): wall
  clock to a device synchronise, median; and the fluid-row kernel alone: CUDA events, median,
* one block-Jacobi BiCGStab solve of the first Newton update: iterations and status as they come out,
* the host path it replaces (tetrahedral mesh only): ``pb.Tpsa`` + ``pb.Mpfa`` discretization to scipy and the scipy
  assembly of the mechanics rows and of the linear part of the fluid rows.

``--small`` runs tiny meshes (a rehearsal of the script, not a measurement)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import porepy_b200 as pb  # noqa: E402
from porepy_b200 import _lib  # noqa: E402
from bench_tpsa import device_info, problem  # noqa: E402


def poro_problem(g, seed=13):
    nc, nf = g.num_cells, g.num_faces
    bc, mu = problem(g)
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.standard_normal(nc))
    bf = np.asarray(g.get_all_boundary_faces(), np.int64)
    x = g.face_centers[0, bf]
    dirf = bf[(x < x.min() + 1e-9) | (x > x.max() - 1e-9)]
    is_dir = np.zeros(nf, bool)
    is_dir[dirf] = True
    is_neu = np.zeros(nf, bool)
    is_neu[bf] = True
    is_neu[dirf] = False
    from types import SimpleNamespace
    fbc = SimpleNamespace(is_dir=is_dir, is_neu=is_neu, is_rob=np.zeros(nf, bool), is_internal=np.zeros(nf, bool),
                          robin_weight=np.ones(nf), bc_type="scalar", num_faces=nf)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.exp(0.5 * rng.standard_normal(nc))),
                                           "bc": fbc})
    pb.initialize_data(data, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
    fluid = dict(compressibility=0.05, density=1.7, viscosity=1.3, reference_pressure=0.3)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.7, bulk_modulus=3.0)
    mech = np.zeros((3, nf))
    rob = np.asarray(bc.is_rob, bool)[2]
    mech[2, rob] = -1e-3 * g.face_areas[rob]
    return pb.TpsaPoromechanics(g, data, fluid, solid, np.where(is_dir, rng.random(nf), 0.0), mech.ravel("F"), fbc,
                                np.where(is_dir, 1.7 / 1.3, 0.0), fluid_source=rng.standard_normal(nc) * g.cell_volumes)


def host_path_seconds(prob) -> float:
    """pb.Tpsa + pb.Mpfa discretization (matrices to scipy) and the scipy assembly of the mechanics rows and of the
    linear part of the fluid rows (div @ flux and the p_t / p storage diagonals), field-wise."""
    g, data = prob.sd, prob.data
    nd, nc = g.dim, g.num_cells
    nr = 3 if nd == 3 else 1
    C = data[pb.PARAMETERS]["mechanics"]["fourth_order_tensor"]
    t0 = time.perf_counter()
    pb.Tpsa("mechanics").discretize(g, data)
    pb.Mpfa("flow").discretize(g, data)
    M = data[pb.DISCRETIZATION_MATRICES]["mechanics"]
    F = data[pb.DISCRETIZATION_MATRICES]["flow"]
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr = sps.kron(div, sps.eye(nd)).tocsr(), sps.kron(div, sps.eye(nr)).tocsr()
    vol = g.cell_volumes
    a_l = vol * prob.alpha / C.lmbda
    A = sps.bmat([[-dn @ M["stress"], -dn @ M["stress_rotation"], -dn @ M["stress_total_pressure"], None],
                  [dr @ M["rotation_displacement"], dr @ M["rotation_rotation"] - sps.diags(np.repeat(vol / C.mu, nr)),
                   None, None],
                  [div @ M["solid_mass_displacement"], None,
                   div @ M["solid_mass_total_pressure"] - sps.diags(vol / C.lmbda), sps.diags(-a_l)],
                  [None, None, sps.diags(a_l), div @ sps.csr_matrix(F["flux"]) + sps.diags(a_l * prob.alpha)]]).tocsr()
    assert A.shape[0] == (nd + nr + 2) * nc
    return time.perf_counter() - t0


def bench(name, g, args, info, host_path: bool) -> dict:
    import torch
    prob = poro_problem(g)
    n, bs = prob.num_dofs, prob.block_size
    walls = []
    for _ in range(args.warmup + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        prob.discretize()
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    rng = np.random.default_rng(5)
    x_prev = torch.zeros(n, dtype=torch.float64, device="cuda")
    x = torch.as_tensor(1e-3 * rng.standard_normal(n), device="cuda")
    lin, fluid_ms = [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(args.warmup + args.launches):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        J, rhs = prob.linearize(x, x_prev, 0.25)
        torch.cuda.synchronize()
        if i >= args.warmup:
            lin.append(time.perf_counter() - t0)
    eq = prob.fluid_equation(x, x_prev, 0.25)
    jf, neg = eq.jac, -eq.val
    for i in range(args.warmup + args.launches):
        e0.record()
        prob._fg.tpsa_poro_fluid_rows(prob.A, jf, neg, rhs, prob._missing)
        e1.record()
        e1.synchronize()
        if i >= args.warmup:
            fluid_ms.append(e0.elapsed_time(e1))
    assert int(prob._missing.sum()) == 0
    from porepy_b200 import krylov
    J, rhs = prob.linearize(x_prev, x_prev, 0.25)
    loc = krylov.LocalSystem(0, 1, np.arange(n), np.zeros(0, np.int64), J, [0], [np.zeros(0, np.int64)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dx, sinfo = krylov.solve_local(loc, rhs, tol=args.tol, maxiter=args.maxiter,
                                   block_inv=(J.block_diagonal_inverse(bs), bs))
    torch.cuda.synchronize()
    solve_s = time.perf_counter() - t0
    out = {
        "mesh": name, "cells": g.num_cells, "faces": g.num_faces, **info, "rows": int(n), "nnz": int(J.nnz),
        "nnz_per_cell": J.nnz / g.num_cells,
        "discretize_first_call_s_incl_pattern": walls[0], "discretize_later_s": float(np.median(walls[1:])),
        "linearize_end_to_end_s_median": float(np.median(lin)), "linearize_s_min": float(np.min(lin)),
        "fluid_row_kernel_ms_median": float(np.median(fluid_ms)), "fluid_row_kernel_ms_min": float(np.min(fluid_ms)),
        "launches": len(lin), "bicgstab_tol": args.tol, "bicgstab_converged": bool(sinfo["converged"]),
        "bicgstab_iterations": int(sinfo["iterations"]), "bicgstab_breakdown": bool(sinfo.get("breakdown", False)),
        "bicgstab_s": solve_s,
    }
    del J, rhs, dx, jf, neg, eq
    out["host_path_discretize_plus_scipy_assembly_s"] = (host_path_seconds(prob) if host_path
                                                         else "not measured on this mesh")
    del prob
    torch.cuda.empty_cache()
    _lib.load().pb_device_pool_trim()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--maxiter", type=int, default=2000)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()
    _lib.require_gpu()
    info = device_info()
    meshes = ([("structured_tet_grid((2,2,2))", pb.structured_tet_grid((2, 2, 2)), True),
               ("cart_grid_3d((3,3,3))", pb.cart_grid_3d((3, 3, 3)), False)] if args.small else
              [("structured_tet_grid((55,55,55))", pb.structured_tet_grid((55, 55, 55)), True),
               ("cart_grid_3d((100,100,100))", pb.cart_grid_3d((100, 100, 100)), False)])
    for name, g, host in meshes:
        print(json.dumps(bench(name, g, args, info, host)), flush=True)


if __name__ == "__main__":
    main()
