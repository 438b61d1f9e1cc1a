"""Time the device Jacobian of the TPSA thermo-poromechanics model (``porepy_b200.TpsaThermoporomechanics``,
``pb_tpsa_thm_system`` / ``pb_tpsa_thm_balance_rows``) and its 9 x 9 block-Jacobi BiCGStab on one GPU.

    python tools/bench_tpsa_thm.py [--launches 10] [--warmup 2] [--tol 1e-8] [--maxiter 2000] [--small]

Meshes: the bench mesh (``structured_tet_grid((55, 55, 55))``, 998,250 tetrahedra) and a Cartesian 100^3 grid, with the
mechanical faces, lambda, permeability, Darcy boundary data and fluid source of tools/bench_tpsa_poromech.py, Dirichlet
temperatures on the two x-sides and the thermal constants of the thermo-poromechanics fixtures.  Per mesh one JSON line
with

* the device, its power limit and SM clock limit (read in the same run),
* ``discretize`` (Darcy and Fourier MPFA, TPSA face terms, the mechanics rows, the row pattern on the first call): wall
  clock to the end of the call, first call and median of later calls,
* one ``linearize`` end to end (both upwindings from the iterate, the AD mass and energy balances, b0 - A x, the balance
  rows): wall clock to a device synchronise, median; the balance-row kernel alone and the 9 x 9 block-inverse kernel
  alone: CUDA events, median,
* one block-Jacobi BiCGStab solve of the first Newton update: iterations and status as they come out.

``--small`` runs tiny meshes (a rehearsal of the script, not a measurement)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import porepy_b200 as pb  # noqa: E402
from porepy_b200 import _lib  # noqa: E402
from bench_tpsa import device_info  # noqa: E402
from bench_tpsa_poromech import poro_problem  # noqa: E402


def thm_problem(g, seed=13):
    """The poromechanics bench problem of ``bench_tpsa_poromech.poro_problem`` with the energy balance added."""
    p = poro_problem(g, seed)
    nf = g.num_faces
    fbc = p.bc_fluid_flux
    pb.initialize_data(p.data, "fourier", {"bc": fbc})
    rng = np.random.default_rng(seed + 1)
    fluid = dict(compressibility=0.05, density=1.7, viscosity=1.3, reference_pressure=0.3, thermal_expansion=0.2,
                 heat_capacity=2.0, conductivity=0.7, reference_temperature=0.4)
    solid = dict(reference_porosity=0.2, biot_coefficient=0.8, bulk_modulus=3.0, thermal_expansion=0.1,
                 heat_capacity=1.5, conductivity=1.1, density=2.5)
    t_bc = np.where(fbc.is_dir, rng.random(nf), 0.0)
    return pb.TpsaThermoporomechanics(g, p.data, fluid, solid, p.flow_bc, t_bc, p.mech_bc, fbc, p.ff_values, fbc,
                                      np.where(fbc.is_dir, 2.0 * (t_bc - 0.4) * 1.7 / 1.3, 0.0),
                                      fluid_source=p.fluid_source)


def bench(name, g, args, info) -> dict:
    import torch
    from porepy_b200 import ad, krylov
    prob = thm_problem(g)
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
    lin, rows_ms, inv_ms = [], [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(args.warmup + args.launches):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        J, rhs = prob.linearize(x, x_prev, 0.25)
        torch.cuda.synchronize()
        if i >= args.warmup:
            lin.append(time.perf_counter() - t0)
    jf, neg = ad.assemble(prob.balance_equations(x, x_prev, 0.25))
    for i in range(args.warmup + args.launches):
        e0.record()
        prob._fg.tpsa_thm_balance_rows(prob.A, jf, neg, rhs, prob._missing)
        e1.record()
        e1.synchronize()
        if i >= args.warmup:
            rows_ms.append(e0.elapsed_time(e1))
    assert int(prob._missing.sum()) == 0
    J, rhs = prob.linearize(x_prev, x_prev, 0.25)
    for i in range(args.warmup + args.launches):
        e0.record()
        minv = J.block_diagonal_inverse(bs)
        e1.record()
        e1.synchronize()
        if i >= args.warmup:
            inv_ms.append(e0.elapsed_time(e1))
    loc = krylov.LocalSystem(0, 1, np.arange(n), np.zeros(0, np.int64), J, [0], [np.zeros(0, np.int64)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dx, sinfo = krylov.solve_local(loc, rhs, tol=args.tol, maxiter=args.maxiter, block_inv=(minv, bs))
    torch.cuda.synchronize()
    solve_s = time.perf_counter() - t0
    out = {
        "mesh": name, "cells": g.num_cells, "faces": g.num_faces, **info, "rows": int(n), "nnz": int(J.nnz),
        "nnz_per_cell": J.nnz / g.num_cells,
        "discretize_first_call_s_incl_pattern": walls[0], "discretize_later_s": float(np.median(walls[1:])),
        "linearize_end_to_end_s_median": float(np.median(lin)), "linearize_s_min": float(np.min(lin)),
        "balance_row_kernel_ms_median": float(np.median(rows_ms)),
        "balance_row_kernel_ms_min": float(np.min(rows_ms)),
        "block_inverse_9x9_ms_median": float(np.median(inv_ms)), "block_inverse_9x9_ms_min": float(np.min(inv_ms)),
        "launches": len(lin), "bicgstab_tol": args.tol, "bicgstab_converged": bool(sinfo["converged"]),
        "bicgstab_iterations": int(sinfo["iterations"]), "bicgstab_breakdown": bool(sinfo.get("breakdown", False)),
        "bicgstab_s": solve_s,
    }
    del J, rhs, dx, jf, neg, minv, prob
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
    meshes = ([("structured_tet_grid((2,2,2))", pb.structured_tet_grid((2, 2, 2))),
               ("cart_grid_3d((3,3,3))", pb.cart_grid_3d((3, 3, 3)))] if args.small else
              [("structured_tet_grid((55,55,55))", pb.structured_tet_grid((55, 55, 55))),
               ("cart_grid_3d((100,100,100))", pb.cart_grid_3d((100, 100, 100)))])
    for name, g in meshes:
        print(json.dumps(bench(name, g, args, info)), flush=True)


if __name__ == "__main__":
    main()
