"""Time the device assembly and solve of the TPSA three-field elasticity system (``porepy_b200.TpsaElasticity``,
``pb_tpsa_system`` / ``pb_tpsa_rhs``) on one GPU.

    python tools/bench_tpsa_solve.py [--launches 20] [--warmup 3] [--tol 1e-8] [--maxiter 5000] [--small]

Meshes: the bench mesh (``structured_tet_grid((55, 55, 55))``, 998,250 tetrahedra) and a Cartesian 100^3 grid, with the
faces of tools/bench_tpsa.py (Dirichlet west, a roller south, Robin top, Neumann elsewhere), its seeded shear modulus, a
seeded lambda field exp(N(0, 1)), a body force of -1 per unit volume in z and a traction of -1e-3 per unit area in z on
the Robin faces.  Per mesh one JSON line with

* the device, its power limit and SM clock limit (read in the same run),
* stage 1 (face terms, ``tpsa_kernel``) and stage 2 (row gather, ``tpsa_system_kernel``): CUDA events, median and min
  over ``--launches`` assemblies after ``--warmup``,
* the rows and non-zeros of A,
* the first ``pb_tpsa_system`` call on a new grid handle (builds the row pattern) against the median of later calls,
  wall clock to the end of the call,
* the block-diagonal inverse (7 x 7 per cell): CUDA events, median of ``--launches``,
* block-Jacobi BiCGStab from x = 0 to ``--tol``: iterations, seconds, converged or not, the true relative residual
  recomputed on the device,
* host arrays -> solution on the host, end to end, on a new ``TpsaElasticity`` (grid handle, pattern, assembly, block
  inverse, solve, download),
* the host path it replaces, on the tetrahedral mesh only: ``pb.Tpsa.discretize`` (GPU face kernel, matrices to scipy)
  plus the scipy assembly of A (a host direct solve at this size is not run).

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


def inputs(g):
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    bc, mu = problem(g)
    lam = np.exp(np.random.default_rng(11).standard_normal(nc))
    bcv = np.zeros((nd, nf))
    rob = np.asarray(bc.is_rob, bool)[nd - 1]
    bcv[nd - 1, rob] = -1e-3 * g.face_areas[rob]
    f = np.zeros((nd, nc))
    f[nd - 1] = -g.cell_volumes
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": pb.FourthOrderTensor(mu, lam), "bc": bc})
    return data, bcv.ravel("F"), f.ravel("F")


def host_path_seconds(g, data, bcv, f) -> float:
    """pb.Tpsa.discretize (matrices to the host as scipy CSR) + the scipy assembly of A and b in field-wise order."""
    nd, nc = g.dim, g.num_cells
    nr = 3 if nd == 3 else 1
    C = data[pb.PARAMETERS]["mech"]["fourth_order_tensor"]
    t0 = time.perf_counter()
    pb.Tpsa("mech").discretize(g, data)
    M = data[pb.DISCRETIZATION_MATRICES]["mech"]
    div = sps.csr_matrix(g.cell_faces).T.tocsr()
    dn, dr = sps.kron(div, sps.eye(nd)).tocsr(), sps.kron(div, sps.eye(nr)).tocsr()
    vol = g.cell_volumes
    A = sps.bmat([[-dn @ M["stress"], -dn @ M["stress_rotation"], -dn @ M["stress_total_pressure"]],
                  [dr @ M["rotation_displacement"], dr @ M["rotation_rotation"] - sps.diags(np.repeat(vol / C.mu, nr)),
                   None],
                  [div @ M["solid_mass_displacement"], None,
                   div @ M["solid_mass_total_pressure"] - sps.diags(vol / C.lmbda)]]).tocsr()
    b = np.concatenate([dn @ (M["bound_stress"] @ bcv) + f, -(dr @ (M["bound_rotation_displacement"] @ bcv)),
                        -(div @ (M["bound_mass_displacement"] @ bcv))])
    assert A.shape[0] == b.size == (nd + nr + 1) * nc
    return time.perf_counter() - t0


def bench(name, g, args, info, host_path: bool) -> dict:
    import torch
    nd = g.dim
    bs = nd + (3 if nd == 3 else 1) + 1
    data, bcv, f = inputs(g)
    prob = pb.TpsaElasticity(g, data, "mech", bcv, body_force=f)
    walls, s1, s2 = [], [], []
    for i in range(args.warmup + args.launches):
        t0 = time.perf_counter()
        prob.discretize()
        walls.append(time.perf_counter() - t0)
        if i >= args.warmup:
            s1.append(prob.last_timing["face_terms_ms"])
            s2.append(prob.last_timing["rows_ms"])
    A, b = prob.assemble()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    inv_ms = []
    for i in range(args.warmup + args.launches):
        e0.record()
        A.block_diagonal_inverse(bs)
        e1.record()
        e1.synchronize()
        if i >= args.warmup:
            inv_ms.append(e0.elapsed_time(e1))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    x, sinfo = prob.solve(tol=args.tol, maxiter=args.maxiter)
    torch.cuda.synchronize()
    solve_s = time.perf_counter() - t0
    true_rel = float(torch.linalg.norm(b - A @ x) / torch.linalg.norm(b))
    del x
    # host arrays -> solution on the host, on a new problem (new grid handle: the pattern is built again)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    p2 = pb.TpsaElasticity(g, data, "mech", bcv, body_force=f)
    x2, info2 = p2.solve(tol=args.tol, maxiter=args.maxiter)
    xh = x2.cpu().numpy()
    e2e_s = time.perf_counter() - t0
    assert xh.size == A.shape[0]
    del p2, x2
    out = {
        "mesh": name, "cells": g.num_cells, "faces": g.num_faces, **info,
        "stage1_face_terms_ms_median": float(np.median(s1)), "stage1_ms_min": float(np.min(s1)),
        "stage2_row_gather_ms_median": float(np.median(s2)), "stage2_ms_min": float(np.min(s2)),
        "launches": len(s1), "rows": int(A.shape[0]), "nnz": int(A.nnz), "nnz_per_cell": A.nnz / g.num_cells,
        "system_first_call_s_incl_pattern": walls[0], "system_later_calls_s_median": float(np.median(walls[1:])),
        "block_inverse_ms_median": float(np.median(inv_ms)),
        "bicgstab_tol": args.tol, "bicgstab_converged": bool(sinfo["converged"]),
        "bicgstab_iterations": int(sinfo["iterations"]), "bicgstab_breakdown": bool(sinfo["breakdown"]),
        "bicgstab_s": solve_s, "bicgstab_recurrence_relres": float(sinfo["relres"]), "true_relres": true_rel,
        "end_to_end_host_arrays_to_solution_s": e2e_s, "end_to_end_converged": bool(info2["converged"]),
    }
    del A, b, prob
    torch.cuda.empty_cache()
    _lib.load().pb_device_pool_trim()
    out["host_path_discretize_plus_scipy_assembly_s"] = (host_path_seconds(g, data, bcv, f) if host_path
                                                         else "not measured on this mesh")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tol", type=float, default=1e-8)
    ap.add_argument("--maxiter", type=int, default=5000)
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
