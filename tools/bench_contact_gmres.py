"""Time the device solve of the Newton updates of frictional contact (``krylov.gmres`` with the grouped block-Jacobi of
``FracturedMomentumBalance.preconditioner_groups()``) against the host path it replaces, on one GPU.

    python tools/bench_contact_gmres.py [--sizes 16 32 48] [--restart 30] [--maxiter 3000] [--out FILE]

The problem is a live ``pp.MomentumBalance`` of the unmodified reference (oracle/_ref): the unit cube on a Cartesian grid
of size^3 matrix cells, cut by the compressed and sheared fracture of tools/make_contact_golden.py (sliding load case),
turned into a device problem by ``model_bridge.fractured_momentum_from_model``.  One time step of semismooth Newton; for
every Newton step one record with

* ``assemble_s``: ``linearize`` (J and -R on the device), wall clock to a device synchronise,
* ``group_inv_ms``: the group-inverse kernel (``GroupedBlockJacobi``), CUDA events,
* ``gmres_ms``, ``iterations``, ``restarts``, ``converged``, ``relres``: the GMRES solve, CUDA events, as it comes out,
* ``host_s``: the host path in the same run, ``DeviceCsr.to_scipy()`` plus scipy ``spsolve``, wall clock,
* ``update_diff``: |dx_gmres - dx_host| / |dx_host|.

The Newton loop continues with the host update, so a GMRES that does not converge is reported and the step sequence is
the same for both solvers.  The card name and its power limit are read in the same run.  One JSON line per size on
stdout; ``--out`` also writes the list of them to a file."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse.linalg as spla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tpsa import device_info  # noqa: E402


def build_problem(size: int):
    import make_contact_golden as gc
    from make_contact_golden import pp
    from porepy_b200.porepy_plugin import plugin

    class Model(gc.Model):
        def meshing_arguments(self):
            return {"cell_size": 1.0 / size}
    solid = pp.SolidConstants(lame_lambda=2.0, shear_modulus=1.5, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1)
    model = Model({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 1.0, constant_dt=True),
                   "material_constants": {"solid": solid}})
    model.prepare_simulation()
    model.time_manager.increase_time()
    model.time_manager.increase_time_index()
    prob, cm = plugin(pp).fractured_momentum_from_model(model)
    x_prev = model.equation_system.get_variable_values(time_step_index=0)[cm]
    return prob, x_prev


def run(size: int, restart: int, maxiter: int, newton_tol: float = 1e-10, max_newton: int = 30) -> dict:
    import torch
    from porepy_b200 import krylov
    t0 = time.perf_counter()
    prob, x_prev = build_problem(size)
    setup_s = time.perf_counter() - t0
    prob.discretize()
    groups = prob.preconditioner_groups()
    x_prev = torch.as_tensor(x_prev, dtype=torch.float64, device="cuda")
    x = x_prev.clone()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    steps, r0 = [], None
    for it in range(max_newton + 1):
        torch.cuda.synchronize()
        t = time.perf_counter()
        J, rhs = prob.linearize(x, x_prev)
        torch.cuda.synchronize()
        assemble_s = time.perf_counter() - t
        rn = float(torch.linalg.vector_norm(rhs))
        r0 = rn if r0 is None else r0
        rec = {"newton": it, "residual": rn, "assemble_s": assemble_s}
        if rn <= newton_tol * max(r0, 1e-300):
            steps.append(rec)
            break
        ev[0].record()
        M = krylov.GroupedBlockJacobi(J, groups)
        ev[1].record()
        ev[2].record()
        dx, info = krylov.gmres(J, rhs, M, tol=1e-12, restart=restart, maxiter=maxiter)
        ev[3].record()
        torch.cuda.synchronize()
        t = time.perf_counter()
        dxh = spla.spsolve(J.to_scipy().tocsc(), rhs.cpu().numpy())
        host_s = time.perf_counter() - t
        rec.update(group_inv_ms=ev[0].elapsed_time(ev[1]), gmres_ms=ev[2].elapsed_time(ev[3]),
                   iterations=info["iterations"], restarts=info["restarts"], converged=info["converged"],
                   breakdown=info["breakdown"], relres=info["relres"], host_s=host_s,
                   update_diff=float(np.linalg.norm(dx.cpu().numpy() - dxh) / max(np.linalg.norm(dxh), 1e-300)))
        steps.append(rec)
        x = x + torch.as_tensor(dxh, device="cuda")
    return {"size": size, "matrix_cells": int(prob.nc), "fracture_cells": int(sum(f.num_cells for f in prob.fractures)),
            "unknowns": int(prob.num_dofs), "groups": int(groups.num_groups), "nnz_J": int(J.nnz),
            "model_setup_s": setup_s, "restart": restart, "maxiter": maxiter, "newton": steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 32, 48])
    ap.add_argument("--restart", type=int, default=30)
    ap.add_argument("--maxiter", type=int, default=3000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = device_info()
    results = []
    for size in a.sizes:
        res = {**info, **run(size, a.restart, a.maxiter)}
        print(json.dumps(res), flush=True)
        results.append(res)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
