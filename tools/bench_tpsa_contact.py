"""Time TPSA elasticity with fractures in frictional contact on one GPU: the assembly of the Jacobian
(``pb_tpsa_contact_system``), the per-step contact rows, ``linearize`` and the device GMRES with the grouped block-Jacobi
of ``TpsaFracturedMomentumBalance.preconditioner_groups()``.

    python tools/bench_tpsa_contact.py [--cases 16 32 2d256] [--restart 30] [--maxiter 3000] [--out FILE]

The problems are live ``pp.MomentumBalance`` + ``TpsaMomentumBalanceMixin`` models of the unmodified reference
(oracle/_ref): ``16`` / ``32`` are the unit cube of tools/make_contact_golden.py (``Model``, sliding load) on size^3
matrix cells, ``2d256`` the unit square on 256 x 256 cells with a vertical line fracture (``Model2d``, sliding load),
through ``model_bridge.tpsa_fractured_momentum_from_model``.  Per case: the first and a later ``pb_tpsa_contact_system``
wall time with the device times of its face kernel and row writes (CUDA events); then one time step of semismooth
Newton, with per Newton step

* ``linearize_s``: ``linearize`` (the contact laws on the AD chain, b0 - A x, the contact rows), wall clock to a device
  synchronise, and ``rows_ms``: the contact-row kernel alone (``pb_tpsa_contact_rows``), CUDA events;
* ``gmres_ms``, ``iterations``, ``restarts``, ``converged``, ``relres``: the GMRES solve (preconditioner set-up included),
  CUDA events;
* at 16^3 only, ``host_s``: the host path, ``DeviceCsr.to_scipy()`` plus scipy ``spsolve``, wall clock.

The Newton loop stops at the first GMRES that does not converge; that step is the last record, so a failed solve is
reported, not hidden, and no case waits on a host solve of a large system.  Every Newton record also goes to stderr as it
is taken.  The card name and its power limit are read in the
same run.  One JSON line per case on stdout; ``--out`` also writes the list of them to a file."""
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


def build_problem(case: str):
    import make_contact_golden as gc
    from make_contact_golden import pp
    from porepy_b200.porepy_plugin import plugin
    if case.startswith("2d"):
        n = int(case[2:])

        class Base(gc.Model2d):
            def set_geometry(self):
                self.set_domain()
                self.mdg = pp.meshing.cart_grid([np.array([[0.5, 0.5], [0.25, 0.75]])], [n, n], physdims=[1, 1])
                self.nd = self.mdg.dim_max()
                pp.set_local_coordinate_projections(self.mdg)
                self.set_well_network()
    else:
        n = int(case)

        class Base(gc.Model):
            def meshing_arguments(self):
                return {"cell_size": 1.0 / n}
    M = type("Bench", (pp.models.momentum_balance.TpsaMomentumBalanceMixin, Base), {})
    solid = pp.SolidConstants(lame_lambda=2.0, shear_modulus=1.5, friction_coefficient=0.4, fracture_gap=1e-4,
                              dilation_angle=0.1)
    model = M({"times_to_export": [], "time_manager": pp.TimeManager([0, 1.0], 1.0, constant_dt=True),
               "material_constants": {"solid": solid}})
    model.prepare_simulation()
    model.time_manager.increase_time()
    model.time_manager.increase_time_index()
    prob, cm, _ = plugin(pp).tpsa_fractured_momentum_from_model(model)
    x_prev = model.equation_system.get_variable_values(time_step_index=0)[cm]
    return prob, x_prev


def run(case: str, restart: int, maxiter: int, newton_tol: float = 1e-10, max_newton: int = 30) -> dict:
    import torch
    from porepy_b200 import ad, krylov
    t0 = time.perf_counter()
    prob, x_prev = build_problem(case)
    setup_s = time.perf_counter() - t0
    assembly = []
    for _ in range(3):                       # the first call builds the row pattern, the later ones reuse it
        torch.cuda.synchronize()
        t = time.perf_counter()
        prob.discretize()
        torch.cuda.synchronize()
        assembly.append(dict(wall_s=time.perf_counter() - t, face_terms_ms=prob.last_timing["face_terms_ms"],
                             rows_ms=prob.last_timing["rows_ms"]))
    groups = prob.preconditioner_groups()
    x_prev = torch.as_tensor(x_prev, dtype=torch.float64, device="cuda")
    x = x_prev.clone()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    steps, r0, host = [], None, case == "16"
    for it in range(max_newton + 1):
        torch.cuda.synchronize()
        t = time.perf_counter()
        J, rhs = prob.linearize(x, x_prev)
        torch.cuda.synchronize()
        lin_s = time.perf_counter() - t
        jac, neg_res = ad.assemble(prob.contact_equations(x, x_prev))
        scratch = rhs.clone()
        ev[0].record()
        prob._fg.tpsa_contact_rows(J, jac, neg_res, scratch, prob._missing)
        ev[1].record()
        rn = float(torch.linalg.vector_norm(rhs))
        r0 = rn if r0 is None else r0
        rec = {"newton": it, "residual": rn, "linearize_s": lin_s}
        torch.cuda.synchronize()
        rec["rows_ms"] = ev[0].elapsed_time(ev[1])
        if rn <= newton_tol * max(r0, 1e-300):
            steps.append(rec)
            break
        ev[2].record()
        dx, info = krylov.gmres(J, rhs, krylov.GroupedBlockJacobi(J, groups), tol=1e-12, restart=restart,
                                maxiter=maxiter)
        ev[3].record()
        torch.cuda.synchronize()
        rec.update(gmres_ms=ev[2].elapsed_time(ev[3]), iterations=info["iterations"], restarts=info["restarts"],
                   converged=info["converged"], breakdown=info["breakdown"], relres=info["relres"])
        if host:
            t = time.perf_counter()
            spla.spsolve(J.to_scipy().tocsc(), rhs.cpu().numpy())
            rec["host_s"] = time.perf_counter() - t
        steps.append(rec)
        print(json.dumps({"case": case, **rec}), file=sys.stderr, flush=True)
        if not info["converged"]:            # reported, not replaced: the time step ends at the first failed solve
            break
        x = x + dx
    return {"case": case, "matrix_cells": int(prob.nc), "fracture_cells": int(sum(f.num_cells for f in prob.fractures)),
            "unknowns": int(prob.num_dofs), "groups": int(groups.num_groups), "nnz_J": int(J.nnz),
            "model_setup_s": setup_s, "assembly": assembly, "restart": restart, "maxiter": maxiter, "newton": steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["16", "32", "2d256"])
    ap.add_argument("--restart", type=int, default=30)
    ap.add_argument("--maxiter", type=int, default=3000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = device_info()
    results = []
    for case in a.cases:
        res = {**info, **run(case, a.restart, a.maxiter)}
        print(json.dumps(res), flush=True)
        results.append(res)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
