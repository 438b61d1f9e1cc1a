"""Measure the hybridized solve of the mixed schemes (``MVEM.solve`` / ``RT0.solve``, csrc/dual_hybrid.cuh) on
998,250 tetrahedra (MVEM and RT0) and on 100^3 hexahedra (MVEM): a linear pressure with Dirichlet data on the whole
boundary and a random source.  Reports the condensation and recovery kernel times (CUDA events, median of 20), the
BiCGStab iterations and time, the wall time from host arrays to [u; p] and algorithmic bytes over kernel time, with the
card's name and power limit read in the same run.  One JSON line per workload.
   python tools/bench_dual_hybrid.py [--out FILE]"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        limit = "unknown"
    return name, limit


def workload(which):
    import porepy_b200 as pb
    from porepy_b200 import _lib, fv
    from porepy_b200.grid import cart_grid_3d, structured_tet_grid
    g = cart_grid_3d([100, 100, 100]) if which == "mvem_cart" else structured_tet_grid([55, 55, 55])
    d = pb.RT0("flow") if which.startswith("rt0") else pb.MVEM("flow")
    a, p0 = np.array([0.7, -1.3, 0.4]), 0.25
    bf = g.get_all_boundary_faces()
    bcv = np.zeros(g.num_faces)
    bcv[bf] = a @ g.face_centers[:, bf] + p0
    data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor(np.ones(g.num_cells)),
                                           "bc": pb.BoundaryCondition(g, bf, ["dir"] * bf.size), "bc_values": bcv})
    d.discretize(g, data)
    _, b = d.assemble_matrix_rhs(g, data)
    b = b.copy()
    b[g.num_faces:] += np.random.default_rng(9).standard_normal(g.num_cells) * g.cell_volumes
    up = d.solve(g, data, b)           # warm-up: loads the kernels, builds nothing that is kept
    up = d.solve(g, data, b)
    info = dict(d.last_solve)
    dg = fv.DualGrid.for_grid(g)
    codes = fv.dual_bc_codes(g, data["parameters"]["flow"]["bc"])
    rw, areas = np.ones(g.num_faces), g.face_areas
    cond, rec = [], []
    lam = None
    for _ in range(20):
        H, rhs, _, ms = dg.hybrid_system(_lib.DUAL_HYBRID_SADDLE, None, codes, rw, areas, b)
        cond.append(ms)
        if lam is None:
            from porepy_b200.krylov import bicgstab_solver
            lam = fv._to_host(bicgstab_solver(1e-10, 5000)(H, rhs))
        _, ms = dg.hybrid_recover(_lib.DUAL_HYBRID_SADDLE, None, codes, b, lam)
        rec.append(ms)
    nc, nf, ncf = g.num_cells, g.num_faces, int(dg.cf_ip[-1])
    nmass = int(dg.mass_pattern()[1].size)
    # algorithmic bytes: topology (cell_faces, face_nodes of the cell), geometry per cell and face read once, the
    # written face matrix values (8 B per entry) and rhs; the recovery reads the same plus lambda and writes u, p
    geo_bytes = 8 * (nc * (3 + 1 + 9) + 2 * 3 * nf) + 4 * (2 * ncf + nc)
    cond_bytes = geo_bytes + 8 * nmass + 8 * (nf + nc) + 8 * nf
    rec_bytes = geo_bytes + 8 * (2 * nf + 2 * nc) + 8 * (nf + nc)
    mc, mr = float(np.median(cond)), float(np.median(rec))
    return dict(workload=which, cells=nc, faces=nf, face_nnz=nmass, condense_ms=mc, recover_ms=mr,
                condense_GBps=cond_bytes / mc / 1e6, recover_GBps=rec_bytes / mr / 1e6,
                bicgstab_iterations=info["iterations"], bicgstab_s=info["solve_s"], converged=info["converged"],
                face_residual=info["face_residual"], wall_s=info["wall_s"])


def main():
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    name, limit = card()
    lines = []
    for which in ("mvem_tet", "rt0_tet", "mvem_cart"):
        r = workload(which)
        r.update(card=name, power_limit=limit)
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
