"""Time the two-point stress approximation (``porepy_b200.Tpsa``, csrc/tpsa_face.cuh) on one GPU.

    python tools/bench_tpsa.py [--launches 20] [--warmup 3] [--calls 5] [--small]

Meshes: the bench mesh (``structured_tet_grid((55, 55, 55))``, 998,250 tetrahedra) and a Cartesian 100^3 grid, each
with Dirichlet, roller, Robin and Neumann faces and a seeded shear modulus.  Per mesh it prints one JSON line with

* the device and its power limit (read in the same run),
* kernel time: CUDA events around ``tpsa_kernel``, median and min over ``--launches`` calls after ``--warmup``,
* algorithmic bytes (every input once, every output value once, from the shapes) and bytes/s over the kernel time
  against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (a share of that figure, not a measured peak),
* ``pb.Tpsa.discretize`` end to end (host arrays in, scipy CSR matrices out): the first call on the grid, which also
  builds the index patterns, and the median of ``--calls`` later calls; and the time of a
  device-to-host copy of the output bytes into page-locked memory alone, as its share of the end-to-end time,
* the unmodified reference's ``pp.Tpsa.discretize`` on a 3,072-cell sample (``structured_tet_grid((8, 8, 8))``) when
  oracle/_ref is present, else "not measured".

``--small`` runs tiny meshes (a rehearsal of the script, not a measurement)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import porepy_b200 as pb  # noqa: E402
from porepy_b200 import _lib, fv  # noqa: E402

HBM_DATASHEET = 3.35e12


def device_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (s.strip() for s in out[0].split(","))
        return {"device": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"device": "unknown", "power_limit": f"not read ({e})"}


def problem(g, seed=7):
    nd, nf = g.dim, g.num_faces
    bf = g.get_all_boundary_faces()
    xf = g.face_centers[:, bf]
    bc = pb.BoundaryConditionVectorial(g)
    west = bf[xf[0] < 1e-10]
    south = bf[(xf[1] < 1e-10) & (xf[0] > 1e-10)]
    top = bf[(xf[2] > 1 - 1e-10) & (xf[0] > 1e-10) & (xf[1] > 1e-10)]
    bc.is_dir[:, west], bc.is_neu[:, west] = True, False
    bc.is_dir[1, south], bc.is_neu[1, south] = True, False
    bc.is_rob[:, top], bc.is_neu[:, top] = True, False
    rng = np.random.default_rng(seed)
    w = np.zeros((nd, nd, nf))
    for i in range(nd):
        w[i, i] = 0.2 + 5 * rng.random(nf)
    bc.robin_weight = w
    mu = np.exp(rng.standard_normal(g.num_cells))
    return bc, mu


def algorithmic_bytes(nd, nc, nf, nnz, robin: bool) -> tuple:
    inputs = (3 * nf * 8 * 2 + nf * 8 + 3 * nc * 8      # face normals, face centres, face areas, cell centres
              + nc * 8 + nd * nf + nf                    # mu, codes, face flags
              + (nd * nf * 8 if robin else 0)            # Robin diagonals
              + 2 * nf * 4 + (nf + 1) * 4)               # face -> cell table, fc_indptr
    outputs = 8 * sum(fv.tpsa_value_counts(nd, nf, nnz))
    return inputs, outputs


def d2h_seconds(nbytes: int, reps: int = 5) -> float:
    import torch
    n = nbytes // 8
    dev = torch.empty(n, dtype=torch.float64, device="cuda")
    host = torch.empty(n, dtype=torch.float64, pin_memory=True)
    host.copy_(dev, non_blocking=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        host.copy_(dev, non_blocking=True)
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(ts))


def reference_sample_seconds(small: bool):
    from ref_loader import load_porepy, reference_available
    from oracle.ref_loader import reference_grid
    if not reference_available():
        return "not measured (oracle/_ref not present)"
    pp = load_porepy()
    g = pb.structured_tet_grid((2, 2, 2) if small else (8, 8, 8))
    bc, mu = problem(g)
    r = reference_grid(pp, g)
    rbc = pp.BoundaryConditionVectorial(r)
    rbc.is_dir, rbc.is_neu, rbc.is_rob = bc.is_dir.copy(), bc.is_neu.copy(), bc.is_rob.copy()
    rbc.robin_weight = bc.robin_weight.copy()
    data = pp.initialize_data({}, "mech", {"fourth_order_tensor": pp.FourthOrderTensor(mu, np.ones_like(mu)),
                                           "bc": rbc})
    pp.Tpsa("mech").discretize(r, data)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        pp.Tpsa("mech").discretize(r, data)
        ts.append(time.perf_counter() - t0)
    return {"cells": g.num_cells, "seconds_median": float(np.median(ts))}


def bench(name, g, args, info) -> dict:
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    bc, mu = problem(g)
    codes, robin = fv.tpsa_bc_arrays(bc, nd, nf)
    import scipy.sparse as sps
    fc = sps.csr_matrix(g.cell_faces)
    fc.sort_indices()
    ip = fc.indptr
    flags = np.zeros(nf, np.uint8)
    flags[g.get_all_boundary_faces()] = 1
    fg = fv.FaceGrid(g)
    ms = []
    for i in range(args.warmup + args.launches):
        _, k = fg.tpsa(nd, mu, codes, robin, flags, ip, g.face_areas)
        if i >= args.warmup:
            ms.append(k)
    bin_, bout = algorithmic_bytes(nd, nc, nf, int(ip[-1]), robin is not None)
    kmed = float(np.median(ms)) / 1e3
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": pb.FourthOrderTensor(mu, np.ones_like(mu)),
                                           "bc": bc})
    disc = pb.Tpsa("mech")
    t0 = time.perf_counter()
    disc.discretize(g, data)        # builds the grid's index patterns, reused by the later calls
    first_s = time.perf_counter() - t0
    e2e = []
    for _ in range(args.calls):
        t0 = time.perf_counter()
        disc.discretize(g, data)
        e2e.append(time.perf_counter() - t0)
    e2e_s = float(np.median(e2e))
    d2h = d2h_seconds(bout)
    return {
        "mesh": name, "cells": nc, "faces": nf, **info,
        "kernel_ms_median": kmed * 1e3, "kernel_ms_min": float(np.min(ms)), "kernel_launches": len(ms),
        "bytes_in": bin_, "bytes_out": bout,
        "bytes_per_s": (bin_ + bout) / kmed,
        "share_of_datasheet_hbm_3.35TBps": (bin_ + bout) / kmed / HBM_DATASHEET,
        "discretize_first_call_s": first_s,
        "discretize_end_to_end_s_median": e2e_s, "discretize_calls": len(e2e),
        "d2h_of_outputs_pinned_s": d2h, "d2h_share_of_end_to_end": d2h / e2e_s,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
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
    print(json.dumps({"reference_tpsa_discretize_sample": reference_sample_seconds(args.small)}), flush=True)


if __name__ == "__main__":
    main()
