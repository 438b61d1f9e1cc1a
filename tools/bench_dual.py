"""Time ``pb.MVEM`` / ``pb.RT0`` on the GPU: 998,250 tetrahedra (both schemes) and a Cartesian 100^3 grid (MVEM).
Prints one JSON line per case with the card name and power limit read in the same run: the per-cell kernel time
(CUDA events, median of 20), the mass-pattern build of the first call, ``discretize`` wall time of the first and of
later calls, the saddle-point assembly on the device (first and later calls) and with the host formulas, and the algorithmic bytes (inputs read once, outputs written once) over
the kernel time against 3.35 TB/s.  With ``--reference`` also times the unmodified reference's ``discretize`` on a
3,072-tetrahedron and a 16^3 grid from oracle/_ref (host CPU).
   python tools/bench_dual.py [--reference]"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import porepy_b200 as pb  # noqa: E402
from porepy_b200 import fv  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:
        return f"unknown ({e})"


def case(label, g, cls):
    rng = np.random.default_rng(0)
    nc = g.num_cells
    k = pb.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc), 0.2 * rng.random(nc),
                             0.2 * rng.random(nc), 0.2 * rng.random(nc))
    bf = g.get_all_boundary_faces()
    bc = pb.BoundaryCondition(g, bf, ["dir"] * bf.size)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc, "bc_values": np.zeros(g.num_faces)})
    d = cls("flow")
    t0 = time.perf_counter()
    d.discretize(g, data)
    first = time.perf_counter() - t0
    pattern_s = d.last_timing["pattern_s"]
    walls, kms = [], []
    for _ in range(20):
        t0 = time.perf_counter()
        d.discretize(g, data)
        walls.append(time.perf_counter() - t0)
        kms.append(d.last_timing["kernel_ms"])
    dev = []
    for _ in range(3):   # the first call also builds the system pattern
        t0 = time.perf_counter()
        A, _ = d.assemble_matrix_rhs(g, data)
        dev.append(time.perf_counter() - t0)
    assert A.device_csr is not None
    mass = data[pb.DISCRETIZATION_MATRICES]["flow"]["mass"]
    mass.data   # download: the host formulas from here on
    t0 = time.perf_counter()
    d.assemble_matrix_rhs(g, data)
    asm = time.perf_counter() - t0
    ncf = int(abs(g.cell_faces).sum())
    # inputs: geometry (3 nodes, 3+3 per face, 3+1 per cell), tensor 9 per cell, topology (int32); outputs: values
    nbytes = 8 * (3 * g.num_nodes + 6 * g.num_faces + 13 * nc + mass.nnz + 3 * ncf) + 4 * (3 * ncf + mass.nnz)
    km = float(np.median(kms))
    return dict(case=label, cells=nc, kernel_ms_median=km, pattern_first_s=pattern_s, discretize_first_s=first,
                discretize_repeat_s=float(np.median(walls)), device_assembly_first_s=dev[0],
                device_assembly_repeat_s=float(np.median(dev[1:])), host_assembly_s=asm,
                achieved_TBps=nbytes / (km * 1e-3) / 1e12, share_of_3_35TBps=nbytes / (km * 1e-3) / 3.35e12)


def reference_times():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from ref_loader import load_porepy
    pp = load_porepy()
    out = {}
    for label, g, cls in [("ref_mvem_tet3072", pp.StructuredTetrahedralGrid([8, 8, 8]), pp.MVEM),
                          ("ref_rt0_tet3072", pp.StructuredTetrahedralGrid([8, 8, 8]), pp.RT0),
                          ("ref_mvem_cart16", pp.CartGrid([16, 16, 16]), pp.MVEM)]:
        g.compute_geometry()
        data = {pp.PARAMETERS: {"flow": {"second_order_tensor": pp.SecondOrderTensor(np.ones(g.num_cells))}},
                pp.DISCRETIZATION_MATRICES: {"flow": {}}}
        t0 = time.perf_counter()
        cls("flow").discretize(g, data)
        s = time.perf_counter() - t0
        out[label] = dict(cells=g.num_cells, seconds=s, cells_per_s=g.num_cells / s)
    return out


def main():
    info = dict(gpu=card())
    rows = [case("mvem_tet998k", pb.structured_tet_grid([55, 55, 55]), pb.MVEM),
            case("rt0_tet998k", pb.structured_tet_grid([55, 55, 55]), pb.RT0),
            case("mvem_cart100", pb.cart_grid_3d([100, 100, 100]), pb.MVEM)]
    for r in rows:
        print(json.dumps({**info, **r}))
    if "--reference" in sys.argv:
        print(json.dumps({**info, "reference": reference_times()}))


if __name__ == "__main__":
    main()
