"""Benchmark-size parity fixtures from the unmodified reference (run in the build container).

The golden cases of tools/make_golden.py are 36-48 cells.  This script runs ``pp.Mpfa / pp.Mpsa /
pp.Biot.discretize`` of the read-only reference on the sizes the benchmark configurations are built from
(Cartesian 32^3 = BASELINE config[0], structured tetrahedra 12^3 x 6 and 16^3 x 6, Biot 16^3) and stores a
DIGEST of every output matrix (tests/cases.py: ``digest_of``): M @ x and |M| @ 1 on a strided subset of the rows,
8 bilinear forms over all entries, 200 sampled rows entrywise -- under 1 MB per case instead of GB (ROW_THINNING).  Grid and parameters are regenerated from the seed on both sides
(tests/cases.py: ``digest_grid``, ``digest_params``); the reference is handed the very same arrays.

    python tools/make_digests.py [case ...]
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from ref_loader import load_porepy  # noqa: E402
from oracle.ref_loader import reference_grid  # noqa: E402

pp = load_porepy()
import cases  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


# every k-th of (at most 20,000 strided) rows in M @ x and |M| @ 1: the finest thinning that keeps each case under 1 MB
ROW_THINNING = {"digest_biot_cart16": 4, "digest_mpfa_cart32": 3, "digest_mpfa_tet12": 5, "digest_mpfa_tet16": 8,
                "digest_mpsa_cart32": 2, "digest_mpsa_tet12": 3, "digest_mpsa_tet16": 3}

def run(name):
    kind, dims, what = cases.DIGEST_CASES[name]
    g = cases.digest_grid(kind, dims)
    k, bc, C, vbc, alpha = cases.digest_params(g)
    r = reference_grid(pp, g)
    t0 = time.perf_counter()
    if what == "mpfa":
        rbc = pp.BoundaryCondition(r)
        rbc.is_dir, rbc.is_neu, rbc.is_rob = bc.is_dir.copy(), bc.is_neu.copy(), bc.is_rob.copy()
        rk = pp.SecondOrderTensor(np.ones(r.num_cells))
        rk.values = k.values.copy()
        data = pp.initialize_data({}, "flow", {"second_order_tensor": rk, "bc": rbc})
        pp.Mpfa("flow").discretize(r, data)
        mats = dict(data[pp.DISCRETIZATION_MATRICES]["flow"])
    else:
        rbc = pp.BoundaryConditionVectorial(r)
        rbc.is_dir, rbc.is_neu, rbc.is_rob = vbc.is_dir.copy(), vbc.is_neu.copy(), vbc.is_rob.copy()
        rC = pp.FourthOrderTensor(C.mu.copy(), C.lmbda.copy())
        assert np.array_equal(rC.values, C.values)
        prm = {"fourth_order_tensor": rC, "bc": rbc}
        if what == "biot":
            ra = pp.SecondOrderTensor(np.ones(r.num_cells))
            ra.values = alpha.values.copy()
            prm["scalar_vector_mappings"] = {"flow": ra}
            data = pp.initialize_data({}, "mech", prm)
            pp.Biot("mech").discretize(r, data)
        else:
            data = pp.initialize_data({}, "mech", prm)
            pp.Mpsa("mech").discretize(r, data)
        mats = {}
        for key, m in data[pp.DISCRETIZATION_MATRICES]["mech"].items():
            if isinstance(m, dict):
                for kk, v in m.items():
                    mats[f"{key}:{kk}"] = v
            else:
                mats[key] = m
    secs = time.perf_counter() - t0
    d = {"seconds_reference": np.float64(secs), "num_cells": np.int64(g.num_cells)}
    for key, m in mats.items():
        stride = max(1, -(-m.shape[0] // 20000)) * ROW_THINNING[name]
        for kk, v in cases.digest_of(m, stride=stride).items():
            d[f"D__{key}__{kk}"] = v
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print(f"{name}: {g.num_cells} cells, reference discretize {secs:.1f} s "
          f"({g.num_cells / secs:.0f} cells/s), {len(mats)} matrices", flush=True)


if __name__ == "__main__":
    for name in (sys.argv[1:] or list(cases.DIGEST_CASES)):
        run(name)
