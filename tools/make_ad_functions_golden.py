"""Generate tests/golden/ad_functions.npz: the inputs of tests/test_ad_functions.py (``cases()``) and the results of the
unmodified reference's ``pp.ad.functions`` / ``AdArray.__pow__`` on them (value, and Jacobian as CSR arrays).

    python tools/make_ad_functions_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from ref_loader import load_porepy  # noqa: E402
from test_ad_functions import GOLDEN, cases, reference_results  # noqa: E402


def put(d: dict, key: str, val, jac=None) -> None:
    d[key + "_val"] = np.asarray(val, dtype=np.float64)
    if jac is not None:
        m = sps.csr_matrix(jac)
        m.sort_indices()
        d[key + "_jac_data"], d[key + "_jac_indices"], d[key + "_jac_indptr"] = m.data, m.indices, m.indptr
        d[key + "_jac_shape"] = np.array(m.shape, dtype=np.int64)


if __name__ == "__main__":
    pp = load_porepy()
    out: dict = {}
    for k, (v, j) in cases().items():
        put(out, f"in_{k}", v, j)
    shift, res = reference_results(pp)
    for name, r in res.items():
        if isinstance(r, pp.ad.AdArray):
            put(out, f"out_{name}", r.val, r.jac)
        else:
            put(out, f"out_{name}", r)
    out["shift"] = np.float64(shift)
    out["names"] = np.array(sorted(res))
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")
