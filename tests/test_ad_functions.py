"""``porepy_b200.ad_functions`` against the reference's ``pp.ad.functions`` / ``AdArray.__pow__`` on random ``AdArray``s
(value and Jacobian), incl. the tie rule of ``maximum`` and the zero-vector rule of ``l2_norm``.  The reference's inputs
and results are stored in tests/golden/ad_functions.npz (tools/make_ad_functions_golden.py).
CPU: the scipy stand-in for the device sparse algebra; GPU leg at the end of the suite."""
import os

import numpy as np
import scipy.sparse as sps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ad_functions.npz")
INPUTS = ("a", "b", "c", "pos")


def cases(n=24, m=40, seed=0):
    rng = np.random.default_rng(seed)

    def jac():
        return sps.random(n, m, 0.2, format="csr", random_state=int(rng.integers(1 << 30)), data_rvs=rng.standard_normal)
    a, b = rng.standard_normal(n), rng.standard_normal(n)
    b[:4] = a[:4]                                      # ties: maximum takes the first argument
    c = rng.standard_normal(n)
    c[3:6] = 0.0                                       # one vanishing 3-vector for l2_norm
    pos = 0.5 + rng.random(n)
    return dict(a=(a, jac()), b=(b, jac()), c=(c, jac()), pos=(pos, jac()))


def reference_results(pp):
    """The reference's results on ``cases()``: what tools/make_ad_functions_golden.py stores."""
    f, A = pp.ad.functions, pp.ad.AdArray
    r = {k: A(v.copy(), j.copy()) for k, (v, j) in cases().items()}
    shift = float(f.l2_norm(3, r["c"]).val.mean())
    b = cases()["b"][0]
    return shift, {
        "exp": f.exp(r["a"]), "log": f.log(r["pos"]), "abs": f.abs(r["a"]), "sin": f.sin(r["a"]),
        "cos": f.cos(r["a"]), "tanh": f.tanh(r["a"]), "pow": r["pos"] ** 2.5, "sqrt": r["pos"] ** 0.5,
        "heaviside": f.heaviside(0.5, r["c"]), "heaviside_smooth": f.heaviside_smooth(r["a"], 1e-2),
        "characteristic": f.characteristic_function(1e-10, r["c"]),
        "maximum ad/ad": f.maximum(r["a"], r["b"]), "maximum ad/array": f.maximum(r["a"], b),
        "maximum array/ad": f.maximum(b, r["a"]), "maximum ad/scalar": f.maximum(r["a"], 0.1),
        "l2_norm": f.l2_norm(3, r["c"]), "l2_norm dim 1": f.l2_norm(1, r["a"]),
        # compositions of the kind the friction law uses: b (f_max - ||t||) clipped at zero
        "composition": f.maximum(r["pos"] - shift, 0.0) * f.exp(r["a"]),
    }


def _csr(g, key):
    return sps.csr_matrix((g[key + "_data"], g[key + "_indices"], g[key + "_indptr"]), shape=tuple(g[key + "_shape"]))


def run_checks(make, fn, to_host):
    """``make(val, jac)`` builds the device array; ``fn`` is porepy_b200.ad_functions."""
    g = np.load(GOLDEN)
    cs = {k: (g[f"in_{k}_val"], _csr(g, f"in_{k}_jac")) for k in INPUTS}
    dev = {k: make(v.copy(), j.copy()) for k, (v, j) in cs.items()}
    b = cs["b"][0]
    got = {
        "exp": fn.exp(dev["a"]), "log": fn.log(dev["pos"]), "abs": fn.abs(dev["a"]), "sin": fn.sin(dev["a"]),
        "cos": fn.cos(dev["a"]), "tanh": fn.tanh(dev["a"]), "pow": fn.power(dev["pos"], 2.5), "sqrt": fn.sqrt(dev["pos"]),
        "heaviside": fn.heaviside(0.5, dev["c"]), "heaviside_smooth": fn.heaviside_smooth(dev["a"], 1e-2),
        "characteristic": fn.characteristic_function(1e-10, dev["c"]),
        "maximum ad/ad": fn.maximum(dev["a"], dev["b"]), "maximum ad/array": fn.maximum(dev["a"], b),
        "maximum array/ad": fn.maximum(b, dev["a"]), "maximum ad/scalar": fn.maximum(dev["a"], 0.1),
        "l2_norm": fn.l2_norm(3, dev["c"]), "l2_norm dim 1": fn.l2_norm(1, dev["a"]),
        "composition": fn.maximum(dev["pos"] - float(g["shift"]), 0.0) * fn.exp(dev["a"]),
    }
    assert sorted(got) == sorted(str(n) for n in g["names"])
    for what, r in got.items():
        rv = g[f"out_{what}_val"]
        gv, gj = to_host(r)
        assert np.allclose(gv, rv, rtol=1e-13, atol=1e-13), what
        if f"out_{what}_jac_data" in g:
            rj = _csr(g, f"out_{what}_jac")
            d = abs(rj - sps.csr_matrix(gj))
            assert (d.max() if d.nnz else 0.0) <= 1e-12 * max(abs(rj).max(), 1.0), what


def test_functions_match_the_reference_host_build(monkeypatch):
    import torch
    import emu_sparse
    from porepy_b200 import ad, ad_functions
    emu_sparse.install(monkeypatch)

    def make(v, j):
        return ad.DeviceAdArray(torch.as_tensor(v.copy()), emu_sparse.HostCsr(j))

    def to_host(g):
        if isinstance(g, ad.DeviceAdArray):
            return g.val.numpy(), g.jac.to_scipy()
        return g.numpy(), None
    run_checks(make, ad_functions, to_host)
