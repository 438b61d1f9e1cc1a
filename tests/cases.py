"""Shared helpers: golden-case -> inputs for oracle / emulation / GPU product."""
from __future__ import annotations

import numpy as np

from golden_io import load_case, rel_err  # noqa: F401


def scalar_codes(bc, nf):
    internal = np.asarray(bc.is_internal, bool)
    codes = np.zeros(nf, np.uint8)
    codes[np.asarray(bc.is_neu, bool) | internal] = 2
    codes[np.asarray(bc.is_dir, bool) & ~internal] = 1
    codes[np.asarray(bc.is_rob, bool) & ~internal] = 3
    return codes


def vector_codes(bc, nd, nf):
    codes = np.zeros((nd, nf), np.uint8)
    codes[np.asarray(bc.is_neu, bool)[:nd]] = 2
    codes[np.asarray(bc.is_dir, bool)[:nd]] = 1
    codes[np.asarray(bc.is_rob, bool)[:nd]] = 3
    return codes


def flatten(out: dict) -> dict:
    """{'key': m, 'key2': {'a': m}} -> {'key': m, 'key2:a': m}"""
    flat = {}
    for k, v in out.items():
        if isinstance(v, dict):
            for ak, m in v.items():
                flat[f"{k}:{ak}"] = m
        else:
            flat[k] = v
    return flat


def max_rel_err(ref: dict, got: dict) -> tuple[float, str]:
    worst, wk = 0.0, ""
    for k, m in flatten(got).items():
        e = rel_err(ref[k], m)
        if e > worst:
            worst, wk = e, k
    return worst, wk


# ------------------------------------------------------------------------------------------
# benchmark-size parity cases (tests/golden/digest_*.npz, written by tools/make_digests.py from the
# unmodified reference): grid and parameters are REGENERATED from the seed by the functions below --
# the same code runs in the generator (on top of the reference) and in the GPU tests
# ------------------------------------------------------------------------------------------
DIGEST_CASES = {
    # name: (grid kind, dims, discretization)
    "digest_mpfa_cart32": ("cart", (32, 32, 32), "mpfa"),          # BASELINE config[0]
    "digest_mpsa_cart32": ("cart", (32, 32, 32), "mpsa"),
    "digest_mpfa_tet12": ("tet", (12, 12, 12), "mpfa"),
    "digest_mpsa_tet12": ("tet", (12, 12, 12), "mpsa"),
    "digest_mpfa_tet16": ("tet", (16, 16, 16), "mpfa"),
    "digest_mpsa_tet16": ("tet", (16, 16, 16), "mpsa"),
    "digest_biot_cart16": ("cart", (16, 16, 16), "biot"),
}


def digest_grid(kind, dims, seed=0):
    import porepy_b200 as pb
    if kind == "tet":
        return pb.structured_tet_grid(dims)
    return pb.cart_grid_3d(dims, perturb=0.2, seed=seed)


def digest_params(g, seed=0):
    """Anisotropic heterogeneous permeability, Dirichlet on x = 0 / x = 1 (else Neumann); heterogeneous
    isotropic stiffness, displacement fixed on z = 0 (else traction); a full Biot tensor."""
    import porepy_b200 as pb
    rng = np.random.default_rng(seed)
    nc = g.num_cells
    k = pb.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc),
                             0.3 * rng.random(nc), 0.3 * rng.random(nc), 0.3 * rng.random(nc))
    bf = g.get_all_boundary_faces()
    x = g.face_centers[0, bf]
    bc = pb.BoundaryCondition(g, bf[(x < 1e-10) | (x > 1 - 1e-10)], "dir")
    C = pb.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))
    vbc = pb.BoundaryConditionVectorial(g, bf[g.face_centers[2, bf] < 1e-10], "dir")
    alpha = pb.SecondOrderTensor(0.5 + 0.5 * rng.random(nc), 0.5 + 0.5 * rng.random(nc), 0.5 + 0.5 * rng.random(nc),
                                 0.1 * rng.random(nc), 0.1 * rng.random(nc), 0.1 * rng.random(nc))
    return k, bc, C, vbc, alpha


def digest_of(m, seed=0, nvec=2, nrows=200, max_strided=20000, nbil=8, stride=None):
    """What is stored per output matrix: M @ x_k and |M| @ 1 on every ``stride``-th row (default: <= ``max_strided``
    rows; the row stride is stored with the digest), ``nbil`` bilinear forms y^T M x over ALL entries, and ``nrows``
    sampled rows entrywise (a CSR sub-matrix)."""
    import scipy.sparse as sps
    m = sps.csr_matrix(m)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((m.shape[1], nvec))
    stride = int(stride) if stride else max(1, -(-m.shape[0] // max_strided))
    mx = (m @ x)
    y = rng.standard_normal((m.shape[0], nbil))
    xb = rng.standard_normal((m.shape[1], nbil))
    bil = np.einsum("ik,ik->k", y, m @ xb)
    bil_scale = np.einsum("ik,ik->k", np.abs(y), abs(m) @ np.abs(xb))
    rows = np.sort(rng.choice(m.shape[0], size=min(nrows, m.shape[0]), replace=False))
    sub = m[rows]
    sub.sum_duplicates()
    sub.eliminate_zeros()
    return {"mx": mx[::stride], "abs1": np.asarray(abs(m).sum(axis=1)).ravel()[::stride], "bil": bil,
            "bil_scale": bil_scale, "rows": rows.astype(np.int64), "sub_data": sub.data,
            "sub_indices": sub.indices.astype(np.int32), "sub_indptr": sub.indptr.astype(np.int64),
            "shape": np.array(m.shape, dtype=np.int64), "stride": np.int64(stride)}


def digest_errors(dig: dict, m, seed=0):
    """Relative errors of matrix ``m`` against a stored digest: (M @ x, |M| @ 1, bilinear forms, sampled rows
    entrywise); each normalised by the largest reference magnitude of its kind (the bilinear forms by
    |y|^T |M| |x|, the size of the sum without cancellation)."""
    import scipy.sparse as sps
    m = sps.csr_matrix(m)
    assert tuple(dig["shape"]) == m.shape, (tuple(dig["shape"]), m.shape)
    mine = digest_of(m, seed, nvec=dig["mx"].shape[1], nrows=dig["rows"].size, nbil=dig["bil"].size,
                     stride=int(dig["stride"]))
    assert np.array_equal(mine["rows"], dig["rows"]) and mine["mx"].shape == dig["mx"].shape
    e_mx = np.abs(mine["mx"] - dig["mx"]).max() / max(np.abs(dig["mx"]).max(), 1e-300)
    e_abs = np.abs(mine["abs1"] - dig["abs1"]).max() / max(np.abs(dig["abs1"]).max(), 1e-300)
    e_bil = (np.abs(mine["bil"] - dig["bil"]) / np.maximum(dig["bil_scale"], 1e-300)).max()
    n = dig["rows"].size
    ref = sps.csr_matrix((dig["sub_data"], dig["sub_indices"], dig["sub_indptr"]), shape=(n, m.shape[1]))
    got = sps.csr_matrix((mine["sub_data"], mine["sub_indices"], mine["sub_indptr"]), shape=(n, m.shape[1]))
    d = abs(ref - got)
    e_rows = (d.max() if d.nnz else 0.0) / max(abs(ref).max() if ref.nnz else 0.0, 1e-300)
    return float(e_mx), float(e_abs), float(e_bil), float(e_rows)
