"""The device linear-algebra layer on every code path it dispatches to, against extended-precision references.

Kernels: ``csr_spmv_kernel`` / ``csr_spmv_dots_kernel`` (csrc/spmv.cu) at every lanes-per-row (TPR) variant, with and
without the grid-stride wrap and the autotuner; SpGEMM at every hash-table size, axpby, diagonal scaling and ``bmat``
(csrc/sparse_ops.cu); the block inverses and the three fused BiCGStab kernels (csrc/krylov.cu).

Every value is checked against a sum accumulated in ``np.longdouble`` (80-bit on x86; ``math.fsum`` elsewhere) with the
a-priori bound ``(k + 2) u sum |terms|`` of a k-term float64 sum, u = 2^-53.  Test data have magnitudes in [1, 2] with
random signs, so every single term is far above that bound: a dropped, doubled or misplaced entry fails.

Sizes that must cross a grid-stride or autotune threshold are derived from the SM count and the launch formulas:
SpMV grid <= 32 SMs CTAs of 256 threads (TPR lanes per row), autotuning above 2^20 non-zeros for a mean row length
<= 96; SpGEMM grid <= 4 SMs CTAs of 4 warps (2 at tsize 8192), one warp per row; axpby grid <= 16 SMs CTAs of 128.
The reference self-checks and the host stand-in refusals at the top run without a GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sps
import torch

from porepy_b200 import krylov as kr

U = 2.0 ** -53
LD = np.longdouble
_EXTENDED = np.finfo(np.longdouble).nmant >= 63


# ---------------------------------------------------------------------------------------------------------------------
# references and bounds
# ---------------------------------------------------------------------------------------------------------------------
def _signed(rng, n):
    """Magnitudes in [1, 2], random signs."""
    return rng.uniform(1.0, 2.0, n) * rng.choice([-1.0, 1.0], n)


def _segment_sums(terms, starts, n_terms):
    """Sums of terms[starts[i]:starts[i+1]] (the last segment runs to n_terms); starts strictly increasing."""
    if starts.size == 0:
        return np.zeros(0, LD)
    if _EXTENDED:
        return np.add.reduceat(np.asarray(terms, LD), starts)
    ends = np.r_[starts[1:], n_terms]
    return np.array([math.fsum(terms[a:b]) for a, b in zip(starts, ends)], LD)


def _exact_products(a, b):
    """Products of float64 pairs: in longdouble (64-bit mantissa) or, without it, float64 (the fsum path)."""
    return np.asarray(a, LD) * np.asarray(b, LD) if _EXTENDED else np.asarray(a) * np.asarray(b)


def _row_sums(terms, indptr):
    """Per-CSR-row sums of ``terms`` (empty rows: 0)."""
    n = indptr.size - 1
    out = np.zeros(n, LD)
    nz = np.flatnonzero(np.diff(indptr))
    out[nz] = _segment_sums(terms, indptr[nz], int(indptr[-1]))
    return out


def _spmv_ref(a, x):
    """(y, bound) of y = A x: longdouble row sums of a possibly non-canonical CSR (duplicates summed) and the bound
    (k + 2) u sum_j |a_ij x_j| of each row."""
    prods = _exact_products(a.data, x[a.indices])
    y = _row_sums(prods, a.indptr)
    absum = _row_sums(np.abs(prods), a.indptr).astype(np.float64)
    return y, (np.diff(a.indptr) + 2) * U * absum


def _assert_within(got, exact, bound, what):
    got = np.asarray(got)
    assert got.shape == exact.shape, (what, got.shape, exact.shape)
    err = np.abs(np.asarray(got, LD) - exact).astype(np.float64)
    bad = np.flatnonzero(~(err <= bound))
    assert bad.size == 0, (f"{what}: {bad.size} of {got.size} values outside the rounding bound; first at {bad[:4]}: "
                           f"err {err[bad[:4]]}, bound {bound[bad[:4]]}")


def _csr_from_lengths(lengths, ncols, rng):
    """Non-canonical CSR (unsorted columns, duplicates possible) with the given row lengths and signed values."""
    lengths = np.asarray(lengths, np.int64)
    indptr = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    nnz = int(indptr[-1])
    return sps.csr_matrix((_signed(rng, nnz), rng.integers(0, ncols, nnz), indptr), shape=(lengths.size, ncols))


def _spgemm_ref(a, b):
    """Structural product pattern (exact cancellations kept) and longdouble values of C = A B, with the bound
    (k + 2) u sum |a_ik b_kj| of each output; A, B canonical."""
    alen, blen = np.diff(a.indptr), np.diff(b.indptr)
    reps = blen[a.indices]
    total = int(reps.sum())
    arow = np.repeat(np.repeat(np.arange(a.shape[0]), alen), reps)
    aval = np.repeat(a.data, reps)
    bpos = np.repeat(b.indptr[a.indices], reps) + np.arange(total) - np.repeat(np.cumsum(reps) - reps, reps)
    col = b.indices[bpos]
    prod = _exact_products(aval, b.data[bpos])
    key = arow.astype(np.int64) * b.shape[1] + col
    order = np.argsort(key, kind="stable")
    key, prod = key[order], prod[order]
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]]) if total else np.zeros(0, np.int64)
    vals = _segment_sums(prod, starts, total)
    absum = _segment_sums(np.abs(prod), starts, total).astype(np.float64)
    cnt = np.diff(np.r_[starts, total])
    ukey = key[starts]
    rows, cols = ukey // b.shape[1], ukey % b.shape[1]
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=a.shape[0]))]
    return indptr, cols, vals, (cnt + 2) * U * absum


def _spgemm_launch(a, b):
    """(row bound, tsize, warps per block, refused) as pb_csr_spgemm derives them (csrc/sparse_ops.cu)."""
    bound = int(_row_bounds(a, b).max()) if a.shape[0] else 0
    want = min(2 * bound, 2 * b.shape[1])
    tsize = 64
    while tsize < want and tsize < 8192:
        tsize <<= 1
    return bound, tsize, 2 if tsize > 4096 else 4, tsize < min(bound, b.shape[1]) + 8


def _row_bounds(a, b):
    terms = np.diff(b.indptr)[a.indices]
    return _row_sums(terms.astype(np.float64), a.indptr).astype(np.int64)


class _Rec:
    """Textbook right-preconditioned BiCGStab (the recurrence of ``krylov.bicgstab``), float64 NumPy, x0 = 0; records
    every vector and scalar of each iteration."""

    def __init__(self, a, b, prec, iters):
        x = np.zeros_like(b)
        r, rhat = b.copy(), b.copy()
        p, v = np.zeros_like(b), np.zeros_like(b)
        rho = alpha = omega = 1.0
        self.bb = float(b @ b)
        self.steps = []
        for _ in range(iters):
            rho_new = float(rhat @ r)
            beta = (rho_new / rho) * (alpha / omega)
            p = r + beta * (p - omega * v)
            ph = prec(p)
            v = a @ ph
            rv = float(rhat @ v)
            alpha = rho_new / rv
            s = r - alpha * v
            sh = prec(s)
            t = a @ sh
            ts, tt = float(t @ s), float(t @ t)
            omega = ts / tt
            x = x + alpha * ph + omega * sh
            r = s - omega * t
            rho = rho_new
            self.steps.append(dict(x=x, r=r, p=p, s=s, v=v, t=t, rho=rho_new, alpha=alpha, omega=omega, rv=rv, ts=ts,
                                   tt=tt, rr=float(r @ r), rho_next=float(rhat @ r)))

    def relres(self, k):
        return math.sqrt(self.steps[k - 1]["rr"] / self.bb)


def _krylov_system(n=3360, seed=11):
    """Non-symmetric, kappa ~ 1e2: a 2-D convection-diffusion stencil on 28 x (n / 28) points, shifted, rows scaled by
    random factors in [1, 10] (so every preconditioner changes the iteration); ~40 iterations to 1e-5."""
    rng = np.random.default_rng(seed)
    nx = 28
    ny = n // nx
    lap = lambda m: sps.diags([-1.1, 2.0, -0.9], [-1, 0, 1], shape=(m, m))  # noqa: E731
    a = sps.kron(sps.identity(ny), lap(nx)) + sps.kron(lap(ny), sps.identity(nx)) + 0.15 * sps.identity(n)
    a = (sps.diags(rng.uniform(1.0, 10.0, n)) @ a).tocsr()
    a.sort_indices()
    return a, _signed(rng, n)


def _prec_blocks(a, bs):
    """Preconditioner data as the fused kernels read it: None, the inverse diagonal (bs 1), or inverted bs x bs
    diagonal blocks, row-major; and the same operator in NumPy."""
    n = a.shape[0]
    if bs is None:
        return None, (lambda y: y.copy())
    if bs == 1:
        minv = 1.0 / a.diagonal()
        return minv, (lambda y: minv * y)
    d = np.stack([a[i:i + bs, i:i + bs].toarray() for i in range(0, n, bs)])
    minv = np.linalg.inv(d)
    return minv.ravel(), (lambda y: np.einsum("bij,bj->bi", minv, y.reshape(-1, bs)).ravel())


PRECS = [None, 1, 2, 3, 4, 5, 7, 8]


# ---------------------------------------------------------------------------------------------------------------------
# 1. self-checks of the references (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_reference_sums_are_extended_or_exact():
    """The bound assumes a reference far more accurate than float64: 80-bit longdouble, or fsum of float64 products."""
    rng = np.random.default_rng(0)
    a = _csr_from_lengths(rng.integers(0, 40, 300), 200, rng)
    x = _signed(rng, 200)
    y, bound = _spmv_ref(a, x)
    ref = np.array([math.fsum(_exact_products(a.data[s:e], x[a.indices[s:e]]).astype(np.float64))
                    for s, e in zip(a.indptr[:-1], a.indptr[1:])])
    # fsum of float64-rounded products: at most one rounding per product
    absum = np.array([np.abs(a.data[s:e] * x[a.indices[s:e]]).sum() for s, e in zip(a.indptr[:-1], a.indptr[1:])])
    assert np.all(np.abs(y.astype(np.float64) - ref) <= 2 * U * absum + 1e-300)
    assert np.all(bound[np.diff(a.indptr) == 0] == 0.0)


def test_bound_holds_for_float64_and_catches_single_entry_errors():
    """scipy's float64 SpMV lies inside the bound; one dropped, doubled or misplaced entry does not, even in a row of
    1e5 terms."""
    rng = np.random.default_rng(1)
    lengths = rng.integers(0, 9, 2000)
    lengths[[5, 777, 1998]] = [100_000, 0, 3]
    a = _csr_from_lengths(lengths, 150_000, rng)
    x = _signed(rng, 150_000)
    y, bound = _spmv_ref(a, x)
    _assert_within(a @ x, y, bound, "scipy float64")
    for q in (a.indptr[5], a.indptr[5] + 54_321, a.indptr[6] - 1, a.indptr[1998]):
        row = int(np.searchsorted(a.indptr, q, side="right") - 1)
        for kind in ("drop", "double", "move"):
            m = a.copy()
            if kind == "drop":
                m.data[q] = 0.0
            elif kind == "double":
                m.data[q] *= 2.0
            else:
                m.indices[q] = (m.indices[q] + 1) % m.shape[1]
                if abs(x[m.indices[q]] - x[a.indices[q]]) < 1e-2:
                    continue
            err = abs(float(LD(np.asarray(m @ x)[row]) - y[row]))
            assert err > 100 * bound[row], (kind, row, err, bound[row])


def test_spgemm_reference_against_scipy_and_structure():
    rng = np.random.default_rng(2)
    a = _csr_from_lengths(rng.integers(0, 6, 120), 90, rng)
    b = _csr_from_lengths(rng.integers(0, 9, 90), 70, rng)
    a.sum_duplicates(), b.sum_duplicates()
    # an exact cancellation: two identical B rows with opposite weights -> explicit zeros kept in the pattern
    b = sps.vstack([b, b[3], b[3]]).tocsr()
    a = sps.hstack([a, sps.csr_matrix(([1.0, -1.0], ([7, 7], [0, 1])), shape=(120, 2))]).tocsr()
    a.sort_indices(), b.sort_indices()
    ip, ix, vals, bound = _spgemm_ref(a, b)
    pat = (sps.csr_matrix((np.ones(a.nnz), a.indices, a.indptr), shape=a.shape)
           @ sps.csr_matrix((np.ones(b.nnz), b.indices, b.indptr), shape=b.shape)).tocsr()
    pat.sort_indices()
    assert np.array_equal(ip, pat.indptr) and np.array_equal(ix, pat.indices)
    dense = (a @ b).toarray()
    c = sps.csr_matrix((vals.astype(np.float64), ix, ip), shape=dense.shape).toarray()
    assert np.abs(c - dense).max() <= 1e-12
    assert np.all(vals[ip[7]:ip[8]] == 0) and ip[8] > ip[7]


def test_reference_bicgstab_matches_eager_recurrence():
    """The NumPy reference and ``krylov.bicgstab``'s eager recurrence (scipy matvec stand-in) are the same algorithm:
    x (relative) and |r| / |b| agree within 1e-13 after every one of the first 12 iterations, for every
    preconditioner."""
    a, b = _krylov_system(n=840)
    loc = kr.build_local_system(a, np.zeros(a.shape[0], dtype=np.int64), 0, 1)
    op = kr.DistributedOperator(loc, "cpu", matvec=lambda xb: torch.as_tensor(a @ xb.numpy()))
    bt = torch.as_tensor(b)
    for bs in PRECS:
        minv, prec = _prec_blocks(a, bs)
        ref = _Rec(a, b, prec, 12)
        kw = {}
        if bs == 1:
            kw["diag_own"] = torch.as_tensor(a.diagonal())
        elif bs is not None:
            kw["block_inv"] = (torch.as_tensor(minv), bs)
        for k in range(1, 13):
            x, info = kr.bicgstab(op, bt, tol=1e-30, maxiter=k, **kw)
            want = ref.steps[k - 1]["x"]
            assert info["iterations"] == k and not info["breakdown"]
            assert np.linalg.norm(x.numpy() - want) <= 1e-13 * np.linalg.norm(want), (bs, k)
            assert abs(info["relres"] - ref.relres(k)) <= 1e-13, (bs, k)      # |r| in units of |b|
        assert ref.relres(12) > 1e-6, "the comparison window must stay far from convergence"


# ---------------------------------------------------------------------------------------------------------------------
# 6 (host half). the contract of tensors handed to the library, on the host stand-in
# ---------------------------------------------------------------------------------------------------------------------
def _emu():
    import emu_sparse
    return emu_sparse


def test_host_csr_refuses_what_the_device_cannot_read():
    rng = np.random.default_rng(3)
    a = _emu().HostCsr(_csr_from_lengths(rng.integers(1, 5, 30), 20, rng))
    good = torch.as_tensor(_signed(rng, 30))
    a.scaled(good)
    for bad in (good.float(), torch.as_tensor(_signed(rng, 60))[::2], torch.ones(1, dtype=torch.float64).expand(30)):
        with pytest.raises(TypeError):
            a.scaled(bad)
    with pytest.raises(ValueError):
        a.scaled(good[:29])
    with pytest.raises(TypeError):
        a @ torch.ones(20, dtype=torch.float32)
    with pytest.raises(ValueError):
        a @ torch.ones(19, dtype=torch.float64)


def test_ad_product_with_strided_view_on_host_stand_in(monkeypatch):
    """``DeviceAdArray * v[::2]`` (a user view) is converted before it reaches ``scaled``."""
    from porepy_b200 import ad
    _emu().install(monkeypatch)
    rng = np.random.default_rng(4)
    j = _csr_from_lengths(rng.integers(0, 5, 40), 25, rng)
    j.sum_duplicates()
    val = _signed(rng, 40)
    w = torch.as_tensor(_signed(rng, 80))[::2]
    prod = ad.DeviceAdArray(torch.as_tensor(val), _emu().HostCsr(j)) * w
    v, jac = prod.val.numpy(), prod.jac.to_scipy()
    wn = w.numpy()
    assert np.array_equal(v, val * wn)
    assert np.array_equal(jac.toarray(), (sps.diags(wn) @ j).toarray())


# ---------------------------------------------------------------------------------------------------------------------
# GPU fixtures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def lib():
    from porepy_b200 import _lib
    return _lib.load()


def _dev(a):
    from porepy_b200.sparse import DeviceCsr
    return DeviceCsr(a)


def _cuda(v):
    return torch.as_tensor(np.ascontiguousarray(v, np.float64), device="cuda")


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _check(rc):
    from porepy_b200 import _lib
    _lib.check(rc)


# ---------------------------------------------------------------------------------------------------------------------
# 2. SpMV and SpMV with dot products
# ---------------------------------------------------------------------------------------------------------------------
def _spmv_case(name, sm, rng):
    """(matrix, expected TPR or None for the autotuner, grid wraps) of each SpMV case; sizes from the SM count."""
    ri = rng.integers
    if name == "tpr2":            # mean <= 3, rows end mid-warp (16 groups) and mid-CTA (128 groups)
        return _csr_from_lengths(ri(0, 5, 4099), 3000, rng), 2, False
    if name == "tpr2-wrap-longrow":   # > 128 rows per CTA x 32 SMs CTAs, nnz <= 2^20, one row of 1e5 entries
        n = 128 * 32 * sm + 37
        lengths = ri(0, 3, n)
        lengths[n // 3] = 100_000
        return _csr_from_lengths(lengths, 200_000, rng), 2, True
    if name == "tpr4":
        return _csr_from_lengths(ri(3, 7, 3001), 5000, rng), 4, False
    if name == "tpr8":
        lengths = ri(0, 25, 2050)
        lengths[::97] = 0
        return _csr_from_lengths(lengths, 4000, rng), 8, False
    if name == "tpr8-wrap":       # > 32 rows per CTA x 32 SMs CTAs, mean in (6, 2^20 / rows]
        n = 32 * 32 * sm + 5
        return _csr_from_lengths(ri(6, 8, n), 50_000, rng), 8, True
    if name == "tpr16":
        return _csr_from_lengths(ri(25, 49, 513), 3000, rng), 16, False
    if name == "tpr32":
        return _csr_from_lengths(ri(49, 150, 257), 3000, rng), 32, False
    if name == "tpr32-wrap":      # > 8 rows per CTA x 32 SMs CTAs; mean > 96 skips the autotuner above 2^20 non-zeros
        return _csr_from_lengths(ri(97, 131, 8 * 32 * sm + 3), 40_000, rng), 32, True
    if name == "autotuned":       # nnz > 2^20, mean <= 96: timed candidates
        return _csr_from_lengths(ri(10, 31, 70_001), 80_000, rng), None, None
    if name == "single-row":
        return _csr_from_lengths([37], 100, rng), 16, False
    if name == "all-empty":
        return sps.csr_matrix((300, 40)), 2, False
    if name == "duplicates":      # uploaded with duplicate column entries: summed like scipy's sum_duplicates()
        a = _csr_from_lengths(ri(8, 20, 1001), 12, rng)
        assert not sps.csr_matrix(a, copy=True).has_canonical_format
        return a, 8, False
    raise KeyError(name)


SPMV_CASES = ["tpr2", "tpr2-wrap-longrow", "tpr4", "tpr8", "tpr8-wrap", "tpr16", "tpr32", "tpr32-wrap", "autotuned",
              "single-row", "all-empty", "duplicates"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SPMV_CASES)
def test_spmv_and_spmv_dots_every_lanes_per_row(name, sm, lib):
    rng = np.random.default_rng(100 + SPMV_CASES.index(name))
    a, tpr_want, wraps = _spmv_case(name, sm, rng)
    d = _dev(a)
    tpr = lib.pb_csr_lanes_per_row(d.h)
    if tpr_want is None:
        assert a.nnz > 2**20 and a.nnz / a.shape[0] <= 96 and tpr in (2, 4, 8, 16, 32)
    else:
        assert tpr == tpr_want, (name, tpr)
        assert (a.nnz <= 2**20) or (a.nnz / a.shape[0] > 96), "heuristic path"
    n, m = a.shape
    rows_per_pass = 32 * sm * 256 // tpr
    assert wraps is None or (n > rows_per_pass) == wraps, (name, n, rows_per_pass)
    print(f"SpMV case {name}: {n} rows, nnz {a.nnz}, TPR {tpr}, grid-stride wrap {n > rows_per_pass}")
    x = _signed(rng, m)
    ref_mat = a.copy()
    if name == "duplicates":
        ref_mat.sum_duplicates()
    y_ref, _ = _spmv_ref(ref_mat, x)
    _, bound = _spmv_ref(a, x)
    xt = _cuda(x)
    _assert_within((d @ xt).cpu().numpy(), y_ref, bound, f"{name} spmv")

    # SpMV with dots, straight on torch buffers; the slots are pre-seeded (the kernel accumulates into them)
    w1, w2 = _signed(rng, n), _signed(rng, n)
    w1t, w2t = _cuda(w1), _cuda(w2)
    s1, s2 = 0.625, -1.375
    y64 = y_ref.astype(np.float64)
    for combo in ("d1", "d1+yy", "d1+w2"):
        y = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        slots = _cuda([s1, s2])
        d1, d2 = C.c_void_p(slots.data_ptr()), C.c_void_p(slots.data_ptr() + 8)
        w2p = _p(w2t) if combo == "d1+w2" else None
        _check(lib.pb_csr_spmv_dots_dev(d.h, _p(xt), _p(y), _p(w1t), d1, w2p, d2 if combo != "d1" else None,
                                        torch.cuda.current_stream().cuda_stream))
        got = slots.cpu().numpy()
        _assert_within(y.cpu().numpy(), y_ref, bound, f"{name} {combo} y")
        e1 = LD(s1) + np.sum(np.asarray(w1, LD) * y_ref)
        b1 = float(np.abs(w1) @ bound) + (n + 3) * U * (abs(s1) + float(np.abs(w1 * y64).sum()))
        _assert_within(got[:1], np.array([e1]), np.array([b1]), f"{name} {combo} d1")
        if combo == "d1":
            assert got[1] == s2
            continue
        if combo == "d1+yy":
            e2 = LD(s2) + np.sum(y_ref * y_ref)
            b2 = float(((2 * np.abs(y64) + bound) * bound).sum()) + (n + 3) * U * (abs(s2) + float((y64 * y64).sum()))
        else:
            e2 = LD(s2) + np.sum(np.asarray(w2, LD) * y_ref)
            b2 = float(np.abs(w2) @ bound) + (n + 3) * U * (abs(s2) + float(np.abs(w2 * y64).sum()))
        _assert_within(got[1:], np.array([e2]), np.array([b2]), f"{name} {combo} d2")


@pytest.mark.gpu
def test_spmv_zero_rows_and_zero_columns(lib):
    """A 0 x n and an n x 0 matrix: the kernels launch on 0 rows / read no x; ``@`` returns the empty / zero vector."""
    stream = torch.cuda.current_stream().cuda_stream
    d = _dev(sps.csr_matrix((0, 7)))
    assert lib.pb_csr_lanes_per_row(d.h) == 2
    x, y, slots = _cuda(np.ones(7)), _cuda([5.0]), _cuda([0.5, 0.25])
    _check(lib.pb_csr_spmv_dev(d.h, _p(x), _p(y), stream))
    _check(lib.pb_csr_spmv_dots_dev(d.h, _p(x), _p(y), _p(y), _p(slots), None, C.c_void_p(slots.data_ptr() + 8),
                                    stream))
    assert y.cpu().item() == 5.0 and slots.cpu().tolist() == [0.5, 0.25]
    assert (d @ x).numel() == 0
    d0 = _dev(sps.csr_matrix((9, 0)))
    assert np.array_equal((d0 @ torch.zeros(0, dtype=torch.float64, device="cuda")).cpu().numpy(), np.zeros(9))


@pytest.mark.gpu
def test_spmv_on_a_non_default_stream(sm):
    rng = np.random.default_rng(5)
    a, _, _ = _spmv_case("tpr8-wrap", sm, rng)
    d = _dev(a)
    x = _signed(rng, a.shape[1])
    y_ref, bound = _spmv_ref(a, x)
    xt = _cuda(x)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        y1 = d @ xt
        y2 = torch.full((a.shape[0],), float("nan"), dtype=torch.float64, device="cuda")
        d.spmv_device(xt.data_ptr(), y2.data_ptr(), side.cuda_stream)
    torch.cuda.current_stream().wait_stream(side)
    _assert_within(y1.cpu().numpy(), y_ref, bound, "side stream @")
    _assert_within(y2.cpu().numpy(), y_ref, bound, "side stream spmv_device")


# ---------------------------------------------------------------------------------------------------------------------
# 3. SpGEMM, axpby, scaling, bmat
# ---------------------------------------------------------------------------------------------------------------------
def _boundary_lengths(lmax):
    """Distinct output counts around every 32-lane chunk and power-of-two (bitonic P) boundary up to lmax."""
    out = {1, lmax}
    p = 32
    while p <= lmax + 1:
        out.update(q for q in (p - 1, p, p + 1) if 1 <= q <= lmax)
        p <<= 1
    return sorted(out)


def _spgemm_case(tsize, sm, rng):
    """A, B with a largest row bound that lands on ``tsize``: rows with the boundary output counts, empty rows in A
    and B, a row whose columns all collide in the table, rows that merge overlapping B rows, an exact cancellation,
    and enough short rows (n = 1024 k +- 1) to wrap the grid and the 1024-row chunks of the scan."""
    lmax = 32 if tsize == 64 else (8184 if tsize == 8192 else tsize // 2)
    lens = _boundary_lengths(lmax)
    lc = min(lmax, 64)                      # colliding row: columns c0 + j tsize
    ncols = max(4 * lmax, lc * tsize + 8)
    brows = [rng.choice(ncols, L, replace=False) for L in lens]
    brows.append(3 + tsize * np.arange(lc))
    brows.append(np.zeros(0, np.int64))     # empty B row
    half = lmax // 2
    shared = rng.choice(ncols, 2 * half, replace=False)
    brows += [shared[:half], shared[half // 2:half // 2 + half]]   # two B rows that overlap by half
    nspecial = len(brows)
    brows += [rng.choice(ncols, int(k), replace=False) for k in rng.integers(1, 6, 200)]   # short rows
    bl = np.array([r.size for r in brows])
    b = sps.csr_matrix((_signed(rng, int(bl.sum())), np.concatenate(brows).astype(np.int64),
                        np.r_[0, np.cumsum(bl)]), shape=(len(brows), ncols))
    b.sort_indices()
    twin = len(brows)                       # a copy of a B row (same values): +1 / -1 cancels exactly
    b = sps.vstack([b, b[0]]).tocsr()
    arows, avals = [[]], [[]]               # row 0 empty
    for i in range(nspecial):
        arows.append([i]), avals.append(list(_signed(rng, 1)))
    arows.append([nspecial - 2, nspecial - 1]), avals.append(list(_signed(rng, 2)))      # merge overlapping rows
    arows.append([0, twin]), avals.append([1.5, -1.5])                                  # exact cancellation
    k = 16 * sm // 1024 + 1
    n = 1024 * k + (1 if (tsize.bit_length() & 1) else -1)
    while len(arows) < n:
        if len(arows) % 9 == 0:
            arows.append([]), avals.append([])
            continue
        c = np.unique(rng.integers(nspecial, twin, rng.integers(1, 4)))
        arows.append(list(c)), avals.append(list(_signed(rng, c.size)))
    al = np.array([len(r) for r in arows])
    a = sps.csr_matrix((np.concatenate([np.asarray(v, float) for v in avals]),
                        np.concatenate([np.asarray(r, np.int64) for r in arows]), np.r_[0, np.cumsum(al)]),
                       shape=(n, b.shape[0]))
    a.sort_indices()
    return a, b


def _check_spgemm(a, b, what):
    c = _dev(a).matmul(_dev(b)).to_scipy()
    ip, ix, vals, bound = _spgemm_ref(a, b)
    assert c.shape == (a.shape[0], b.shape[1])
    assert np.array_equal(c.indptr, ip), f"{what}: row lengths differ from the structural product"
    assert np.array_equal(c.indices, ix), f"{what}: columns differ from the structural product (sorted rows)"
    _assert_within(c.data, vals, bound, what)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("tsize", [64, 128, 256, 512, 1024, 2048, 4096, 8192], ids=lambda t: f"tsize{t}")
def test_spgemm_every_table_size(tsize, sm):
    rng = np.random.default_rng(tsize)
    a, b = _spgemm_case(tsize, sm, rng)
    bound, ts, wpb, refused = _spgemm_launch(a, b)
    assert ts == tsize and not refused, (bound, ts)
    assert a.shape[0] > 4 * sm * wpb, "the grid must wrap"
    print(f"SpGEMM tsize {ts}: {wpb} warps per block, row bound {bound}, {a.shape[0]} rows")
    _check_spgemm(a, b, f"tsize {tsize}")


@pytest.mark.gpu
def test_spgemm_capacity_edge_and_refusal():
    """A row bound of 8184 is accepted (tsize 8192, 2 warps per block); 8185 with B.ncols >= 8185 is refused on the
    host before the product kernels run; a huge bound over few columns of B is accepted at a small table."""
    rng = np.random.default_rng(8)
    ncols = 9000
    b = sps.csr_matrix((_signed(rng, 8185), rng.choice(ncols, 8185, replace=False), [0, 8184, 8185, 8185]),
                       shape=(3, ncols))
    b.sort_indices()
    a = sps.csr_matrix((_signed(rng, 3), [0, 2, 0], [0, 1, 1, 2, 3]), shape=(4, 3))
    assert _spgemm_launch(a, b)[1:] == (8192, 2, False)
    _check_spgemm(a, b, "bound 8184")
    a2 = sps.csr_matrix((_signed(rng, 2), [0, 1], [0, 2]), shape=(1, 3))
    assert _spgemm_launch(a2, b)[0] == 8185 and _spgemm_launch(a2, b)[3]
    with pytest.raises(NotImplementedError, match="8184"):
        _dev(a2).matmul(_dev(b))
    # B.ncols small against the bound: outputs that sum hundreds of products (tsize 64)
    a3 = _csr_from_lengths(rng.integers(250, 400, 300), 400, rng)
    a3.sum_duplicates()
    b3 = _csr_from_lengths(np.r_[np.zeros(5, int), rng.integers(3, 6, 395)], 5, rng)
    b3.sum_duplicates()
    bound, ts, _, refused = _spgemm_launch(a3, b3)
    assert bound > 500 and ts == 64 and not refused
    _check_spgemm(a3, b3, "few columns")


@pytest.mark.gpu
def test_axpby_patterns_scalars_and_grid_wrap(sm):
    """Disjoint, identical, one-sided and empty row patterns over more rows than the 16 SMs x 128 threads grid;
    alpha / beta zero and negative; A - A keeps its pattern with exact zeros."""
    rng = np.random.default_rng(9)
    n, m = 16 * sm * 128 + 3, 64
    kind = np.arange(n) % 4                       # 0 disjoint, 1 identical, 2 only A, 3 both empty
    la = np.where(kind == 3, 0, rng.integers(1, 5, n))
    a = _csr_from_lengths(la, 32, rng)            # columns 0..31
    a.sum_duplicates()
    lb = np.where(kind >= 2, 0, rng.integers(1, 5, n))
    b = _csr_from_lengths(lb, 32, rng)
    b.indices += 32                               # columns 32..63: disjoint from A
    b = sps.csr_matrix((b.data, b.indices, b.indptr), shape=(n, m))
    b.sum_duplicates()
    a = sps.csr_matrix((a.data, a.indices, a.indptr), shape=(n, m))
    same = np.flatnonzero(kind == 1)              # identical pattern in the rows of kind 1
    sel = sps.csr_matrix((np.ones(same.size), (same, same)), shape=(n, n))
    b = (b - sel @ b + sel @ sps.csr_matrix((_signed(rng, a.nnz), a.indices, a.indptr), shape=(n, m))).tocsr()
    b.eliminate_zeros()
    b.sort_indices()
    da, db = _dev(a), _dev(b)
    union = (abs(sps.csr_matrix((np.ones(a.nnz), a.indices, a.indptr), shape=(n, m)))
             + abs(sps.csr_matrix((np.ones(b.nnz), b.indices, b.indptr), shape=(n, m)))).tocsr()
    union.sort_indices()
    keys = np.repeat(np.arange(n), np.diff(union.indptr)) * m + union.indices

    def on_union(x):
        out = np.zeros(keys.size)
        out[np.searchsorted(keys, np.repeat(np.arange(n), np.diff(x.indptr)) * m + x.indices)] = x.data
        return out
    ua, ub = on_union(a), on_union(b)
    for alpha, beta in ((1.0, -1.0), (0.0, 2.5), (-1.5, 0.0), (-0.75, -2.0), (0.0, 0.0)):
        c = da.axpby(alpha, db, beta).to_scipy()
        assert np.array_equal(c.indptr, union.indptr) and np.array_equal(c.indices, union.indices), (alpha, beta)
        exact = np.asarray(alpha * ua, LD) + np.asarray(beta * ub, LD)
        _assert_within(c.data, exact, 4 * U * (np.abs(alpha * ua) + np.abs(beta * ub)), f"axpby {alpha} {beta}")
    z = (da - da).to_scipy()
    assert np.array_equal(z.indptr, a.indptr) and np.array_equal(z.indices, a.indices) and not z.data.any()


@pytest.mark.gpu
def test_scaled_by_rows_and_columns_also_after_truncate_rows():
    rng = np.random.default_rng(10)
    a = _csr_from_lengths(rng.integers(0, 40, 5001), 3001, rng)
    a.sum_duplicates()
    for keep in (None, 2999):
        d = _dev(a)
        ref = a
        if keep is not None:
            d.truncate_rows(keep)
            ref = a[:keep]
        for by_cols in (False, True):
            s = _signed(rng, ref.shape[1] if by_cols else ref.shape[0])
            c = d.scaled(_cuda(s), by_cols=by_cols).to_scipy()
            assert c.shape == ref.shape
            assert np.array_equal(c.indptr, ref.indptr) and np.array_equal(c.indices, ref.indices)
            f = s[ref.indices] if by_cols else np.repeat(s, np.diff(ref.indptr))
            _assert_within(c.data, _exact_products(ref.data, f), 3 * U * np.abs(ref.data * f), f"scaled {by_cols}")


@pytest.mark.gpu
def test_bmat_many_block_rows_empty_blocks_and_none():
    """45 block rows (the kernel finds a row's block row by a linear search), 0-row and 0-column blocks, None blocks;
    values are copied, so the result equals the host assembly bit for bit."""
    from porepy_b200.sparse import DeviceCsr
    rng = np.random.default_rng(12)
    rs = rng.integers(0, 60, 45)
    rs[[3, 17, 44]] = 0
    cs = np.array([37, 0, 51])
    blocks, ref = [], []
    for i, r in enumerate(rs):
        row, rrow = [], []
        for j, c in enumerate(cs):
            if (i + j) % 3 == 1 and j != (i % 3):
                row.append(None), rrow.append(None)
                continue
            m = _csr_from_lengths(rng.integers(0, 6, r), c, rng) if c else sps.csr_matrix((r, 0))
            m.sum_duplicates()
            row.append(m), rrow.append(m)
        blocks.append([None if m is None else _dev(m) for m in row])
        ref.append(rrow)
    got = DeviceCsr.bmat(blocks).to_scipy()
    ro, co = np.r_[0, np.cumsum(rs)], np.r_[0, np.cumsum(cs)]
    r_, c_, v_ = [], [], []
    for i in range(len(rs)):
        for j in range(len(cs)):
            m = ref[i][j]
            if m is not None and m.nnz:
                cm = m.tocoo()
                r_.append(cm.row + ro[i]), c_.append(cm.col + co[j]), v_.append(cm.data)
    want = sps.csr_matrix((np.concatenate(v_), (np.concatenate(r_), np.concatenate(c_))), shape=(ro[-1], co[-1]))
    want.sort_indices()
    assert got.shape == want.shape
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data, want.data)


# ---------------------------------------------------------------------------------------------------------------------
# 4. block inverses
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bs", [1, 2, 3, 4, 5, 7, 8])
def test_block_inverse_partial_rectangular_duplicates(bs):
    """nblocks < nrows / bs on a rectangular matrix; entries outside the diagonal blocks (also beyond the square part)
    are ignored, duplicate in-block entries summed.  Residual |E D - I|_inf <= c bs u kappa_inf(D); a singular block
    falls back to the inverse of its diagonal (1 where that is 0)."""
    rng = np.random.default_rng(40 + bs)
    nb, nblocks = 150, 143
    n, ncols = nb * bs + 2, nb * bs + 9
    dblk = rng.standard_normal((nb, bs, bs)) + 2 * bs * np.eye(bs) * rng.choice([-1.0, 1.0], (nb, 1, 1))
    if bs > 1:
        dblk[5, 0, 0] = 0.0                       # pivoting needed
    sing = 9                                      # singular: [0] (bs 1); rows 0 and 1 parallel, diagonal (3, 0, ...)
    dblk[sing] = 0.0
    if bs > 1:
        dblk[sing, 0, 0], dblk[sing, 1, 0] = 3.0, 6.0
    # each in-block entry split in two (duplicates), plus off-block noise
    rows, cols, vals = [], [], []
    for k in range(nb):
        i, j = np.meshgrid(np.arange(bs), np.arange(bs), indexing="ij")
        part = rng.uniform(0.2, 0.8, (bs, bs)) * dblk[k] * (k != sing)
        for v in (part, dblk[k] - part):
            rows.append((k * bs + i).ravel()), cols.append((k * bs + j).ravel()), vals.append(v.ravel())
    dup_d = np.stack([sum(v.reshape(bs, bs) for v in vals[2 * k:2 * k + 2]) for k in range(nb)])
    noise = sps.random(n, ncols, density=5.0 / ncols, random_state=bs, format="coo")
    keep = (noise.row // bs != noise.col // bs) | (noise.row >= nb * bs)
    rows.append(noise.row[keep]), cols.append(noise.col[keep]), vals.append(_signed(rng, int(keep.sum())))
    r, c, v = (np.concatenate(z) for z in (rows, cols, vals))
    order = np.lexsort((c, r))
    r, c, v = r[order], c[order], v[order]
    a = sps.csr_matrix((v, c, np.r_[0, np.cumsum(np.bincount(r, minlength=n))]), shape=(n, ncols))
    got = _dev(a).block_diagonal_inverse(bs, nblocks).cpu().numpy()
    assert got.size == nblocks * bs * bs
    got = got.reshape(nblocks, bs, bs)
    eye = np.eye(bs, dtype=LD)
    for k in range(nblocks):
        dk = dup_d[k]
        if k == sing:
            dg = np.diagonal(dk)
            assert np.array_equal(got[k], np.diag(np.where(dg != 0, 1.0 / np.where(dg != 0, dg, 1.0), 1.0))), k
            continue
        res = np.abs(np.asarray(got[k], LD) @ np.asarray(dk, LD) - eye).sum(axis=1).max()
        kappa = np.abs(dk).sum(axis=1).max() * np.abs(np.linalg.inv(dk)).sum(axis=1).max()
        assert float(res) <= 8 * bs * U * kappa, (bs, k, float(res), kappa)


def _gj_pivots(d):
    """Row swaps and pivot magnitudes of Gauss-Jordan with partial pivoting in float64, as the block-inverse kernels
    choose them (first row of the largest magnitude)."""
    d = np.array(d, dtype=np.float64)
    n = d.shape[0]
    perm, best = [], []
    for k in range(n):
        piv = k + int(np.argmax(np.abs(d[k:, k])))
        perm.append(piv), best.append(abs(d[piv, k]))
        if not best[-1] > 0.0:
            break
        d[[k, piv]] = d[[piv, k]]
        d[k] /= d[k, k]
        for i in range(n):
            if i != k:
                d[i] -= d[i, k] * d[k]
    return perm, best


def _blocks8():
    """Two 8 x 8 blocks for the in-place kernel's deferred column permutation:
    cyclic -- a scaled cyclic shift plus a small perturbation: pivoting swaps at every step k < 7 and the swaps
    compose to one 8-cycle;
    last_singular -- small integers with power-of-two pivots, the last row the sum of rows 1 and 4: elimination is
    exact and the pivot at k = 7 is exactly 0 after seven regular steps."""
    rng = np.random.default_rng(47)
    cyclic = np.zeros((8, 8))
    cyclic[np.arange(8), (np.arange(8) + 1) % 8] = rng.uniform(2.0, 4.0, 8) * rng.choice([-1.0, 1.0], 8)
    cyclic += 1e-2 * rng.uniform(-1.0, 1.0, (8, 8))
    last = np.triu(rng.integers(-2, 3, (8, 8)).astype(np.float64), 1)
    last[np.arange(7), np.arange(7)] = 8.0 * rng.choice([-1.0, 1.0], 7)
    last[7] = last[1] + last[4]
    return cyclic, last


def test_block8_cases_pivot_as_intended():
    cyclic, last = _blocks8()
    perm, best = _gj_pivots(cyclic)
    assert all(perm[k] != k for k in range(7)) and len(best) == 8 and min(best) > 0.5
    order = np.arange(8)
    for k, p in enumerate(perm):
        order[[k, p]] = order[[p, k]]
    seen, j = {0}, int(order[0])
    while j != 0:
        seen.add(j)
        j = int(order[j])
    assert len(seen) == 8, "the row swaps form a single cycle"
    perm, best = _gj_pivots(last)
    assert len(best) == 8 and min(best[:7]) > 0 and best[7] == 0.0


@pytest.mark.gpu
def test_block_inverse_8_cyclic_pivoting_and_last_pivot_singular():
    """The in-place 8 x 8 Gauss-Jordan on a block that swaps rows at every step (its inverse needs the whole deferred
    column permutation) and on one that is singular only at the last pivot (the diagonal fallback, with the ``ok``
    flag carried through the unrolled loop)."""
    cyclic, last = _blocks8()
    rng = np.random.default_rng(48)
    regular = rng.standard_normal((8, 8)) + 16 * np.eye(8)
    blocks = [cyclic, last, regular, cyclic.T]
    a = sps.csr_matrix(sps.block_diag([sps.csr_matrix(b) for b in blocks]))
    got = _dev(a).block_diagonal_inverse(8).cpu().numpy().reshape(len(blocks), 8, 8)
    eye = np.eye(8, dtype=LD)
    for k, dk in enumerate(blocks):
        if k == 1:
            dg = np.diagonal(dk)
            assert np.array_equal(got[k], np.diag(np.where(dg != 0, 1.0 / np.where(dg != 0, dg, 1.0), 1.0)))
            continue
        res = np.abs(np.asarray(got[k], LD) @ np.asarray(dk, LD) - eye).sum(axis=1).max()
        kappa = np.abs(dk).sum(axis=1).max() * np.abs(np.linalg.inv(dk)).sum(axis=1).max()
        assert float(res) <= 8 * 8 * U * kappa, (k, float(res), kappa)


# ---------------------------------------------------------------------------------------------------------------------
# 5. the fused recurrence, step by step and through krylov.bicgstab
# ---------------------------------------------------------------------------------------------------------------------
def _rel_close(got, want, scale, tol, what):
    assert abs(got - want) <= tol * scale, (what, got, want, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("bs", PRECS, ids=lambda b: "none" if b is None else f"bs{b}")
def test_fused_kernels_step_by_step(bs, lib):
    """pb_kry_init / seed / p / s / xr and pb_csr_spmv_dots_dev driven as ``_bicgstab_fused.iterations`` does (one
    rank): after each of 12 iterations x, r, p, s and the 14-double scalar buffer match the NumPy recurrence."""
    a, b = _krylov_system()
    n = a.shape[0]
    minv_np, prec = _prec_blocks(a, bs)
    ref = _Rec(a, b, prec, 12)
    d = _dev(a)
    z = lambda: torch.zeros(n, dtype=torch.float64, device="cuda")  # noqa: E731
    x, r, rhat, p, v, s, t, ph, sh = (z() for _ in range(9))
    bt = _cuda(b)
    minv = None if minv_np is None else _cuda(minv_np)
    scal = torch.zeros(14, dtype=torch.float64, device="cuda")
    S = lambda i: C.c_void_p(scal.data_ptr() + 8 * i)  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    tol = 1e-30
    _check(lib.pb_kry_init(n, _p(bt), _p(x), _p(r), _p(rhat), _p(p), _p(v), _p(scal), tol, st))
    _check(lib.pb_kry_seed(_p(scal), st))
    kb = 1 if bs is None else bs
    nb2 = float(b @ b)
    for it in range(12):
        cur = it & 1
        g = 5 * cur
        _check(lib.pb_kry_p(n, _p(r), _p(p), _p(v), _p(minv), _p(ph), _p(scal), cur, kb, st))
        _check(lib.pb_csr_spmv_dots_dev(d.h, _p(ph), _p(v), _p(rhat), S(g), None, None, st))
        _check(lib.pb_kry_s(n, _p(r), _p(v), _p(minv), _p(s), _p(sh), _p(scal), cur, kb, st))
        _check(lib.pb_csr_spmv_dots_dev(d.h, _p(sh), _p(t), _p(s), S(g + 1), None, S(g + 2), st))
        _check(lib.pb_kry_xr(n, _p(x), _p(ph), _p(sh), _p(s), _p(t), _p(r), _p(rhat), _p(scal), cur, 1, st))
        w = ref.steps[it]
        for name, vec in (("x", x), ("r", r), ("p", p), ("s", s)):
            got = vec.cpu().numpy()
            assert np.linalg.norm(got - w[name]) <= 1e-10 * np.linalg.norm(w[name]), (bs, it, name)
        h = scal.cpu().numpy()
        gc, gn = h[g:g + 5], h[5 * (cur ^ 1):5 * (cur ^ 1) + 5]
        nr = lambda u: float(np.linalg.norm(u))  # noqa: E731
        _rel_close(gc[0], w["rv"], nr(b) * nr(w["v"]), 1e-10, (bs, it, "RHATV"))
        _rel_close(gc[1], w["ts"], nr(w["t"]) * nr(w["s"]), 1e-10, (bs, it, "TS"))
        _rel_close(gc[2], w["tt"], w["tt"], 1e-10, (bs, it, "TT"))
        _rel_close(gc[4], w["rho"], nb2 if it == 0 else nr(b) * nr(ref.steps[it - 1]["r"]), 1e-10, (bs, it, "RHO"))
        _rel_close(gc[1] / gc[2], w["omega"], abs(w["omega"]), 1e-10, (bs, it, "omega"))
        _rel_close(gc[4] / gc[0], w["alpha"], abs(w["alpha"]), 1e-10, (bs, it, "alpha"))
        assert gn[0] == gn[1] == gn[2] == 0.0, "the other parity group is cleared by the s-update"
        _rel_close(gn[3], w["rr"], w["rr"], 1e-10, (bs, it, "RR next"))
        _rel_close(gn[4], w["rho_next"], nr(b) * nr(w["r"]), 1e-10, (bs, it, "RHO next"))
        assert h[10] == pytest.approx(nb2, rel=1e-14) and h[11] == 0.0 and h[12] == it + 1 and h[13] == tol * tol


def _fused_solve(a, b, bs, tol, maxiter):
    minv, _ = _prec_blocks(a, bs)
    loc = kr.LocalSystem(0, 1, np.arange(a.shape[0]), np.zeros(0, np.int64), _dev(a), [0], [np.zeros(0, np.int64)])
    op = kr.DistributedOperator(loc, torch.device("cuda", torch.cuda.current_device()))
    return kr.bicgstab(op, _cuda(b), tol=tol, maxiter=maxiter, block_inv=(_cuda(minv), bs))


@pytest.mark.gpu
@pytest.mark.parametrize("graph", ["0", "1"], ids=["plain", "cuda-graph"])
def test_bicgstab_done_freeze_and_tail_block(graph, monkeypatch):
    """Convergence at an iteration j that is not a multiple of check_every: info["iterations"] == j and, with
    maxiter = j + 7, x is the reference x_j (the sticky DONE flag froze the vectors).  A maxiter that leaves a tail
    block after the full blocks gives the reference x_maxiter."""
    monkeypatch.setenv("POREB200_KRYLOV_GRAPH", graph)
    a, b = _krylov_system()
    bs = 3
    _, prec = _prec_blocks(a, bs)
    ref = _Rec(a, b, prec, 30)
    rel = [ref.relres(k) for k in range(1, 31)]
    # first j (not a multiple of 8) whose residual is clearly below every earlier one
    j = next(k for k in range(9, 31) if k % 8 and 1.5 * rel[k - 1] < min(rel[:k - 1]))
    tol = math.sqrt(min(rel[:j - 1]) * rel[j - 1])
    x, info = _fused_solve(a, b, bs, tol, j + 7)
    assert info["converged"] and info["iterations"] == j, (j, info)
    assert info["cuda_graph"] == (graph == "1")
    want = ref.steps[j - 1]["x"]
    assert np.linalg.norm(x.cpu().numpy() - want) <= 1e-10 * np.linalg.norm(want)
    for maxiter in (13, 19):                      # 8 + 5 and 16 + 3 (check_every 8)
        x, info = _fused_solve(a, b, bs, 1e-30, maxiter)
        assert not info["converged"] and info["iterations"] == maxiter, info
        want = ref.steps[maxiter - 1]["x"]
        assert np.linalg.norm(x.cpu().numpy() - want) <= 1e-10 * np.linalg.norm(want), maxiter


# ---------------------------------------------------------------------------------------------------------------------
# 6. tensors handed to the library
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_strided_view_in_device_ad_product():
    from porepy_b200 import ad
    rng = np.random.default_rng(20)
    j = _csr_from_lengths(rng.integers(0, 6, 500), 300, rng)
    j.sum_duplicates()
    val = _signed(rng, 500)
    w = _cuda(_signed(rng, 1000))[::2]
    prod = ad.DeviceAdArray(_cuda(val), _dev(j)) * w
    v, jac = prod.host()
    wn = w.cpu().numpy()
    assert np.array_equal(v, val * wn)
    ref = (sps.diags(wn) @ j).tocsr()
    ref.sort_indices()
    assert np.array_equal(jac.indptr, ref.indptr) and np.array_equal(jac.indices, ref.indices)
    assert np.array_equal(jac.data, ref.data)


@pytest.mark.gpu
def test_strided_view_in_device_spmv():
    rng = np.random.default_rng(21)
    a = _csr_from_lengths(rng.integers(0, 30, 700), 400, rng)
    full = _signed(rng, 800)
    y_ref, bound = _spmv_ref(a, full[::2])
    _assert_within((_dev(a) @ _cuda(full)[::2]).cpu().numpy(), y_ref, bound, "strided x")
    xe = _signed(rng, 1)
    y_ref, bound = _spmv_ref(a, np.repeat(xe, 400))
    _assert_within((_dev(a) @ _cuda(xe).expand(400)).cpu().numpy(), y_ref, bound, "expanded x")


@pytest.mark.gpu
def test_tensors_the_device_cannot_read_are_refused():
    rng = np.random.default_rng(22)
    a = _csr_from_lengths(rng.integers(1, 5, 30), 20, rng)
    d = _dev(a)
    good = _cuda(_signed(rng, 30))
    for bad in (good.float(), good.cpu(), _cuda(_signed(rng, 60))[::2], _cuda([1.5]).expand(30)):
        with pytest.raises(TypeError):
            d.scaled(bad)
    with pytest.raises(ValueError):
        d.scaled(good[:29])
    for bad in (torch.ones(20, dtype=torch.float32, device="cuda"), torch.ones(20, dtype=torch.float64)):
        with pytest.raises(TypeError):
            d @ bad
    with pytest.raises(ValueError):
        d @ torch.ones(19, dtype=torch.float64, device="cuda")
    # the fused BiCGStab: preconditioner data of the wrong dtype or device
    ak, bk = _krylov_system(n=84)
    minv, _ = _prec_blocks(ak, 3)
    loc = kr.LocalSystem(0, 1, np.arange(84), np.zeros(0, np.int64), _dev(ak), [0], [np.zeros(0, np.int64)])
    op = kr.DistributedOperator(loc, torch.device("cuda", torch.cuda.current_device()))
    bt = _cuda(bk)
    for bad in (_cuda(minv).float(), torch.as_tensor(minv)):
        with pytest.raises(TypeError):
            kr.bicgstab(op, bt, block_inv=(bad, 3))
    for bad in (_cuda(ak.diagonal()).float(), torch.as_tensor(ak.diagonal())):
        with pytest.raises(TypeError):
            kr.bicgstab(op, bt, diag_own=bad)
    x, info = kr.bicgstab(op, bt, tol=1e-12, block_inv=(_cuda(minv), 3))
    assert info["converged"]
