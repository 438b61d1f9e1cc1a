"""The dense local solvers of the node routines (TileGJ / SmemGJ, porepy_b200/csrc/node_kernels.cuh), run
on their own through tests/gpu_harness for every solver configuration Cfg0..Cfg6 of porepy_b200/csrc/plan.hpp, and
compared with an extended-precision reference.

Shapes are those the dispatcher can send a configuration: every (n, nrhs) with n <= max_n and
W = (n + nrhs) | 1 <= max_w, read from the compiled types.  Matrix families (seeded):
  F1  random, well conditioned, rows at unit 1-norm (as the node routines scale them): the fast path of TileGJ
  F2  diagonally dominant, rows shifted cyclically by >= 5 so that every natural 4x4 pivot block holds only small
      off-diagonal entries: every panel of TileGJ takes the partial-pivoting path and later panels find their rows
      used
  F3  block lower triangular with diagonal blocks whose max |A11^-1| is just below / just above the growth threshold
  F4  F2 at scale 1e-6 and 1e-8, a more strongly dominant F2 at 1e5, and matrices whose trailing Schur complement
      is delta * C (kappa ~ 1/delta)
  F5  exactly singular: a zero column, two identical rows, a NaN entry (the solver must report failure)
"""
from __future__ import annotations

import numpy as np
import pytest
import scipy.linalg as sla

import solver_harness as sh

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
GROWTH = 64.0          # TileGJ::kGrowth
SENT = np.array([0x7FF8DEADBEEF0001], np.uint64).view(np.float64)[0]   # NaN with a payload of its own
GUARD = 24             # sentinel doubles after every system
CFGS = list(range(sh.NUM_CFG))
CATCH_ALL = 6


# ------------------------------------------------------------------------------------------------ shapes
def n_grid(max_n: int):
    ns = {1, 2, 3, 4, 5, 7, 8, 9, max_n}
    for k in range(1, max_n // 8 + 1):
        ns |= {8 * k - 1, 8 * k, 8 * k + 1}
    return sorted(n for n in ns if 1 <= n <= max_n)


def shapes(cfg: int):
    """(n, nrhs) pairs: nrhs = 1 and the two widest reachable (both parities of n + nrhs)."""
    _, max_n, max_w = sh.limits(cfg)
    out = []
    if cfg == CATCH_ALL:
        # whatever the tensor-core configurations reject: n beyond 112, or rows wider than 256
        for n in sorted(set(n_grid(16)) | {63, 64, 65, 111, 112, 113, 120, 127, 128, 129, 160}):
            rh = {1, 2} | {r for r in (257 - n, 258 - n) if r >= 1}
            out += [(n, r) for r in sorted(rh)]
        return out
    for n in n_grid(max_n):
        top = max_w - 1 - n            # (n + top) | 1 = max_w - 1: the widest row the dispatcher sends here
        rh = {1} | {r for r in (top, top - 1) if r >= 1}
        if top >= 1:
            out += [(n, r) for r in sorted(rh)]
    return out


# ------------------------------------------------------------------------------------------------ families
def _unit_rows(A):
    return A / np.abs(A).sum(axis=1, keepdims=True)


def f1(rng, n, shift=2.0):
    return _unit_rows(rng.uniform(-1, 1, (n, n)) + shift * np.sqrt(n) * np.eye(n))


def f2_shift(n):
    """Smallest cyclic row shift >= 5 that moves every dominant entry out of its natural 4x4 block (None if none)."""
    i = np.arange(n)
    for s in range(5, 5 + n):
        if np.all(i // 4 != ((i - s) % n) // 4):
            return s
    return None


def f2(rng, n, offdiag=1e-2, shift=None):
    """Diagonally dominant (off-diagonal entries <= offdiag relative), rows shifted cyclically.  With f2_shift(n),
    the natural blocks hold only off-diagonal entries: their inverse is far above kGrowth, so TileGJ pivots."""
    A = _unit_rows(np.eye(n) + offdiag * rng.uniform(-1, 1, (n, n)))
    return np.roll(A, shift if shift is not None else (f2_shift(n) or 1), axis=0)


def _block_at_growth(rng, m, target, scale):
    """m x m block B with max |B^-1| = target, rows at 1-norm `scale` (bisection towards a singular matrix)."""
    M = np.eye(m) + 0.2 * rng.uniform(-1, 1, (m, m))
    N = M.copy()
    if m == 1:
        N[0, 0] = 0.0
    else:
        N[-1] = N[0] if m == 2 else N[0] + N[1]

    def blk(t):
        B = (1 - t) * M + t * N
        if m == 1:          # a 1 x 1 block: its size is its growth
            return scale * B
        return scale * B / np.abs(B).sum(axis=1, keepdims=True)

    def g(t):
        try:
            return np.abs(np.linalg.inv(blk(t))).max()
        except np.linalg.LinAlgError:
            return np.inf

    lo, hi = 0.0, 1.0
    assert g(lo) < target
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if g(mid) < target:
            lo = mid
        else:
            hi = mid
    B = blk(lo if abs(g(lo) / target - 1) < abs(g(hi) / target - 1) else hi)
    assert abs(np.abs(np.linalg.inv(B)).max() / target - 1) < 1e-9
    return B


def f3(rng, n, side):
    """Block lower triangular: block k couples to block k-1 with row 1-norm c, so that the Schur complement a panel
    sees is its diagonal block exactly.  Every third block (and the last) sits at (1 + side * 1e-3) * kGrowth."""
    c = 0.05
    A = np.zeros((n, n))
    nb = (n + 3) // 4
    for k in range(nb):
        r0, m = 4 * k, min(4, n - 4 * k)
        cc = c if k else 0.0
        if k % 3 == 0 or k == nb - 1:
            B = _block_at_growth(rng, m, GROWTH * (1 + side * 1e-3), 1 - cc)
        else:
            B = (1 - cc) * _unit_rows(np.eye(m) + 0.1 * rng.uniform(-1, 1, (m, m)))
        A[r0:r0 + m, r0:r0 + m] = B
        if k:
            L = rng.uniform(-1, 1, (m, 4))
            A[r0:r0 + m, r0 - 4:r0] = cc * L / np.abs(L).sum(axis=1, keepdims=True)
    return A


SCHUR_DELTAS = (1e-4, 1e-6, 1e-8)


def f4_schur(rng, n, delta):
    m = max(1, n // 3)
    n1 = n - m
    A11 = f1(rng, n1, shift=4.0)
    A12 = rng.uniform(-1, 1, (n1, m))
    A21 = rng.uniform(-1, 1, (m, n1))
    Cm = np.eye(m) + 0.3 * rng.uniform(-1, 1, (m, m))
    A22 = A21 @ np.linalg.solve(A11, A12) + delta * Cm
    return _unit_rows(np.block([[A11, A12], [A21, A22]]))


def f5(rng, n, kind):
    if kind == "zero_column":
        A = f1(rng, n)
        A[:, n // 2] = 0.0
    elif kind == "identical_rows":
        # exact in every solver's arithmetic (entries 0 / 1, unit pivots): the second row cancels to zero
        A = np.eye(n)
        r1, r2 = min(1, n - 2), n - 1
        A[r1] = A[r2] = 0.0
        A[r1, r1] = A[r1, r2] = A[r2, r1] = A[r2, r2] = 1.0
    else:
        A = f1(rng, n)
        A[rng.integers(n), rng.integers(n)] = np.nan
    return A


def families(rng, n, schur=True):
    """(name, A, expect_ok, check_backward) for one order n."""
    out = [("F3-below", f3(rng, n, -1), True, True), ("F3-above", f3(rng, n, +1), True, True)]
    if f2_shift(n):     # (no shift empties the natural blocks of a single panel: see the fast-path test below)
        out.append(("F2", f2(rng, n), True, True))
    for s in (1e-6, 1e-8):   # far below kGrowth^-1: every natural block is rejected, whatever the shift
        out.append((f"F4-scale{s:g}", s * f2(rng, n), True, False))
    if f2_shift(n):
        # The growth test assumes rows at unit 1-norm: at 1e5 it accepts natural blocks of entries 1e5 * 1e-2
        # (their inverse is tiny), so the partial-pivoting path is reached only when those blocks are below 1/64.
        out.append(("F4-scale1e+05", 1e5 * f2(rng, n, offdiag=1e-9), True, False))
    if n >= 2:
        if schur:
            out += [(f"F4-schur{d:g}", f4_schur(rng, n, d), True, False) for d in SCHUR_DELTAS]
        out += [(f"F5-{k}", f5(rng, n, k), False, False) for k in ("zero_column", "identical_rows", "nan")]
    return out


# ------------------------------------------------------------------------------------------------ packing
class Batch:
    def __init__(self):
        self.sys = []   # (name, A, B, expect_ok, check_backward)

    def add(self, name, A, B, expect_ok=True, bwd=True):
        self.sys.append((name, A, B, expect_ok, bwd))

    def pack(self, idx):
        ns, nr, Ws, offs, blocks = [], [], [], [0], []
        for i in idx:
            _, A, B, _, _ = self.sys[i]
            n, nrhs = B.shape
            W = (n + nrhs) | 1
            blk = np.full(n * W + GUARD, SENT)
            v = blk[:n * W].reshape(n, W)
            v[:, :n] = A
            v[:, n:n + nrhs] = B
            ns.append(n), nr.append(nrhs), Ws.append(W), blocks.append(blk)
            offs.append(offs[-1] + blk.size)
        return (np.array(ns), np.array(nr), np.array(Ws), np.array(offs, np.int64),
                np.ascontiguousarray(np.concatenate(blocks)))


def run(cfg, a_global, batch, idx):
    n, nrhs, W, off, A = batch.pack(idx)
    A0 = A.copy()
    rowidx, ok = sh.solve(cfg, a_global, n, nrhs, W, off, A)
    roff = np.r_[0, np.cumsum(n)]
    res = []
    for k in range(len(idx)):
        span = A[off[k]:off[k + 1]]
        res.append(dict(n=int(n[k]), nrhs=int(nrhs[k]), W=int(W[k]), A=span, A0=A0[off[k]:off[k + 1]],
                        rowidx=rowidx[roff[k]:roff[k + 1]], ok=int(ok[k])))
    return res


# ------------------------------------------------------------------------------------------------ reference
def reference(A, B):
    """scipy.linalg.solve refined twice with residuals in np.longdouble; also returns the plain solve."""
    x0 = sla.solve(A, B)
    Al = A.astype(np.longdouble)
    Bl = B.astype(np.longdouble)
    x = x0.copy()
    for _ in range(2):
        r = (Bl - Al @ x.astype(np.longdouble)).astype(np.float64)
        x = x + sla.solve(A, r)
    return x, x0


def fwd_err(X, Xref):
    return float(np.abs(X - Xref).max() / np.abs(Xref).max())


def bwd_err(A, X, B):
    """normwise backward error per right-hand side (residual in np.longdouble), max over the columns"""
    Al = A.astype(np.longdouble)
    r = np.abs(B.astype(np.longdouble) - Al @ X.astype(np.longdouble)).max(axis=0).astype(np.float64)
    nA = np.abs(A).sum(axis=1).max()
    return float((r / (nA * np.abs(X).max(axis=0) + np.abs(B).max(axis=0))).max())


def cond_skeel(A, X):
    """cond(A, x) = || |A^-1| |A| |x| || / ||x|| (infinity norm), max over the right-hand sides"""
    v = np.abs(np.linalg.inv(A)) @ (np.abs(A) @ np.abs(X))
    return float((v.max(axis=0) / np.abs(X).max(axis=0)).max())


# Bounds.  Gauss-Jordan elimination is forward stable but not backward stable: its residual is bounded by
# c_n u |A| |A^-1| |A| |x| rather than c_n u |A| |x| (Peters & Wilkinson 1975; Higham, Accuracy and Stability of
# Numerical Algorithms, 2nd ed., section 14.4).  So the normwise backward error may exceed c n u by the factor cond(A, x); the bound is
# 20 n u max(1, cond(A, x)), which stays within a small factor of 20 n u on the well-conditioned F1-F3.  The forward
# error of both LU and Gauss-Jordan is O(n u cond(A, x)); one observed LAPACK error can undershoot that by orders of
# magnitude on an ill-conditioned input, so the first-order bound n u cond(A, x) is admitted next to 16x LAPACK.
TILE_CFGS = (0, 1, 2, 3, 4, 5)   # the TileGJ configurations


def bwd_bound(n, cond):
    return 20 * n * U * max(1.0, cond)


def check_one(tag, r, A, B, expect_ok, check_bwd, stats):
    """list of failure messages (empty: the system passed)"""
    n, nrhs, W = r["n"], r["nrhs"], r["W"]
    if r["ok"] != (1 if expect_ok else 0):
        return [f"{tag}: ok = {r['ok']}"]
    out = r["A"]
    bits, bits0 = out.view(np.uint64), r["A0"].view(np.uint64)
    # nothing outside columns [0, n + nrhs) of rows < n: the padding column and the guard keep their sentinels
    if not np.array_equal(bits[n * W:], bits0[n * W:]):
        return [f"{tag}: guard region written"]
    if not np.array_equal(bits[:n * W].reshape(n, W)[:, n + nrhs:], bits0[:n * W].reshape(n, W)[:, n + nrhs:]):
        return [f"{tag}: padding column written"]
    if not expect_ok:
        return []
    ri = r["rowidx"]
    if not np.array_equal(np.sort(ri), np.arange(n)):
        return [f"{tag}: rowidx is not a permutation {ri}"]
    X = out[:n * W].reshape(n, W)[ri, n:n + nrhs]
    if not np.isfinite(X).all():
        return [f"{tag}: non-finite solution"]
    Xref, Xlapack = reference(A, B)
    cond = cond_skeel(A, Xref)
    fe, fe_lapack = fwd_err(X, Xref), fwd_err(Xlapack, Xref)
    fails = []
    if fe > max(16 * fe_lapack, n * U * cond, 1e-13):
        fails.append(f"{tag}: forward error {fe:.3e} (LAPACK {fe_lapack:.3e}, n u cond {n * U * cond:.3e})")
    stats["fwd"] = max(stats["fwd"], fe)
    if check_bwd:
        be = bwd_err(A, X, B)
        if be > bwd_bound(n, cond):
            fails.append(f"{tag}: backward error {be:.3e} > {bwd_bound(n, cond):.3e} (cond {cond:.2f})")
        stats["bwd"] = max(stats["bwd"], be)
        stats["bwd_units"] = max(stats["bwd_units"], be / (n * U))
    return fails


def build_batch(cfg):
    rng = np.random.default_rng(1000 + cfg)
    batch = Batch()
    shp = shapes(cfg)
    for n, nrhs in shp:
        batch.add(f"F1 n={n} nrhs={nrhs}", f1(rng, n), rng.uniform(-1, 1, (n, nrhs)))
    # the other families at the widest right-hand side of each order (F1 covers the widths)
    widest = {}
    for n, nrhs in shp:
        widest[n] = max(widest.get(n, 0), nrhs)
    for n, nrhs in sorted(widest.items()):
        for name, A, expect, bwd in families(rng, n, schur=cfg not in TILE_CFGS):
            B = rng.uniform(-1, 1, (n, nrhs))
            batch.add(f"{name} n={n} nrhs={nrhs}", A, B, expect, bwd)
    return batch


@pytest.mark.parametrize("cfg", CFGS)
def test_local_solver_against_extended_precision(cfg):
    batch = build_batch(cfg)
    allidx = list(range(len(batch.sys)))
    res_g = run(cfg, True, batch, allidx)
    max_n = max(B.shape[0] for _, _, B, _, _ in batch.sys)
    shared = [i for i in allidx
              if sh.fits_shared(cfg, max_n, batch.sys[i][2].shape[0] * ((sum(batch.sys[i][2].shape)) | 1) + GUARD)]
    res_s = run(cfg, False, batch, shared) if shared else []
    # A in shared memory and in the global workspace: the same arithmetic, bitwise the same results
    for i, rs in zip(shared, res_s):
        rg = res_g[i]
        assert rs["ok"] == rg["ok"], batch.sys[i][0]
        assert np.array_equal(rs["A"].view(np.uint64), rg["A"].view(np.uint64)), batch.sys[i][0]
        assert np.array_equal(rs["rowidx"], rg["rowidx"]), batch.sys[i][0]
    stats = {"fwd": 0.0, "bwd": 0.0, "bwd_units": 0.0}
    fails = []
    for i, rg in enumerate(res_g):
        name, A, B, expect_ok, bwd = batch.sys[i]
        fails += check_one(f"cfg {cfg} {name}", rg, A, B, expect_ok, bwd, stats)
    print(f"\ncfg {cfg}: {len(allidx)} systems (global A), {len(shared)} also with A in shared memory; "
          f"max forward error {stats['fwd']:.2e}, max backward error (F1-F3) {stats['bwd']:.2e} "
          f"= {stats['bwd_units']:.1f} n u; {len(fails)} failed")
    assert not fails, f"{len(fails)} of {len(allidx)} systems failed:\n" + "\n".join(fails[:30])


@pytest.mark.parametrize("cfg", CFGS)
def test_team_reuse_across_systems_is_bitwise_stable(cfg):
    """More systems than resident teams, mixed sizes, neighbours in one CTA different: every system of the batch
    equals the same system solved alone, bitwise (catches teams of one CTA overlapping in shared memory)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    team, _, _ = sh.limits(cfg)
    resident = sms * (2048 // team)      # upper bound: 2048 threads per SM
    rng = np.random.default_rng(77 + cfg)
    _, cmax, _ = sh.limits(cfg)
    cmax = min(cmax, 160)
    shp = [(n, r) for n, r in shapes(cfg) if sh.fits_shared(cfg, cmax, n * ((n + r) | 1) + GUARD)]
    K = 7                               # coprime to the 4 teams of a CTA
    pick = [shp[j] for j in rng.choice(len(shp), K, replace=False)] if len(shp) >= K else \
        [shp[j % len(shp)] for j in range(K)]
    base = Batch()
    for n, nrhs in pick:
        base.add(f"n={n} nrhs={nrhs}", f2(rng, n) if rng.random() < 0.5 else f1(rng, n), rng.uniform(-1, 1, (n, nrhs)))
    nsys = 2 * resident + 3
    for a_global in (True, False):
        mx = max(B.shape[0] for _, _, B, _, _ in base.sys)
        spans = [B.shape[0] * (sum(B.shape) | 1) + GUARD for _, _, B, _, _ in base.sys]
        if not a_global and not sh.fits_shared(cfg, mx, max(spans)):
            continue
        alone = [run(cfg, a_global, base, [k])[0] for k in range(K)]
        big = Batch()
        big.sys = [base.sys[i % K] for i in range(nsys)]
        res = run(cfg, a_global, big, list(range(nsys)))
        for i, r in enumerate(res):
            a = alone[i % K]
            assert r["ok"] == a["ok"] == 1, (cfg, a_global, i)
            assert np.array_equal(r["A"].view(np.uint64), a["A"].view(np.uint64)), (cfg, a_global, i)
            assert np.array_equal(r["rowidx"], a["rowidx"]), (cfg, a_global, i)


@pytest.mark.xfail(strict=True, reason="TileGJ's partial-pivoting path forms R = A11^-1 * (pivot rows) from an explicit "
                   "inverse of the chosen 4x4 block; when the trailing Schur complement is delta * C, that block has "
                   "condition ~1/delta and R, and the update A22 -= A21 R, lose accuracy like 1/delta^2")
@pytest.mark.parametrize("cfg", TILE_CFGS)
def test_tilegj_ill_conditioned_schur_complement(cfg):
    """F4 with a trailing Schur complement delta * C (kappa ~ 1/delta): SmemGJ meets the forward-error bound
    (test above); the tensor-core configurations do not, by orders of magnitude at delta = 1e-6 and 1e-8."""
    rng = np.random.default_rng(2000 + cfg)
    batch = Batch()
    widest = {}
    for n, nrhs in shapes(cfg):
        widest[n] = max(widest.get(n, 0), nrhs)
    for n, nrhs in sorted(widest.items()):
        if n >= 2:
            for d in SCHUR_DELTAS:
                batch.add(f"F4-schur{d:g} n={n} nrhs={nrhs}", f4_schur(rng, n, d), rng.uniform(-1, 1, (n, nrhs)),
                          True, False)
    res = run(cfg, True, batch, list(range(len(batch.sys))))
    stats = {"fwd": 0.0, "bwd": 0.0, "bwd_units": 0.0}
    fails = []
    for (name, A, B, expect_ok, bwd), r in zip(batch.sys, res):
        fails += check_one(f"cfg {cfg} {name}", r, A, B, expect_ok, bwd, stats)
    assert not fails, f"{len(fails)} of {len(res)} systems failed:\n" + "\n".join(fails[:30])


@pytest.mark.xfail(strict=True, reason="the fast path of TileGJ accepts a natural 4x4 block on the size of its "
                   "inverse alone and inverts it without pivoting inside: a block whose dominant entries lie off its "
                   "diagonal has a tame inverse but small leading pivots, and the inverse loses ~1/pivot digits")
@pytest.mark.parametrize("cfg", TILE_CFGS)
def test_tilegj_fast_path_block_with_small_leading_pivots(cfg):
    """Rows of every 4x4 block shifted by one (dominant entries off the block diagonal, 1e-6 relative on it): the
    final inverse is ~ a permutation, so the growth test accepts the block; well conditioned (cond ~ 1)."""
    _, max_n, max_w = sh.limits(cfg)
    n = min(16, max_n)
    rng = np.random.default_rng(3000 + cfg)
    P = np.kron(np.eye(n // 4), np.roll(np.eye(4), 1, axis=0))
    A = _unit_rows(P + 1e-6 * rng.uniform(0.5, 1.0, (n, n)))
    batch = Batch()
    batch.add(f"shifted blocks n={n}", A, rng.uniform(-1, 1, (n, 1)))
    r = run(cfg, True, batch, [0])[0]
    stats = {"fwd": 0.0, "bwd": 0.0, "bwd_units": 0.0}
    fails = check_one(f"cfg {cfg} shifted blocks", r, A, batch.sys[0][2], True, True, stats)
    assert not fails, fails
