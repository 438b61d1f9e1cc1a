"""The shared steps of the device CSR builders (porepy_b200/csrc/csr_build.cuh), run on their own through
tests/gpu_harness: the offset scan every builder turns its row counts into row offsets with, and the warp bitonic
sort and unique-compaction of the plan's pattern rows, its sub-cell topology and the SpGEMM rows.

The overflow paths cannot be reached through the public ABI without several GB of device memory: here the scan is
given counts whose exact total is 2^31 - 1 or 2^31, where an int32 accumulation would wrap to a negative number, and
each builder's limit rule is applied to the total it returns.
"""
from __future__ import annotations

import numpy as np
import pytest

import csr_build_harness as cb

pytestmark = pytest.mark.gpu

I32_MAX = 2 ** 31 - 1
# the refusal rule of each builder on the exact total (the offsets are int32 everywhere but Tpsa poromechanics'
# block offsets; its column indices are int32 all the same)
REFUSES = {
    "plan patterns": lambda t: t > I32_MAX,          # PB_EINVAL "pattern exceeds 2^31 entries; split the grid"
    "sub-cell topology": lambda t: t > I32_MAX,      # PB_EINVAL "grid too large for 32-bit sub-cell indices; ..."
    "sparse algebra": lambda t: t >= I32_MAX,        # PB_ENOTIMPL "... exceeds int32 indices"
    "Tpsa system": lambda t: t >= I32_MAX,           # PB_ENOTIMPL "Tpsa system: the matrix does not fit int32 indices"
}


@pytest.mark.parametrize("off64", [False, True], ids=["int32", "int64"])
@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 3_000_017])
def test_scan_matches_cumsum(n, off64):
    rng = np.random.default_rng(n)
    counts = rng.integers(0, 60, n).astype(np.int32)
    if n > 1:
        counts[rng.integers(0, n, max(1, n // 7))] = 0           # empty rows
    l0 = cb.launches()
    offsets, total = cb.scan(counts, off64)
    assert cb.launches() - l0 == 1
    ref = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
    assert offsets.dtype == (np.int64 if off64 else np.int32)
    np.testing.assert_array_equal(offsets, ref)
    assert total == int(ref[-1])


@pytest.mark.parametrize("off64", [False, True], ids=["int32", "int64"])
def test_scan_on_the_legacy_default_stream(off64):
    counts = np.random.default_rng(5).integers(0, 9, 200_003).astype(np.int32)
    offsets, total = cb.scan(counts, off64, legacy_stream=True)
    np.testing.assert_array_equal(offsets, np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]))
    assert total == int(counts.sum(dtype=np.int64))


@pytest.mark.parametrize("counts,expect,refused_by", [
    ([2 ** 30, 2 ** 30 - 1], I32_MAX, {"sparse algebra", "Tpsa system"}),
    ([2 ** 30, 2 ** 30], 2 ** 31, set(REFUSES)),
    ([2 ** 31 - 1] * 3, 3 * I32_MAX, set(REFUSES)),
])
def test_scan_total_is_exact_past_int32(counts, expect, refused_by):
    # an int32 accumulation reports a wrong total: negative at 2^31, positive again at 3 (2^31 - 1)
    wrapped = int(np.cumsum(np.array(counts, np.int32), dtype=np.int32)[-1])
    assert (wrapped == expect) == (expect <= I32_MAX)
    _, t32 = cb.scan(counts, off64=False)
    off64, t64 = cb.scan(counts, off64=True)
    assert t32 == expect and t64 == expect
    np.testing.assert_array_equal(off64, np.concatenate([[0], np.cumsum(np.array(counts, np.int64))]))
    assert {name for name, refuses in REFUSES.items() if refuses(t32)} == refused_by


def _check_sort_unique(keys, where):
    pay = np.arange(keys.size, dtype=np.float64)
    k, p, u = cb.sort_unique(keys, pay)
    np.testing.assert_array_equal(k, np.sort(keys), err_msg=where)
    idx = p.astype(np.int64)
    np.testing.assert_array_equal(np.sort(idx), np.arange(keys.size), err_msg=where)   # payload permuted, not lost
    np.testing.assert_array_equal(keys[idx], k, err_msg=where)                          # and moved with its key
    np.testing.assert_array_equal(u, np.unique(keys), err_msg=where)


# spans up to the largest capacity of each caller: 256 pattern candidates, 1024 (cell, face) keys per node,
# 8192 slots of the SpGEMM hash table
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 255, 256, 1000, 1024, 4097, 8192])
def test_warp_sort_unique_int32(n):
    rng = np.random.default_rng(100 + n)
    for keys in (rng.integers(0, max(1, n // 3), n), rng.integers(0, 2 ** 31 - 1, n), np.full(n, 7),
                 np.arange(n)[::-1], np.arange(n)):
        _check_sort_unique(keys.astype(np.int32), f"n={n}")


@pytest.mark.parametrize("n", [1, 3, 32, 64, 65, 700, 1024])
def test_warp_sort_unique_uint64(n):
    rng = np.random.default_rng(200 + n)
    cell = rng.integers(0, max(1, n // 4), n).astype(np.uint64)
    face = rng.integers(0, 6, n).astype(np.uint64)
    big = (np.uint64(0xFFFFFFFE) << np.uint64(32)) | rng.integers(0, 2 ** 32 - 1, n).astype(np.uint64)
    for keys in ((cell << np.uint64(32)) | face, big):
        _check_sort_unique(keys, f"n={n}")
