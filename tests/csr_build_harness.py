"""ctypes binding of tests/gpu_harness/_csr_build_harness.so -- the offset scan, warp sort and unique-compaction of
porepy_b200/csrc/csr_build.cuh on caller-supplied data.  TEST INFRASTRUCTURE ONLY (see
tests/gpu_harness/csr_build_harness.cu); the product never loads it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "gpu_harness", "csr_build_harness.cu")
LIB = os.path.join(HERE, "gpu_harness", "_csr_build_harness.so")
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "porepy_b200", "csrc")


def _deps():
    from porepy_b200 import build as b
    return [SRC, os.path.abspath(b.__file__), os.path.join(ROOT, "include", "poreb200.h")] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".hpp"))]


def _build():
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in _deps()):
        return
    from porepy_b200 import build as b
    subprocess.check_call([b._nvcc(), *b.NVCC_FLAGS, "-shared", "-o", LIB, SRC])


_lib = None


def lib():
    global _lib
    if _lib is None:
        _build()
        L = C.CDLL(LIB)
        L.cb_last_error.restype = C.c_char_p
        L.cb_launches.restype = C.c_int64
        _lib = L
    return _lib


def launches() -> int:
    return lib().cb_launches()


def scan(counts, off64: bool, legacy_stream: bool = False):
    """(offsets, total): offsets (n + 1 entries, int64 with off64 else int32) and the exact int64 total."""
    counts = np.ascontiguousarray(counts, np.int32)
    offsets = np.full(counts.size + 1, -7, np.int64 if off64 else np.int32)
    total = C.c_int64(-7)
    rc = lib().cb_scan(C.c_int(int(off64)), C.c_int(int(legacy_stream)),
                       counts.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int64(counts.size),
                       offsets.ctypes.data_as(C.c_void_p), C.byref(total))
    if rc:
        raise RuntimeError(lib().cb_last_error().decode())
    return offsets, total.value


def sort_unique(keys, payload):
    """(sorted keys, their payload, unique keys) from one warp; keys int32 or uint64, payload float64."""
    keys = np.array(keys)
    key64 = keys.dtype == np.uint64
    assert key64 or keys.dtype == np.int32
    keys = np.ascontiguousarray(keys)
    pay = np.ascontiguousarray(payload, np.float64).copy()
    uniq = np.zeros_like(keys)
    nuniq = C.c_int(-1)
    rc = lib().cb_sort_unique(C.c_int(int(key64)), C.c_int(keys.size), keys.ctypes.data_as(C.c_void_p),
                              pay.ctypes.data_as(C.POINTER(C.c_double)), uniq.ctypes.data_as(C.c_void_p),
                              C.byref(nuniq))
    if rc:
        raise RuntimeError(lib().cb_last_error().decode())
    return keys, pay, uniq[:nuniq.value]
