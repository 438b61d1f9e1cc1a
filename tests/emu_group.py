"""ctypes binding of tests/emu/_emu_group.so -- the host build of the grouped block-Jacobi inverse
(porepy_b200/csrc/group_block.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_group.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_group.cpp")
LIB = os.path.join(HERE, "emu", "_emu_group.so")
CSRC = os.path.join(os.path.dirname(HERE), "porepy_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "group_block.cuh"), os.path.join(CSRC, "views.hpp")]

_lib = None


def _build():
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in DEPS):
        return
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", LIB, SRC])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        _lib.emu_group_inv.restype = C.c_int64
    return _lib


def group_inverses(a, groups):
    """(inverses as a flat array at ``groups.inv_offsets``, lowest failing group or -1) for the CSR matrix ``a``."""
    a = sps.csr_matrix(a)
    ip, ix = a.indptr.astype(np.int32), a.indices.astype(np.int32)
    data = np.ascontiguousarray(a.data, np.float64)
    rows, cols = groups.rows.astype(np.int32), groups.cols.astype(np.int32)
    ptr, off = np.ascontiguousarray(groups.ptr), np.ascontiguousarray(groups.inv_offsets[:-1])
    out = np.full(int(groups.inv_offsets[-1]), np.nan)
    p = lambda arr, t: arr.ctypes.data_as(C.POINTER(t))  # noqa: E731
    bad = lib().emu_group_inv(p(ip, C.c_int32), p(ix, C.c_int32), p(data, C.c_double), C.c_int64(groups.num_groups),
                              p(ptr, C.c_int64), p(rows, C.c_int32), p(cols, C.c_int32), p(off, C.c_int64),
                              p(out, C.c_double))
    return out, int(bad)
