"""ctypes binding of tests/gpu_harness/_solver_harness.so -- the dense local solvers of the node routines
(Cfg0..Cfg7 of porepy_b200/csrc/plan.hpp) on caller-supplied systems.  TEST INFRASTRUCTURE ONLY (see
tests/gpu_harness/solver_harness.cu); the product never loads it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "gpu_harness", "solver_harness.cu")
LIB = os.path.join(HERE, "gpu_harness", "_solver_harness.so")
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "porepy_b200", "csrc")
NUM_CFG = 8


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
        L.sh_last_error.restype = C.c_char_p
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def limits(cfg: int):
    """(team, max_n, max_w) of configuration cfg, read from the compiled solver types."""
    team, max_n, max_w = C.c_int(), C.c_int(), C.c_int()
    if lib().sh_limits(C.c_int(cfg), C.byref(team), C.byref(max_n), C.byref(max_w)):
        raise ValueError(lib().sh_last_error().decode())
    return team.value, max_n.value, max_w.value


def fits_shared(cfg: int, max_n: int, span: int) -> bool:
    """Whether systems of order <= max_n spanning <= span doubles fit configuration cfg's shared memory."""
    return bool(lib().sh_fits_shared(C.c_int(cfg), C.c_int(max_n), C.c_int64(span)))


def solve(cfg: int, a_global: bool, n, nrhs, W, a_off, A):
    """One launch over all systems.  ``A`` (float64, contiguous) is updated in place; returns (rowidx, ok) with
    rowidx concatenated over the systems (n[i] entries each)."""
    n = np.ascontiguousarray(n, np.int32)
    nrhs = np.ascontiguousarray(nrhs, np.int32)
    W = np.ascontiguousarray(W, np.int32)
    a_off = np.ascontiguousarray(a_off, np.int64)
    assert A.dtype == np.float64 and A.flags.c_contiguous and A.size >= a_off[-1]
    rowidx = np.full(int(n.sum()), -1, np.int32)
    ok = np.full(n.size, -1, np.int32)
    rc = lib().sh_solve(C.c_int(cfg), C.c_int(int(a_global)), C.c_int(n.size), _p(n, C.c_int32),
                        _p(nrhs, C.c_int32), _p(W, C.c_int32), _p(a_off, C.c_int64), _p(A, C.c_double),
                        _p(rowidx, C.c_int32), _p(ok, C.c_int32))
    if rc:
        raise RuntimeError(lib().sh_last_error().decode())
    return rowidx, ok
