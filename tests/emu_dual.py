"""ctypes binding of tests/emu/_emu_dual.so -- the host build of the per-(cell, face) routines of MVEM and RT0
(porepy_b200/csrc/dual_cell.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_dual.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from porepy_b200.fv import DevicePlan, DualGrid

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_dual.cpp")
LIB = os.path.join(HERE, "emu", "_emu_dual.so")
CSRC = os.path.join(os.path.dirname(HERE), "porepy_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "dual_cell.cuh"), os.path.join(CSRC, "views.hpp")]

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
        _lib.emu_dual_discretize.restype = C.c_int64
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


class EmuDualGrid(DualGrid):
    """``fv.DualGrid`` on the host build of dual_cell.cuh: same patterns, same value arrays, kernel time 0 (no device
    system: ``assemble_matrix_rhs`` then uses the host formulas)."""

    def __init__(self, sd):
        cf = sps.csc_matrix(sd.cell_faces, copy=True)
        cf.sort_indices()
        fn = sps.csc_matrix(sd.face_nodes)
        self.nd, self.nc, self.nf, self.nn = int(sd.dim), sd.num_cells, sd.num_faces, sd.num_nodes
        self.cf_ip, self.cf_ix = cf.indptr.astype(np.int32), cf.indices.astype(np.int32)
        self.cf_sg = np.asarray(cf.data).astype(np.int8)
        self.fn_ip, self.fn_ix = fn.indptr.astype(np.int32), fn.indices.astype(np.int32)
        self.fingerprint = DevicePlan._fingerprint(sd, sd.cell_faces, sd.face_nodes)
        self.h = None   # no device handle: assemble_matrix_rhs takes the host formulas
        self._mass = None
        self._proj = None
        self._values = None
        self.pattern_seconds = 0.0
        self.live, self.current = [], None

    def mass_pattern(self):
        if self._mass is None:
            L = lib()
            nnz = C.c_int64(0)
            L.emu_dual_pattern(C.c_int64(self.nc), C.c_int64(self.nf), _p(self.cf_ip, C.c_int32),
                               _p(self.cf_ix, C.c_int32), C.byref(nnz), None, None)
            ip, ix = np.empty(self.nf + 1, np.int32), np.empty(nnz.value, np.int32)
            L.emu_dual_pattern(C.c_int64(self.nc), C.c_int64(self.nf), _p(self.cf_ip, C.c_int32),
                               _p(self.cf_ix, C.c_int32), C.byref(nnz), _p(ip, C.c_int32), _p(ix, C.c_int32))
            self._mass = (ip, ix)
        return self._mass

    def discretize(self, method, geo, perm, rot):
        ip, ix = self.mass_pattern()
        arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in list(geo) + [perm, rot]]
        mass, proj = np.zeros(ix.size), np.zeros(3 * int(self.cf_ip[-1]))
        bad = lib().emu_dual_discretize(
            C.c_int(self.nd), C.c_int(int(method)), C.c_int64(self.nc), C.c_int64(self.nf), C.c_int64(self.nn),
            _p(self.cf_ip, C.c_int32), _p(self.cf_ix, C.c_int32), _p(self.cf_sg, C.c_int8), _p(self.fn_ip, C.c_int32),
            _p(self.fn_ix, C.c_int32), _p(ip, C.c_int32), _p(ix, C.c_int32), *[_p(a, C.c_double) for a in arrs],
            _p(mass, C.c_double), _p(proj, C.c_double))
        self._values = (mass, proj)
        return int(bad), 0.0

    def download(self):
        return tuple(a.copy() for a in self._values)

    @classmethod
    def for_grid(cls, sd) -> "EmuDualGrid":
        return cls(sd)
