"""ctypes binding of tests/emu/_emu_tpsa.so -- the host build of the per-face TPSA routine
(porepy_b200/csrc/tpsa_face.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_tpsa.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emu_binding import EmuBackedFaceGrid, _p

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_tpsa.cpp")
LIB = os.path.join(HERE, "emu", "_emu_tpsa.so")
CSRC = os.path.join(os.path.dirname(HERE), "porepy_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "tpsa_face.cuh"), os.path.join(CSRC, "views.hpp")]

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
    return _lib


class EmuTpsaFaceGrid(EmuBackedFaceGrid):
    """``EmuBackedFaceGrid`` (TPFA, upwinding on the host build) plus ``FaceGrid.tpsa`` on the host build of
    tpsa_face.cuh: same arguments, same value arrays (``fv.tpsa_value_counts``), kernel time 0."""

    def tpsa(self, nd, mu, codes, robin_diag, face_flags, fc_indptr, face_areas):
        from porepy_b200.fv import tpsa_value_counts
        L = lib()
        ip = np.ascontiguousarray(fc_indptr, np.int32)
        mu = np.ascontiguousarray(mu, np.float64)
        cod = np.ascontiguousarray(codes, np.uint8)
        rob = None if robin_diag is None else np.ascontiguousarray(robin_diag, np.float64)
        flags = np.ascontiguousarray(face_flags, np.uint8)
        area = np.ascontiguousarray(face_areas, np.float64)
        out = [np.zeros(n) for n in tpsa_value_counts(nd, self.nf, int(ip[-1]))]
        ptrs = (C.POINTER(C.c_double) * len(out))(*[_p(a, C.c_double) for a in out])
        rc = L.emu_facegrid_tpsa(*self._cf(), _p(self.geo[0], C.c_double), _p(self.geo[1], C.c_double),
                                 _p(area, C.c_double), _p(self.geo[2], C.c_double), C.c_int(nd), _p(mu, C.c_double),
                                 _p(cod, C.c_uint8), _p(rob, C.c_double), _p(flags, C.c_uint8), _p(ip, C.c_int32), ptrs)
        if rc:
            raise ValueError("face with more than two neighbouring cells")
        return out, 0.0
