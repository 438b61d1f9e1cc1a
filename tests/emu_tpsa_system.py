"""ctypes binding of tests/emu/_emu_tpsa_system.so -- the host build of the TPSA system assembly
(porepy_b200/csrc/tpsa_system.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_tpsa_system.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from emu_binding import _p
from emu_tpsa import EmuTpsaFaceGrid

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_tpsa_system.cpp")
LIB = os.path.join(HERE, "emu", "_emu_tpsa_system.so")
CSRC = os.path.join(os.path.dirname(HERE), "porepy_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "tpsa_face.cuh"), os.path.join(CSRC, "tpsa_system.cuh"), os.path.join(CSRC, "views.hpp")]

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
        _lib.emu_tpsa_system.restype = C.c_int
        _lib.emu_tpsa_system_get.restype = None
    return _lib


class EmuTpsaSystemFaceGrid(EmuTpsaFaceGrid):
    """``EmuTpsaFaceGrid`` plus ``FaceGrid.tpsa_system`` / ``tpsa_rhs`` on the host build of tpsa_system.cuh: the same
    arguments; the matrix comes back as a scipy CSR and b as a NumPy array, stage times 0."""

    def _run(self, nd, mu, lmbda, vol, codes, robin_diag, face_flags, face_areas, g, f=None, sr=None, sp=None):
        L = lib()
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)  # noqa: E731
        mu, lam, vol, rob, area, g, f, sr, sp = (f64(a) for a in (mu, lmbda, vol, robin_diag, face_areas, g, f, sr, sp))
        cod = np.ascontiguousarray(codes, np.uint8)
        flags = np.ascontiguousarray(face_flags, np.uint8)
        h, nrows, nnz = C.c_void_p(), C.c_int64(), C.c_int64()
        rc = L.emu_tpsa_system(*self._cf(), _p(self.geo[0], C.c_double), _p(self.geo[1], C.c_double),
                               _p(area, C.c_double), _p(self.geo[2], C.c_double), C.c_int(nd), _p(mu, C.c_double),
                               _p(lam, C.c_double), _p(vol, C.c_double), _p(cod, C.c_uint8), _p(rob, C.c_double),
                               _p(flags, C.c_uint8), _p(g, C.c_double), _p(f, C.c_double), _p(sr, C.c_double),
                               _p(sp, C.c_double), C.byref(h), C.byref(nrows), C.byref(nnz))
        if rc:
            raise ValueError("face with more than two neighbouring cells" if rc == 1 else "too many face neighbours")
        n, z = nrows.value, nnz.value
        ip, ix, a, b = np.zeros(n + 1, np.int32), np.zeros(max(z, 1), np.int32), np.zeros(max(z, 1)), np.zeros(n)
        L.emu_tpsa_system_get(h, _p(ip, C.c_int32), _p(ix, C.c_int32), _p(a, C.c_double), _p(b, C.c_double))
        return sps.csr_matrix((a[:z], ix[:z], ip), shape=(n, n)), b

    def tpsa_system(self, nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas):
        self._args = (nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas)
        A, _ = self._run(*self._args, np.zeros(nd * self.nf))
        return A, [0.0, 0.0]

    def tpsa_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        _, b = self._run(*self._args, bc_values, body_force, angular_source, mass_source)
        assert b.size == n
        return b
