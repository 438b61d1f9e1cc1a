"""ctypes binding of tests/emu/_emu_dual_hybrid.so -- the host build of the hybridization of MVEM and RT0
(porepy_b200/csrc/dual_hybrid.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_dual_hybrid.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from emu_dual import CSRC, EmuDualGrid, _p

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_dual_hybrid.cpp")
LIB = os.path.join(HERE, "emu", "_emu_dual_hybrid.so")
DEPS = [SRC, os.path.join(CSRC, "dual_cell.cuh"), os.path.join(CSRC, "dual_hybrid.cuh"),
        os.path.join(CSRC, "group_block.cuh"), os.path.join(CSRC, "views.hpp"),
        os.path.join(os.path.dirname(HERE), "include", "poreb200.h")]

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
        _lib.emu_dual_hybrid.restype = C.c_int64
    return _lib


class EmuHybridDualGrid(EmuDualGrid):
    """``EmuDualGrid`` with ``DualGrid.hybrid_system`` / ``hybrid_recover`` on the host build of dual_hybrid.cuh.  Like
    the device handle, it keeps the geometry and the method of the last ``discretize`` for the saddle-point mode."""

    def discretize(self, method, geo, perm, rot):
        out = super().discretize(method, geo, perm, rot)
        self._geo = list(geo) + [perm, rot]
        self._method = int(method)
        return out

    def _hybrid(self, mode, geo, codes, robin_weight, face_areas, values, lam):
        """One call of emu_dual_hybrid: H values, rhs, [u; p] and the status."""
        ip, ix = self.mass_pattern()
        if mode == 0:   # PB_DUAL_HYBRID_VEM: the given geometry, MVEM
            arrs, method, norm = list(geo), 0, 0.0
        else:           # PB_DUAL_HYBRID_SADDLE: the geometry and values of the last discretize
            arrs, method = self._geo + [np.ones(self.nc)], self._method
            mass = self._values[0]
            norm = float(np.abs(sps.csr_matrix((mass, ix, ip), shape=(self.nf, self.nf))).sum(axis=1).max())
        if int(np.diff(self.cf_ip).max()) > 32:
            raise NotImplementedError("hybridization: a cell has more than 32 faces")
        arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in arrs]
        extra = [np.ascontiguousarray(a, dtype=np.float64) for a in (robin_weight, face_areas, values)]
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        hval, rhs, up = np.zeros(ix.size), np.zeros(self.nf), np.zeros(self.nf + self.nc)
        lam = None if lam is None else np.ascontiguousarray(lam, dtype=np.float64)
        st = lib().emu_dual_hybrid(
            C.c_int(self.nd), C.c_int(method), C.c_int(int(mode)), C.c_int64(self.nc), C.c_int64(self.nf),
            C.c_int64(self.nn), _p(self.cf_ip, C.c_int32), _p(self.cf_ix, C.c_int32), _p(self.cf_sg, C.c_int8),
            _p(self.fn_ip, C.c_int32), _p(self.fn_ix, C.c_int32), _p(ip, C.c_int32), _p(ix, C.c_int32),
            *[_p(a, C.c_double) for a in arrs], _p(cod, C.c_uint8), *[_p(a, C.c_double) for a in extra],
            C.c_double(norm), _p(lam, C.c_double), _p(hval, C.c_double), _p(rhs, C.c_double), _p(up, C.c_double))
        if st <= -2:
            raise np.linalg.LinAlgError(f"hybridization: the local matrix of cell {-2 - st} is singular")
        return hval, rhs, up, int(st)

    def hybrid_system(self, mode, geo, codes, robin_weight, face_areas, values):
        """``DualGrid.hybrid_system`` on the host build: H as a ``HostCsr`` (tests/emu_sparse.py)."""
        from emu_sparse import HostCsr
        ip, ix = self.mass_pattern()
        hval, rhs, _, bad = self._hybrid(mode, geo, codes, robin_weight, face_areas, values, None)
        return HostCsr(sps.csr_matrix((hval, ix, ip), shape=(self.nf, self.nf))), rhs, bad, 0.0

    def hybrid_recover(self, mode, geo, codes, values, lam):
        _, _, up, _ = self._hybrid(mode, geo, codes, np.zeros(self.nf), np.zeros(self.nf), values, lam)
        return up, 0.0
