"""ctypes binding of tests/emu/_emu_tpsa_thm.so -- the host build of the TPSA thermo-poromechanics system
(porepy_b200/csrc/tpsa_system.cuh with two scalar balances).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_tpsa_thm.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from emu_binding import _p
from emu_tpsa_poromech import EmuTpsaPoroFaceGrid

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_tpsa_thm.cpp")
LIB = os.path.join(HERE, "emu", "_emu_tpsa_thm.so")
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
        _lib.emu_tpsa_thm_system.restype = C.c_int
        _lib.emu_tpsa_thm_balance_rows.restype = C.c_int
        _lib.emu_tpsa_thm_get.restype = None
    return _lib


class EmuTpsaThmFaceGrid(EmuTpsaPoroFaceGrid):
    """``EmuTpsaPoroFaceGrid`` plus ``FaceGrid.tpsa_thm_system`` / ``tpsa_thm_rhs`` / ``tpsa_thm_balance_rows`` on the host
    build, for the scipy stand-in of the device algebra (tests/emu_sparse.py)."""

    def tpsa_thm_system(self, nd, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                        flux_pattern):
        self._thm = (nd, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                     flux_pattern.to_scipy())
        A, _ = self._run_thm(np.zeros(nd * self.nf))
        from emu_sparse import HostCsr
        H = HostCsr(A)
        H.m = A                              # keep the pattern exactly as built (explicit zeros included)
        return H, [0.0, 0.0]

    def _run_thm(self, g, f=None, sr=None, sp=None):
        L = lib()
        nd, mu, lmbda, alpha, vol, codes, robin_diag, face_flags, face_areas, fp = self._thm
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)  # noqa: E731
        mu, lam, al, vol, rob, area, g, f, sr, sp = (f64(a) for a in (mu, lmbda, alpha, vol, robin_diag, face_areas,
                                                                      g, f, sr, sp))
        cod = np.ascontiguousarray(codes, np.uint8)
        flags = np.ascontiguousarray(face_flags, np.uint8)
        fp = sps.csr_matrix(fp)
        fp.sort_indices()
        fp_ip, fp_ix = fp.indptr.astype(np.int32), fp.indices.astype(np.int32)
        h, nrows, nnz = C.c_void_p(), C.c_int64(), C.c_int64()
        rc = L.emu_tpsa_thm_system(*self._cf(), _p(self.geo[0], C.c_double), _p(self.geo[1], C.c_double),
                                   _p(area, C.c_double), _p(self.geo[2], C.c_double), C.c_int(nd),
                                   _p(mu, C.c_double), _p(lam, C.c_double), _p(al, C.c_double), _p(vol, C.c_double),
                                   _p(cod, C.c_uint8), _p(rob, C.c_double), _p(flags, C.c_uint8),
                                   _p(fp_ip, C.c_int32), _p(fp_ix, C.c_int32), _p(g, C.c_double),
                                   _p(f, C.c_double), _p(sr, C.c_double), _p(sp, C.c_double), C.byref(h),
                                   C.byref(nrows), C.byref(nnz))
        if rc:
            raise ValueError("face with more than two neighbouring cells" if rc == 1 else "too many face neighbours")
        n, z = nrows.value, nnz.value
        ip, ix, a, b = np.zeros(n + 1, np.int32), np.zeros(max(z, 1), np.int32), np.zeros(max(z, 1)), np.zeros(n)
        L.emu_tpsa_thm_get(h, _p(ip, C.c_int32), _p(ix, C.c_int32), _p(a, C.c_double), _p(b, C.c_double))
        return sps.csr_matrix((a[:z], ix[:z], ip), shape=(n, n)), b

    def tpsa_thm_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        import torch
        _, b = self._run_thm(bc_values, body_force, angular_source, mass_source)
        assert b.size == n
        return torch.as_tensor(b)

    def tpsa_thm_balance_rows(self, A, jf, neg_res, rhs, missing=None):
        L = lib()
        a = A.m
        j = sps.csr_matrix(jf.to_scipy())
        assert j.shape == (2 * self.nc, 3 * self.nc)
        jp, jx, ja = j.indptr.astype(np.int32), j.indices.astype(np.int32), np.ascontiguousarray(j.data, np.float64)
        nr = np.ascontiguousarray(neg_res.numpy(), np.float64)
        b = rhs.numpy()                       # a view: the mass and energy entries are written into rhs
        assert a.indptr.dtype == np.int32 and a.indices.dtype == np.int32 and b.flags.c_contiguous
        m = L.emu_tpsa_thm_balance_rows(C.c_int(self._thm[0]), C.c_int64(self.nc), _p(a.indptr, C.c_int32),
                                        _p(a.indices, C.c_int32), _p(jp, C.c_int32), _p(jx, C.c_int32),
                                        _p(ja, C.c_double), _p(nr, C.c_double), _p(a.data, C.c_double),
                                        _p(b, C.c_double))
        if missing is not None:
            missing += m
