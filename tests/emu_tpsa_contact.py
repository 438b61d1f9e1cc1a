"""ctypes binding of tests/emu/_emu_tpsa_contact.so -- the host build of the TPSA contact system
(porepy_b200/csrc/tpsa_system.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_tpsa_contact.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from emu_binding import _p
from emu_tpsa_system import EmuTpsaSystemFaceGrid

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_tpsa_contact.cpp")
LIB = os.path.join(HERE, "emu", "_emu_tpsa_contact.so")
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
        _lib.emu_tpsa_contact_system.restype = C.c_int
        _lib.emu_tpsa_contact_rows.restype = C.c_int
        _lib.emu_tpsa_contact_get.restype = None
    return _lib


class EmuTpsaContactFaceGrid(EmuTpsaSystemFaceGrid):
    """``EmuTpsaSystemFaceGrid`` plus ``FaceGrid.tpsa_contact_system`` / ``tpsa_contact_rhs`` / ``tpsa_contact_rows`` on
    the host build, for the scipy stand-in of the device algebra (tests/emu_sparse.py): the matrix is a ``HostCsr``
    whose values the contact rows overwrite in place, vectors are CPU tensors."""

    def tpsa_contact_system(self, nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas, mortars,
                            frames, characteristic_traction):
        self._ctc = (nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas, mortars, frames,
                     float(characteristic_traction))
        A, _ = self._run_contact(np.zeros(nd * self.nf))
        from emu_sparse import HostCsr
        H = HostCsr(A)
        H.m = A                              # keep the pattern exactly as built (explicit zeros included)
        return H, [0.0, 0.0]

    def _run_contact(self, g, f=None, sr=None, sp=None):
        L = lib()
        nd, mu, lmbda, vol, codes, robin_diag, face_flags, face_areas, mortars, frames, ct = self._ctc
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)  # noqa: E731
        mu, lam, vol, rob, area, g, f, sr, sp, fr = (f64(a) for a in (mu, lmbda, vol, robin_diag, face_areas, g, f, sr,
                                                                      sp, frames))
        face, cell = (np.ascontiguousarray(mortars[k], np.int32) for k in ("face", "cell"))
        w = np.concatenate([f64(mortars[k]) for k in ("m2p", "p2m", "sign", "volume")] + [np.zeros(1)])
        nm, nk = face.size, fr.size // (nd * nd)
        cod = np.ascontiguousarray(codes, np.uint8)
        flags = np.ascontiguousarray(face_flags, np.uint8)
        h, nrows, nnz = C.c_void_p(), C.c_int64(), C.c_int64()
        rc = L.emu_tpsa_contact_system(*self._cf(), _p(self.geo[0], C.c_double), _p(self.geo[1], C.c_double),
                                       _p(area, C.c_double), _p(self.geo[2], C.c_double), C.c_int(nd),
                                       _p(mu, C.c_double), _p(lam, C.c_double), _p(vol, C.c_double),
                                       _p(cod, C.c_uint8), _p(rob, C.c_double), _p(flags, C.c_uint8), C.c_int64(nm),
                                       C.c_int64(nk), _p(face, C.c_int32), _p(cell, C.c_int32), _p(w, C.c_double),
                                       _p(np.concatenate([fr, [0.0]]), C.c_double), C.c_double(ct),
                                       _p(g, C.c_double), _p(f, C.c_double), _p(sr, C.c_double), _p(sp, C.c_double),
                                       C.byref(h), C.byref(nrows), C.byref(nnz))
        if rc:
            raise ValueError({1: "face with more than two neighbouring cells", 2: "too many face neighbours"}.get(
                rc, "a face with more than one mortar cell, or a fracture cell without two mortar cells"))
        n, z = nrows.value, nnz.value
        ip, ix, a, b = np.zeros(n + 1, np.int32), np.zeros(max(z, 1), np.int32), np.zeros(max(z, 1)), np.zeros(n)
        L.emu_tpsa_contact_get(h, _p(ip, C.c_int32), _p(ix, C.c_int32), _p(a, C.c_double), _p(b, C.c_double))
        return sps.csr_matrix((a[:z], ix[:z], ip), shape=(n, n)), b

    def tpsa_contact_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        import torch
        _, b = self._run_contact(bc_values, body_force, angular_source, mass_source)
        assert b.size == n
        return torch.as_tensor(b)

    def tpsa_contact_rows(self, A, jc, neg_res, rhs, missing=None):
        L = lib()
        nd = self._ctc[0]
        nm = np.asarray(self._ctc[8]["face"]).size
        a = A.m
        j = sps.csr_matrix(jc.to_scipy())
        nrows = j.shape[0]
        c0 = (nd + (3 if nd == 3 else 1) + 1) * self.nc          # B nc: B = nd + nr + 1
        row0 = c0 + nd * nm
        e0 = int(a.indptr[row0])
        jp, jx, ja = j.indptr.astype(np.int32), j.indices.astype(np.int32), np.ascontiguousarray(j.data, np.float64)
        nr = np.ascontiguousarray(neg_res.numpy(), np.float64)
        b = rhs.numpy()                       # a view: the contact entries are written into rhs
        assert a.indptr.dtype == np.int32 and a.indices.dtype == np.int32 and b.flags.c_contiguous
        m = L.emu_tpsa_contact_rows(C.c_int(nd), C.c_int64(nrows), C.c_int64(c0), C.c_int64(e0), C.c_int64(row0),
                                    _p(a.indices, C.c_int32), _p(jp, C.c_int32), _p(jx, C.c_int32),
                                    _p(ja, C.c_double), _p(nr, C.c_double), _p(a.data, C.c_double), _p(b, C.c_double))
        if missing is not None:
            missing += m
