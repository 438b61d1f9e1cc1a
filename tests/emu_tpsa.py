"""ctypes binding of tests/emu/_emu_tpsa.so -- the host build of the TPSA family (porepy_b200/csrc/tpsa_face.cuh and
tpsa_system.cuh).  TEST INFRASTRUCTURE ONLY (see tests/emu/emu_tpsa.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import scipy.sparse as sps

from emu_binding import EmuBackedFaceGrid, _p

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "emu_tpsa.cpp")
LIB = os.path.join(HERE, "emu", "_emu_tpsa.so")
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
        _lib.emu_tpsa_assemble.restype = C.c_int
        _lib.emu_tpsa_balance_rows.restype = C.c_int
        _lib.emu_tpsa_contact_rows.restype = C.c_int
        _lib.emu_tpsa_get.restype = None
    return _lib


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)


def _host_csr(A):
    from emu_sparse import HostCsr
    H = HostCsr(A)
    H.m = A                                  # keep the pattern exactly as built (explicit zeros included)
    return H


class EmuTpsaFaceGrid(EmuBackedFaceGrid):
    """``EmuBackedFaceGrid`` (TPFA, upwinding on the host build) plus every TPSA method of ``FaceGrid`` on the host
    build, with the same arguments: ``tpsa`` returns the value arrays (``fv.tpsa_value_counts``) and kernel time 0;
    ``tpsa_system`` / ``tpsa_rhs`` a scipy CSR and a NumPy array; the poromechanics, thermo-poromechanics and contact
    systems, for the scipy stand-in of the device algebra (tests/emu_sparse.py), a ``HostCsr`` whose values the row
    writers overwrite in place and CPU tensors.  Stage times are 0."""

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

    # ---- the systems: the arguments of the last ``*_system`` call of each kind, assembled again with b for ``*_rhs``

    def _run(self, kind, g, f=None, sr=None, sp=None):
        L = lib()
        nd, ns, mu, lmbda, alpha, vol, codes, robin_diag, face_flags, face_areas, fp, mortars, frames, ct = self._sys[kind]
        mu, lam, al, vol, rob, area, g, f, sr, sp = (_f64(a) for a in (mu, lmbda, alpha, vol, robin_diag, face_areas,
                                                                       g, f, sr, sp))
        cod = np.ascontiguousarray(codes, np.uint8)
        flags = np.ascontiguousarray(face_flags, np.uint8)
        fp_ip = fp_ix = face = cell = w = fr = None
        nm = nk = 0
        if fp is not None:
            fp = sps.csr_matrix(fp)
            fp.sort_indices()
            fp_ip, fp_ix = fp.indptr.astype(np.int32), fp.indices.astype(np.int32)
        if mortars is not None:
            face, cell = (np.ascontiguousarray(mortars[k], np.int32) for k in ("face", "cell"))
            w = np.concatenate([_f64(mortars[k]) for k in ("m2p", "p2m", "sign", "volume")] + [np.zeros(1)])
            fr = _f64(frames)
            nm, nk = face.size, fr.size // (nd * nd)
            fr = np.concatenate([fr, [0.0]])
        h, nrows, nnz = C.c_void_p(), C.c_int64(), C.c_int64()
        rc = L.emu_tpsa_assemble(C.c_int(mortars is not None), C.c_int(ns), *self._cf(), _p(self.geo[0], C.c_double),
                                 _p(self.geo[1], C.c_double), _p(area, C.c_double), _p(self.geo[2], C.c_double),
                                 C.c_int(nd), _p(mu, C.c_double), _p(lam, C.c_double), _p(al, C.c_double),
                                 _p(vol, C.c_double), _p(cod, C.c_uint8), _p(rob, C.c_double), _p(flags, C.c_uint8),
                                 _p(fp_ip, C.c_int32), _p(fp_ix, C.c_int32), C.c_int64(nm), C.c_int64(nk),
                                 _p(face, C.c_int32), _p(cell, C.c_int32), _p(w, C.c_double), _p(fr, C.c_double),
                                 C.c_double(ct), _p(g, C.c_double), _p(f, C.c_double), _p(sr, C.c_double),
                                 _p(sp, C.c_double), C.byref(h), C.byref(nrows), C.byref(nnz))
        if rc:
            raise ValueError({1: "face with more than two neighbouring cells", 2: "too many face neighbours"}.get(
                rc, "a face with more than one mortar cell, or a fracture cell without two mortar cells"))
        n, z = nrows.value, nnz.value
        ip, ix, a, b = np.zeros(n + 1, np.int32), np.zeros(max(z, 1), np.int32), np.zeros(max(z, 1)), np.zeros(n)
        L.emu_tpsa_get(h, _p(ip, C.c_int32), _p(ix, C.c_int32), _p(a, C.c_double), _p(b, C.c_double))
        return sps.csr_matrix((a[:z], ix[:z], ip), shape=(n, n)), b

    def _system(self, kind, nd, ns, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                fp=None, mortars=None, frames=None, ct=0.0):
        if not hasattr(self, "_sys"):
            self._sys = {}
        self._sys[kind] = (nd, ns, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas, fp,
                           mortars, frames, float(ct))
        A, _ = self._run(kind, np.zeros(nd * self.nf))
        return A

    def _rhs(self, kind, n, bc_values, body_force, angular_source, mass_source):
        _, b = self._run(kind, bc_values, body_force, angular_source, mass_source)
        assert b.size == n
        return b

    def tpsa_system(self, nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas):
        A = self._system("sys", nd, 0, mu, lmbda, None, cell_volumes, codes, robin_diag, face_flags, face_areas)
        return A, [0.0, 0.0]

    def tpsa_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        return self._rhs("sys", n, bc_values, body_force, angular_source, mass_source)

    def tpsa_poro_system(self, nd, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                         flux_pattern):
        return _host_csr(self._system("poro", nd, 1, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags,
                                      face_areas, flux_pattern.to_scipy())), [0.0, 0.0]

    def tpsa_thm_system(self, nd, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                        flux_pattern):
        return _host_csr(self._system("thm", nd, 2, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags,
                                      face_areas, flux_pattern.to_scipy())), [0.0, 0.0]

    def tpsa_contact_system(self, nd, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas, mortars,
                            frames, characteristic_traction):
        return _host_csr(self._system("contact", nd, 0, mu, lmbda, None, cell_volumes, codes, robin_diag, face_flags,
                                      face_areas, None, mortars, frames, characteristic_traction)), [0.0, 0.0]

    def tpsa_poro_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        import torch
        return torch.as_tensor(self._rhs("poro", n, bc_values, body_force, angular_source, mass_source))

    def tpsa_thm_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        import torch
        return torch.as_tensor(self._rhs("thm", n, bc_values, body_force, angular_source, mass_source))

    def tpsa_contact_rhs(self, n, bc_values, body_force=None, angular_source=None, mass_source=None):
        import torch
        return torch.as_tensor(self._rhs("contact", n, bc_values, body_force, angular_source, mass_source))

    # ---- the row writers: in place on the matrix values and on rhs (a view), as the device writes them

    @staticmethod
    def _jacobian(jac, neg_res, rhs, a):
        j = sps.csr_matrix(jac.to_scipy())
        jp, jx, ja = j.indptr.astype(np.int32), j.indices.astype(np.int32), np.ascontiguousarray(j.data, np.float64)
        nr = np.ascontiguousarray(neg_res.numpy(), np.float64)
        b = rhs.numpy()
        assert a.indptr.dtype == np.int32 and a.indices.dtype == np.int32 and b.flags.c_contiguous
        return j.shape, (_p(jp, C.c_int32), _p(jx, C.c_int32), _p(ja, C.c_double), _p(nr, C.c_double),
                         _p(a.data, C.c_double), _p(b, C.c_double)), (jp, jx, ja, nr)

    def _balance_rows(self, kind, A, jf, neg_res, rhs, missing):
        nd, ns = self._sys[kind][:2]
        a = A.m
        shape, ptrs, _keep = self._jacobian(jf, neg_res, rhs, a)
        assert shape == (ns * self.nc, (1 + ns) * self.nc)
        m = lib().emu_tpsa_balance_rows(C.c_int(nd), C.c_int(ns), C.c_int64(self.nc), _p(a.indptr, C.c_int32),
                                        _p(a.indices, C.c_int32), *ptrs)
        if missing is not None:
            missing += m

    def tpsa_poro_fluid_rows(self, A, jf, neg_res, rhs, missing=None):
        self._balance_rows("poro", A, jf, neg_res, rhs, missing)

    def tpsa_thm_balance_rows(self, A, jf, neg_res, rhs, missing=None):
        self._balance_rows("thm", A, jf, neg_res, rhs, missing)

    def tpsa_contact_rows(self, A, jc, neg_res, rhs, missing=None):
        nd = self._sys["contact"][0]
        nm = np.asarray(self._sys["contact"][11]["face"]).size
        a = A.m
        shape, ptrs, _keep = self._jacobian(jc, neg_res, rhs, a)
        c0 = (nd + (3 if nd == 3 else 1) + 1) * self.nc          # B nc: B = nd + nr + 1
        row0 = c0 + nd * nm
        m = lib().emu_tpsa_contact_rows(C.c_int(nd), C.c_int64(shape[0]), C.c_int64(c0), C.c_int64(int(a.indptr[row0])),
                                        C.c_int64(row0), _p(a.indices, C.c_int32), *ptrs)
        if missing is not None:
            missing += m
