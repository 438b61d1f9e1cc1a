"""Finite-volume discretizations behind PorePy's ``Discretization`` operator API, executed
by the sm_90a kernels of libporeb200.so.

Mirrors (same constructor, attribute names, matrix-dictionary keys, parameter keys and
exceptions) of

* ``pp.Mpfa``   reference src/porepy/numerics/fv/mpfa.py:29  (``discretize`` :65) with the
  ``FVElliptic`` base (numerics/fv/fv_elliptic.py:16, ``assemble_matrix_rhs`` :67-112),
* ``pp.Mpsa``   reference src/porepy/numerics/fv/mpsa.py:38  (``discretize`` :121,
  ``assemble_matrix_rhs`` :486-529),
* ``pp.Biot``   reference src/porepy/numerics/fv/biot.py:40  (``discretize`` :247).

Inputs come from ``data["parameters"][keyword]``, outputs (scipy CSR) go to
``data["discretization_matrices"][keyword][<key>]`` exactly as in the reference, so the classes
drop into ``EquationSystem.discretize`` / the model mixins (see porepy_b200/porepy_plugin.py
for the ``pp.ad.MpfaAd`` subclasses used when the reference is importable).

There is no CPU path: without the built CUDA library or without a GPU every ``discretize``
raises ``RuntimeError``.
"""
from __future__ import annotations

import ctypes as C
import logging
import time

import numpy as np
import scipy.sparse as sps

from . import _lib
from .params import DISCRETIZATION_MATRICES, PARAMETERS

logger = logging.getLogger(__name__)


def determine_eta(sd) -> float:
    """numerics/fv/_fvutils.py:280-305: 1/3 on simplex grids, 0 otherwise."""
    name = getattr(sd, "name", "")
    if not isinstance(name, str):
        name = " ".join(str(n) for n in name)
    return 1.0 / 3.0 if ("TriangleGrid" in name or "TetrahedralGrid" in name) else 0.0


def block_expand(ip: np.ndarray, ix: np.ndarray, br: int, bc: int):
    """Expand a base pattern into br x bc blocks (row r*br+i, column c*bc+j).  The value of
    block entry (i, j) of base entry p in base row r is stored at
    ``br*bc*ip[r] + i*bc*len_r + (p-ip[r])*bc + j`` -- the layout the kernels scatter into."""
    ip = ip.astype(np.int64)
    lens = np.diff(ip)
    new_ip = np.zeros(lens.size * br + 1, dtype=np.int64)
    np.cumsum(np.repeat(lens * bc, br), out=new_ip[1:])
    cols = ix.astype(np.int64)
    if bc > 1:
        cols = (cols[:, None] * bc + np.arange(bc, dtype=np.int64)).reshape(-1)
    if br == 1:
        return new_ip, cols
    out = np.empty(new_ip[-1], dtype=np.int64)
    rep = lens * bc
    row_of = np.repeat(np.arange(lens.size, dtype=np.int64), rep)
    off = np.arange(cols.size, dtype=np.int64) - np.repeat(ip[:-1] * bc, rep)
    for i in range(br):
        out[new_ip[row_of * br + i] + off] = cols
    return new_ip, out


def _index_dtype(nnz: int, ncols: int):
    return np.int32 if max(nnz, ncols) < 2**31 - 1 else np.int64


# ------------------------------------------------------------------------------------------
# 2-D grids embedded in 3-D (fracture planes)
# ------------------------------------------------------------------------------------------


def plane_frame(sd, tol: float = 1e-5):
    """Rotation ``R`` (3, 3) with rows (t1, t2, n) that maps a planar 2-D grid into its own
    plane, or ``None`` when the grid already lies in a plane z = const.

    The reference rotates such grids with ``map_geometry.map_grid`` before discretizing
    (numerics/fv/mpfa.py:733-754).  Any in-plane basis gives the same matrices (the scheme is
    invariant under rotations and reflections), so the frame is taken from the principal axes
    of the node cloud."""
    x = np.asarray(sd.nodes, dtype=np.float64)
    xc = x - x.mean(axis=1, keepdims=True)
    w, v = np.linalg.eigh(xc @ xc.T)          # ascending: v[:, 0] is the plane normal
    n = v[:, 0]
    extent = np.sqrt(max(w[2], 0.0) / max(x.shape[1], 1)) + 1e-300
    if np.abs(n @ xc).max() > tol * max(extent, np.abs(xc).max()):
        raise ValueError("2-D grid is not planar")
    if abs(abs(n[2]) - 1.0) <= 1e-14 and np.ptp(x[2]) <= 1e-12 * max(1.0, np.abs(x).max()):
        return None
    t1 = v[:, 2]
    t2 = np.cross(n, t1)
    return np.vstack((t1, t2 / np.linalg.norm(t2), n))


def plan_geometry(sd):
    """The six geometry arrays the plan reads, and the rotation applied to them (None for 3-D
    grids and for 2-D grids in a plane z = const)."""
    arrs = [sd.nodes, sd.face_normals, sd.face_centers, sd.face_areas, sd.cell_centers, sd.cell_volumes]
    rot = plane_frame(sd) if int(sd.dim) == 2 else None
    if rot is not None:
        for i in (0, 1, 2, 4):
            a = rot @ np.asarray(arrs[i], dtype=np.float64)
            a[2] = 0.0
            arrs[i] = a
    return [_lib.f64(a) for a in arrs], rot


def rotate_second_order(values: np.ndarray, rot: np.ndarray) -> np.ndarray:
    """R K R^T per cell for (3, 3, nc) values (mpfa.py:749-754; the kernels read the leading
    nd x nd block)."""
    return np.einsum("ia,abc,jb->ijc", rot, np.asarray(values, dtype=np.float64), rot)


def lift_vector_source(ip: np.ndarray, ix: np.ndarray, data: np.ndarray, rows: np.ndarray, nc: int):
    """(nf, 2 nc) vector-source matrix in the plane's coordinates -> (nf, amb nc) in the ambient space
    (amb = ``rows.shape[1]``, 2 or 3): every (face, cell) pair of in-plane coefficients is multiplied by the
    two in-plane rows of the rotation, restricted to the first ``amb`` ambient components (mpfa.py:423-466).
    ``ip, ix`` is the FACE x CELL base pattern, ``data`` holds the two coefficients of each base entry
    consecutively."""
    rows = np.asarray(rows, dtype=np.float64)
    amb = rows.shape[1]
    da = np.asarray(data, dtype=np.float64).reshape(-1, 2) @ rows
    dt = _index_dtype(amb * int(ix.size), amb * nc)
    cols = (ix.astype(dt)[:, None] * amb + np.arange(amb, dtype=dt)).ravel()
    return sps.csr_matrix((da.ravel(), cols, ip.astype(dt) * amb), shape=(ip.size - 1, amb * nc))


def _log_throughput(name: str, keyword: str, sd, kernel_ms: float, wall_s: float, out: dict) -> None:
    """One INFO line per discretization (the reference logs the elapsed time of ``discretize``,
    models/solution_strategy.py:435-441): cells/s of the kernels and of the whole call, and the rate at which the
    output values were written."""
    if not logger.isEnabledFor(logging.INFO):
        return
    nbytes = 0
    for m in out.values():
        for mm in (m.values() if isinstance(m, dict) else (m,)):
            nbytes += 8 * int(getattr(mm, "nnz", 0))
    k_s = max(kernel_ms, 1e-6) * 1e-3
    logger.info("porepy_b200 %s(%s): %d cells (dim %d), kernels %.2f ms = %.3g cells/s, %.1f GB/s of output values; "
                "discretize() %.3f s = %.3g cells/s", name, keyword, sd.num_cells, sd.dim, kernel_ms,
                sd.num_cells / k_s, nbytes / k_s / 1e9, wall_s, sd.num_cells / max(wall_s, 1e-9))


def _on_device(*mats) -> bool:
    """All given matrices are ``LazyCsr`` whose values still live only on the device (untouched by the host)."""
    from .sparse import LazyCsr
    return all(isinstance(m, LazyCsr) and m.device_values is not None and not m.on_host for m in mats)


def _lazy_system(a_dev):
    """scipy-compatible view of a device-assembled system matrix; downloaded on first touch."""
    from .sparse import LazyCsr
    cache = {}

    def host():
        if "m" not in cache:
            cache["m"] = a_dev.to_scipy()
        return cache["m"]
    return LazyCsr.lazy(a_dev.shape, a_dev.nnz, lambda: host().data, lambda: host().indices, lambda: host().indptr,
                        device_csr=a_dev)


def _lifted(plan, m, rows: np.ndarray, nc: int):
    """``lift_vector_source`` of the (possibly still device-resident) in-plane matrix ``m``, itself lazy: the
    lifting runs on the host when the lifted matrix is first touched.  Keeps the in-plane device values and the
    rotation rows for ``assemble_matrix_rhs`` (which rotates the vector instead of the matrix)."""
    from .sparse import LazyCsr
    amb = rows.shape[1]
    cache = {}

    def built():
        if "m" not in cache:
            ip, ix = plan.base_pattern(0)
            cache["m"] = lift_vector_source(ip, ix, m.data, rows, nc)
        return cache["m"]
    out = LazyCsr.lazy((m.shape[0], amb * nc), (m.nnz // 2) * amb, lambda: built().data, lambda: built().indices,
                       lambda: built().indptr, device_values=getattr(m, "device_values", None), plan=plan)
    out.__dict__["plane_rows"] = rows
    return out


class DevicePlan:
    """Device-resident sub-cell topology + output patterns of one grid (``pb_plan``).

    Built once per grid topology and cached on the grid object; MPFA, MPSA and Biot share it.
    """

    def __init__(self, sd):
        lib = _lib.load()
        _lib.require_gpu()
        self.lib = lib
        if hasattr(sd, "periodic_face_map"):
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        if sd.dim not in (2, 3):
            raise NotImplementedError(
                f"porepy_b200 discretizes 2-D and 3-D grids; dim={sd.dim} (TPFA fallback of "
                "mpfa.py:690-712) is not part of this build")
        cf = sps.csc_matrix(sd.cell_faces)
        fn = sps.csc_matrix(sd.face_nodes)
        self.nd, self.nc, self.nf, self.nn = int(sd.dim), sd.num_cells, sd.num_faces, sd.num_nodes
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731  (no copy when scipy already holds int32)
        cfp, cfi = i32(cf.indptr), i32(cf.indices)
        cfd = np.asarray(cf.data).astype(np.int8)
        fnp, fni = i32(fn.indptr), i32(fn.indices)
        h = C.c_void_p()
        t0 = time.perf_counter()
        _lib.check(lib.pb_plan_create(self.nd, self.nc, self.nf, self.nn,
                                      _lib.ptr(cfp, _lib._i32p), _lib.ptr(cfi, _lib._i32p),
                                      _lib.ptr(cfd, _lib._i8p), _lib.ptr(fnp, _lib._i32p),
                                      _lib.ptr(fni, _lib._i32p), C.byref(h)))
        self.plan_seconds = time.perf_counter() - t0
        self.h = h
        self.fingerprint = self._fingerprint(sd, cf, fn)
        self._base = {}
        self._expanded = {}
        self.rotation = None

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            try:
                self.lib.pb_plan_destroy(h)
            except Exception:
                pass
            self.h = None

    @staticmethod
    def _fingerprint(sd, cf, fn):
        """Counts plus a strided checksum of the index arrays: a topology edit that keeps the counts (split faces
        renumbered, ...) must not reuse a stale plan."""
        ci, fi = np.asarray(cf.indices), np.asarray(fn.indices)
        return (int(sd.dim), sd.num_cells, sd.num_faces, sd.num_nodes, int(cf.nnz), int(fn.nnz),
                int(ci[::7].astype(np.int64).sum()), int(fi[::7].astype(np.int64).sum()),
                int(np.asarray(cf.indptr)[::5].astype(np.int64).sum()))

    @classmethod
    def for_grid(cls, sd) -> "DevicePlan":
        cf, fn = sd.cell_faces, sd.face_nodes
        fp = cls._fingerprint(sd, cf, fn)
        plan = getattr(sd, "_b200_plan", None)
        if plan is None or plan.fingerprint != fp:
            plan = cls(sd)
            try:
                sd._b200_plan = plan
            except AttributeError:
                pass
        plan.set_geometry(sd)
        return plan

    def set_geometry(self, sd) -> None:
        """Upload the geometry.  2-D grids embedded in 3-D are rotated into their own plane first
        (``plan_geometry``); ``self.rotation`` keeps the rotation for the callers."""
        arrs, self.rotation = plan_geometry(sd)
        _lib.check(self.lib.pb_plan_set_geometry(self.h, *[_lib.ptr(a, _lib._f64p) for a in arrs]))

    def set_cell_map(self, cells, n_source_cells: int) -> None:
        """Cell ``e`` of this plan is cell ``cells[e]`` of a larger grid with ``n_source_cells`` cells: the cell
        tensors of the following uploads may then be the arrays of THAT grid (shape (3, 3, n_source) / (9, 9,
        n_source)); they are restricted on the device.  A shard passes the global tensors as they are."""
        if cells is None:
            _lib.check(self.lib.pb_plan_set_cell_map(self.h, None, 0))
            self.n_source_cells = None
            return
        m = np.ascontiguousarray(cells, dtype=np.int64)
        if m.shape != (self.nc,):
            raise ValueError("cell map must have one entry per cell of this plan")
        _lib.check(self.lib.pb_plan_set_cell_map(self.h, _lib.ptr(m, _lib._i64p), int(n_source_cells)))
        self.n_source_cells = int(n_source_cells)
        self._cell_map_host = m

    def _cells_of(self, arr) -> bool:
        """True when a cell tensor has the source grid's size and must go through the cell map (clears the map when
        the caller passes arrays of this plan's own size instead)."""
        n = arr.shape[-1]
        src = getattr(self, "n_source_cells", None)
        if src is not None and n == src and n != self.nc:
            return True
        if src is not None and n == self.nc:
            self.set_cell_map(None, 0)
        return False

    def set_active_nodes(self, mask) -> None:
        """Assemble only the interaction regions of the flagged nodes (``None``: all).  The multi-GPU path flags
        a shard's own nodes: the outer nodes of its halo layer are incomplete and their rows are discarded."""
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        if m is not None and m.shape != (self.nn,):
            raise ValueError("active-node mask must have one entry per node")
        _lib.check(self.lib.pb_plan_set_active_nodes(self.h, _lib.ptr(m, _lib._u8p)))

    # ---- patterns
    def base_pattern(self, which: int):
        if which not in self._base:
            nr, nz = C.c_int64(), C.c_int64()
            _lib.check(self.lib.pb_plan_pattern_size(self.h, which, C.byref(nr), C.byref(nz)))
            ip = np.zeros(nr.value + 1, np.int32)
            ix = np.zeros(max(nz.value, 1), np.int32)
            _lib.check(self.lib.pb_plan_pattern_get(self.h, which, _lib.ptr(ip, _lib._i32p),
                                                    _lib.ptr(ix, _lib._i32p)))
            ix = ix[:nz.value]
            ip.flags.writeable = ix.flags.writeable = False   # shared by every matrix on this grid
            self._base[which] = (ip, ix)
        return self._base[which]

    def nnz(self, which: int) -> int:
        return int(self.base_pattern(which)[1].size)

    def pattern(self, which: int, br: int, bc: int):
        key = (which, br, bc)
        if key not in self._expanded:
            ip, ix = self.base_pattern(which)
            if br == 1 and bc == 1:
                self._expanded[key] = (ip, ix)
            else:
                ncols = {0: self.nc, 1: self.nf, 2: self.nc, 3: self.nf}[which] * bc
                nnz = int(ix.size) * br * bc
                if max(nnz, ncols) < 2**31 - 1:
                    # expansion on the device, D2H into page-locked buffers
                    nip = _lib.pinned_empty((ip.size - 1) * br + 1, np.int32)
                    nix = _lib.pinned_empty(max(nnz, 1), np.int32)
                    _lib.check(self.lib.pb_plan_pattern_expanded(
                        self.h, which, br, bc, _lib.ptr(nip, _lib._i32p), _lib.ptr(nix, _lib._i32p)))
                    nix = nix[:nnz]
                else:  # beyond int32: host expansion with 64-bit indices
                    nip, nix = block_expand(ip, ix, br, bc)
                nip.flags.writeable = nix.flags.writeable = False
                self._expanded[key] = (nip, nix)
        return self._expanded[key]

    def matrix(self, which: int, br: int, bc: int, data: np.ndarray) -> sps.csr_matrix:
        ip, ix = self.pattern(which, br, bc)
        nrows = (ip.size - 1)
        ncols = {0: self.nc, 1: self.nf, 2: self.nc, 3: self.nf}[which] * bc
        m = sps.csr_matrix((data, ix, ip), shape=(nrows, ncols), copy=False)
        m.has_sorted_indices = True
        return m

    def sizes(self) -> dict:
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        d, e = C.c_int32(), C.c_int32()
        _lib.check(self.lib.pb_plan_sizes(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d),
                                          C.byref(e)))
        return dict(subcells=a.value, subfaces=b.value, subhalffaces=c.value,
                    max_subfaces_per_node=d.value, max_subcells_per_node=e.value)

    def class_counts(self, kind: str) -> dict:
        """Nodes per local-solver class of the classes last built for ``kind`` ("mpfa" or "mpsa"):
        {(cfg, a_in_global_memory): count} over the non-empty classes (solver configurations: csrc/plan.hpp)."""
        counts = np.zeros(14, np.int64)
        _lib.check(self.lib.pb_plan_class_counts(self.h, {"mpfa": 0, "mpsa": 1}[kind], _lib.ptr(counts, _lib._i64p)))
        return {(k // 2, bool(k & 1)): int(v) for k, v in enumerate(counts) if v}

    # ---- MPFA
    def mpfa_upload(self, perm, codes, robw, eta) -> None:
        perm = _lib.f64(perm)
        if not self._cells_of(perm) and perm.shape != (3, 3, self.nc):
            raise ValueError("second_order_tensor.values must have shape (3, 3, num_cells)")
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        robw = None if robw is None else _lib.f64(robw)
        _lib.check(self.lib.pb_mpfa_upload(self.h, _lib.ptr(perm, _lib._f64p),
                                           _lib.ptr(codes, _lib._u8p), _lib.ptr(robw, _lib._f64p),
                                           float(eta)))

    def mpfa_assemble(self, flux=True, trace=True, vector_source=True) -> float:
        ms = C.c_float()
        _lib.check(self.lib.pb_mpfa_assemble(self.h, int(flux), int(trace), int(vector_source),
                                             C.byref(ms)))
        return float(ms.value)

    def mpfa_download(self, flux=True, trace=True, vector_source=True) -> dict:
        nd = self.nd
        nfc, nfb = self.nnz(0), self.nnz(1)
        bufs = {
            "flux": _lib.pinned_empty(nfc) if flux else None,
            "bound_flux": _lib.pinned_empty(nfb) if flux else None,
            "bound_pressure_cell": _lib.pinned_empty(nfc) if trace else None,
            "bound_pressure_face": _lib.pinned_empty(nfb) if trace else None,
            "vector_source": _lib.pinned_empty(nfc * nd) if (flux and vector_source) else None,
            "bound_pressure_vector_source": _lib.pinned_empty(nfc * nd) if (trace and vector_source) else None,
        }
        _lib.check(self.lib.pb_mpfa_download(self.h, *[_lib.ptr(b, _lib._f64p) for b in bufs.values()]))
        shape = {"flux": (0, 1, 1), "bound_flux": (1, 1, 1), "bound_pressure_cell": (0, 1, 1),
                 "bound_pressure_face": (1, 1, 1), "vector_source": (0, 1, nd),
                 "bound_pressure_vector_source": (0, 1, nd)}
        return {k: self.matrix(*shape[k], v) for k, v in bufs.items() if v is not None}

    # ---- device-resident results (lazily downloaded scipy matrices)
    def _ncols(self, which: int, bc: int) -> int:
        return {0: self.nc, 1: self.nf, 2: self.nc, 3: self.nf}[which] * bc

    def take(self, key: int):
        """Move the value array of output ``key`` (``PB_OUT_*``) out of the plan; it stays in HBM."""
        from .sparse import DeviceValues
        h = C.c_void_p()
        _lib.check(self.lib.pb_plan_take_output(self.h, int(key), C.byref(h)))
        return DeviceValues(h, self.lib)

    def lazy_matrix(self, key: int, which: int, br: int, bc: int):
        """Output ``key`` as a ``LazyCsr`` on pattern ``which`` expanded to br x bc blocks: values, indices and
        row pointers are downloaded when (and if) a caller touches them."""
        from .sparse import LazyCsr
        vals = self.take(key)
        nrows = {0: self.nf, 1: self.nf, 2: self.nc, 3: self.nc}[which] * br
        pat_nnz = {w: None for w in range(4)}
        nr, nz = C.c_int64(), C.c_int64()
        _lib.check(self.lib.pb_plan_pattern_size(self.h, which, C.byref(nr), C.byref(nz)))
        del pat_nnz
        m = LazyCsr.lazy((nrows, self._ncols(which, bc)), nz.value * br * bc, vals.download,
                         lambda: self.pattern(which, br, bc)[1], lambda: self.pattern(which, br, bc)[0],
                         device_values=vals, plan=self)
        m.__dict__["pattern_key"] = (which, br, bc)
        return m

    def output_csr(self, values, which: int, br: int, bc: int):
        """A detached output as a ``DeviceCsr`` (block-expanded pattern + a copy of the values), the operand form of
        the device-side AD chain (``porepy_b200.ad``)."""
        from .sparse import DeviceCsr
        h = C.c_void_p()
        _lib.check(self.lib.pb_plan_output_csr(self.h, values.h, which, br, bc, C.byref(h)))
        return DeviceCsr.from_handle(h)

    def mpfa_lazy(self, flux=True, trace=True, vector_source=True) -> dict:
        nd = self.nd
        spec = {"flux": (0, 0, 1, flux), "bound_flux": (1, 1, 1, flux), "bound_pressure_cell": (2, 0, 1, trace),
                "bound_pressure_face": (3, 1, 1, trace), "vector_source": (4, 0, nd, flux and vector_source),
                "bound_pressure_vector_source": (5, 0, nd, trace and vector_source)}
        return {k: self.lazy_matrix(key, which, 1, bc) for k, (key, which, bc, want) in spec.items() if want}

    def mpsa_lazy(self) -> dict:
        nd = self.nd
        return {"stress": self.lazy_matrix(6, 0, nd, nd), "bound_stress": self.lazy_matrix(7, 1, nd, nd),
                "bound_displacement_cell": self.lazy_matrix(8, 0, nd, nd),
                "bound_displacement_face": self.lazy_matrix(9, 1, nd, nd)}

    def biot_lazy(self, q: int) -> dict:
        nd, b = self.nd, 10 + 5 * q
        return {"displacement_divergence": self.lazy_matrix(b, 2, 1, nd),
                "boundary_displacement_divergence": self.lazy_matrix(b + 1, 3, 1, nd),
                "scalar_gradient": self.lazy_matrix(b + 2, 0, nd, 1),
                "mpsa_consistency": self.lazy_matrix(b + 3, 2, 1, 1),
                "bound_displacement_pressure": self.lazy_matrix(b + 4, 0, nd, 1)}

    @staticmethod
    def _vh(values):
        return None if values is None else values.h

    def mpfa_system(self, flux=None):
        """A = div @ flux assembled and kept on the device (``DeviceCsr``) from the flux values given as a
        ``DeviceValues`` handle (``None``: the plan's last assembled array)."""
        from .sparse import DeviceCsr
        h = C.c_void_p()
        _lib.check(self.lib.pb_mpfa_system(self.h, self._vh(flux), C.byref(h)))
        return DeviceCsr.from_handle(h)

    def mpfa_rhs(self, bc_values, vector_source=None, bound_flux=None, vector_source_discr=None) -> np.ndarray:
        """b = -div @ (bound_flux @ bc_values) [- div @ (vector_source_discr @ vector_source)]."""
        bv = _lib.f64(bc_values)
        vs = None if vector_source is None else _lib.f64(vector_source)
        rhs = np.empty(self.nc)
        _lib.check(self.lib.pb_mpfa_rhs(self.h, self._vh(bound_flux), self._vh(vector_source_discr),
                                        _lib.ptr(bv, _lib._f64p), _lib.ptr(vs, _lib._f64p),
                                        _lib.ptr(rhs, _lib._f64p)))
        return rhs

    def mpsa_system(self, stress=None):
        """A = div_nd @ stress assembled and kept on the device (``DeviceCsr``)."""
        from .sparse import DeviceCsr
        h = C.c_void_p()
        _lib.check(self.lib.pb_mpsa_system(self.h, self._vh(stress), C.byref(h)))
        return DeviceCsr.from_handle(h)

    def mpsa_rhs(self, bc_values, source=None, bound_stress=None) -> np.ndarray:
        """b = -div_nd @ (bound_stress @ bc_values) + source   (mpsa.py:486-529)."""
        bv = _lib.f64(bc_values)
        src = None if source is None else _lib.f64(source)
        rhs = np.empty(self.nc * self.nd)
        _lib.check(self.lib.pb_mpsa_rhs(self.h, self._vh(bound_stress), _lib.ptr(bv, _lib._f64p),
                                        _lib.ptr(src, _lib._f64p), _lib.ptr(rhs, _lib._f64p)))
        return rhs

    # ---- MPSA / Biot
    def mpsa_upload(self, stiff, codes, robw, eta, alphas=()) -> None:
        stiff = _lib.f64(stiff)
        mapped = self._cells_of(stiff)
        if not mapped and stiff.shape != (9, 9, self.nc):
            raise ValueError("fourth_order_tensor.values must have shape (9, 9, num_cells)")
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        robw = None if robw is None else _lib.f64(robw)
        nal = len(alphas)
        al = None
        if nal:
            al = np.zeros((nal, 3, 3, self.n_source_cells if mapped else self.nc))
            for q, a in enumerate(alphas):
                a = np.asarray(a)
                if mapped and a.shape[-1] == self.nc:      # a tensor given for this plan's own cells
                    al[q][..., self._cell_map_host] = a
                else:
                    al[q] = a
        _lib.check(self.lib.pb_mpsa_upload(self.h, _lib.ptr(stiff, _lib._f64p),
                                           _lib.ptr(codes, _lib._u8p), _lib.ptr(robw, _lib._f64p),
                                           float(eta), nal, _lib.ptr(al, _lib._f64p)))
        self._nal = nal

    def mpsa_set_basis(self, basis) -> None:
        """``bc.basis`` (nd, nd, nf) or None for the identity; call after ``mpsa_upload``."""
        b = None if basis is None else _lib.f64(basis)
        if b is not None and b.shape != (self.nd, self.nd, self.nf):
            raise ValueError("bc.basis must have shape (nd, nd, num_faces)")
        _lib.check(self.lib.pb_mpsa_set_basis(self.h, _lib.ptr(b, _lib._f64p)))

    def mpsa_assemble(self) -> float:
        ms = C.c_float()
        _lib.check(self.lib.pb_mpsa_assemble(self.h, C.byref(ms)))
        return float(ms.value)

    def mpsa_download(self) -> dict:
        nd = self.nd
        nd2 = nd * nd
        nfc, nfb = self.nnz(0), self.nnz(1)
        bufs = [_lib.pinned_empty(nfc * nd2), _lib.pinned_empty(nfb * nd2), _lib.pinned_empty(nfc * nd2),
                _lib.pinned_empty(nfb * nd2)]
        _lib.check(self.lib.pb_mpsa_download(self.h, *[_lib.ptr(b, _lib._f64p) for b in bufs]))
        return {
            "stress": self.matrix(0, nd, nd, bufs[0]),
            "bound_stress": self.matrix(1, nd, nd, bufs[1]),
            "bound_displacement_cell": self.matrix(0, nd, nd, bufs[2]),
            "bound_displacement_face": self.matrix(1, nd, nd, bufs[3]),
        }

    def biot_download(self, q: int) -> dict:
        nd = self.nd
        nfc, ncc, ncb = self.nnz(0), self.nnz(2), self.nnz(3)
        bufs = [_lib.pinned_empty(ncc * nd), _lib.pinned_empty(ncb * nd), _lib.pinned_empty(nfc * nd),
                _lib.pinned_empty(ncc), _lib.pinned_empty(nfc * nd)]
        _lib.check(self.lib.pb_biot_download(self.h, q, *[_lib.ptr(b, _lib._f64p) for b in bufs]))
        return {
            "displacement_divergence": self.matrix(2, 1, nd, bufs[0]),
            "boundary_displacement_divergence": self.matrix(3, 1, nd, bufs[1]),
            "scalar_gradient": self.matrix(0, nd, 1, bufs[2]),
            "mpsa_consistency": self.matrix(2, 1, 1, bufs[3]),
            "bound_displacement_pressure": self.matrix(0, nd, 1, bufs[4]),
        }


class FaceGrid:
    """Face-indexed device view of a grid of any dimension (``pb_facegrid``): the face -> cell table and
    the face normals / centres and cell centres -- all the per-face schemes (TPFA, upwinding) read.  No
    interaction-region plan is built, so 1-D grids (the reference's TPFA delegation, mpfa.py:690-712,
    mpsa.py:666-697) and 2-D grids anywhere in space work as they are."""

    def __init__(self, sd):
        lib = _lib.load()
        _lib.require_gpu()
        self.lib = lib
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic faces are not supported by porepy_b200")
        cf = sps.csc_matrix(sd.cell_faces)
        self.nc, self.nf = sd.num_cells, sd.num_faces
        cfp, cfi = cf.indptr.astype(np.int32), cf.indices.astype(np.int32)
        cfd = np.asarray(cf.data).astype(np.int8)
        geo = [_lib.f64(a) for a in (sd.face_normals, sd.face_centers, sd.cell_centers)]
        h = C.c_void_p()
        _lib.check(lib.pb_facegrid_create(self.nc, self.nf, _lib.ptr(cfp, _lib._i32p), _lib.ptr(cfi, _lib._i32p),
                                          _lib.ptr(cfd, _lib._i8p), *[_lib.ptr(a, _lib._f64p) for a in geo],
                                          C.byref(h)))
        self.h = h

    @classmethod
    def for_grid(cls, sd) -> "FaceGrid":
        return cls(sd)

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            try:
                self.lib.pb_facegrid_destroy(h)
            except Exception:
                pass
            self.h = None

    def tpfa(self, perm, bc_bits, fc_indptr, vdim: int) -> list:
        """Value arrays of the six TPFA terms in the pattern of ``cell_faces`` (CSR by face):
        [flux, bound_pressure_cell, vector_source, bound_pressure_vector_source] and the diagonals
        [bound_flux, bound_pressure_face]."""
        perm = _lib.f64(perm)
        if perm.shape != (3, 3, self.nc):
            raise ValueError("second_order_tensor.values must have shape (3, 3, num_cells)")
        bits = np.ascontiguousarray(bc_bits, dtype=np.uint8)
        ip = np.ascontiguousarray(fc_indptr, dtype=np.int32)
        nnz = int(ip[-1])
        out = [np.empty(nnz), np.empty(nnz), np.empty(nnz * vdim), np.empty(nnz * vdim), np.empty(self.nf),
               np.empty(self.nf)]
        _lib.check(self.lib.pb_tpfa(self.h, _lib.ptr(perm, _lib._f64p), _lib.ptr(bits, _lib._u8p),
                                    _lib.ptr(ip, _lib._i32p), int(vdim), *[_lib.ptr(a, _lib._f64p) for a in out]))
        return out

    def tpfa_diff(self, k_c, fc_indptr):
        """Differentiable TPFA (``pb_tpfa_diff``): half-face transmissibilities, face transmissibilities and
        dT_f/dk_c (9 values per half-face) for the cell-major 9 * nc permeability vector ``k_c``."""
        k = np.ascontiguousarray(k_c, dtype=np.float64).reshape(-1)
        ip = np.ascontiguousarray(fc_indptr, dtype=np.int32)
        nhf = int(ip[-1])
        t_hf, T, dT = np.empty(nhf), np.empty(self.nf), np.empty(nhf * 9)
        _lib.check(self.lib.pb_tpfa_diff(self.h, _lib.ptr(k, _lib._f64p), _lib.ptr(ip, _lib._i32p),
                                         _lib.ptr(t_hf, _lib._f64p), _lib.ptr(T, _lib._f64p), _lib.ptr(dT, _lib._f64p)))
        return t_hf, T, dT

    def upwind(self, darcy_flux, bc_bits):
        """Upstream cell per face (-1: face not in the matrix) and the two boundary diagonals."""
        q = _lib.f64(darcy_flux)
        bits = np.ascontiguousarray(bc_bits, dtype=np.uint8)
        up = np.empty(self.nf, np.int32)
        neu, dr = np.empty(self.nf), np.empty(self.nf)
        _lib.check(self.lib.pb_upwind(self.h, _lib.ptr(q, _lib._f64p), _lib.ptr(bits, _lib._u8p),
                                      _lib.ptr(up, _lib._i32p), _lib.ptr(neu, _lib._f64p), _lib.ptr(dr, _lib._f64p)))
        return up, neu, dr

    def tpsa(self, nd: int, mu, codes, robin_diag, face_flags, fc_indptr, face_areas) -> tuple:
        """Value arrays of the 14 TPSA terms in ``PB_TPSA_*`` order (layouts in include/poreb200.h; sizes from
        ``tpsa_value_counts``) and the kernel time in ms.  ``codes`` / ``robin_diag``: (nf, nd), ``face_flags``: nf."""
        mu = _lib.f64(mu)
        if mu.shape != (self.nc,):
            raise ValueError("fourth_order_tensor.mu must have one value per cell")
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        rob = None if robin_diag is None else _lib.f64(robin_diag)
        flags = np.ascontiguousarray(face_flags, dtype=np.uint8)
        ip = np.ascontiguousarray(fc_indptr, dtype=np.int32)
        _lib.check(self.lib.pb_facegrid_set_face_areas(self.h, _lib.ptr(_lib.f64(face_areas), _lib._f64p)))
        out = [_lib.pinned_empty(n) for n in tpsa_value_counts(nd, self.nf, int(ip[-1]))]
        ptrs = (_lib._f64p * len(out))(*[_lib.ptr(a, _lib._f64p) for a in out])
        ms = C.c_float(0.0)
        _lib.check(self.lib.pb_tpsa(self.h, int(nd), _lib.ptr(mu, _lib._f64p), _lib.ptr(cod, _lib._u8p),
                                    _lib.ptr(rob, _lib._f64p), _lib.ptr(flags, _lib._u8p), _lib.ptr(ip, _lib._i32p),
                                    ptrs, C.byref(ms)))
        return out, float(ms.value)

    def tpsa_system(self, nd: int, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas) -> tuple:
        """The TPSA three-field system matrix (``pb_tpsa_system``, layout in include/poreb200.h) as a ``DeviceCsr`` and
        the device times of its two stages in ms.  ``codes`` / ``robin_diag``: (nf, nd), ``face_flags``: nf."""
        return self._system(self.lib.pb_tpsa_system, nd, {"fourth_order_tensor.mu": mu,
                                                          "fourth_order_tensor.lmbda": lmbda,
                                                          "cell_volumes": cell_volumes},
                            codes, robin_diag, face_flags, face_areas)

    def tpsa_rhs(self, n: int, bc_values, body_force=None, angular_source=None, mass_source=None):
        """b = -R(0) of the TPSA system last assembled on this grid (``pb_tpsa_rhs``) as a CUDA tensor of ``n``
        doubles."""
        return self._rhs(self.lib.pb_tpsa_rhs, n, bc_values, body_force, angular_source, mass_source)

    def tpsa_poro_system(self, nd: int, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                         flux_pattern) -> tuple:
        """The TPSA poromechanics Jacobian with its mechanics rows (``pb_tpsa_poro_system``, layout in
        include/poreb200.h) as a ``DeviceCsr`` and the device times of its two stages in ms.  ``flux_pattern``: the
        ``DeviceCsr`` div @ flux whose rows give the fluid-row patterns."""
        return self._system(self.lib.pb_tpsa_poro_system, nd, self._poro_cells(mu, lmbda, alpha, cell_volumes), codes,
                            robin_diag, face_flags, face_areas, flux_pattern.h)

    def tpsa_thm_system(self, nd: int, mu, lmbda, alpha, cell_volumes, codes, robin_diag, face_flags, face_areas,
                        flux_pattern) -> tuple:
        """The TPSA thermo-poromechanics Jacobian with its mechanics rows (``pb_tpsa_thm_system``, layout in
        include/poreb200.h) as a ``DeviceCsr`` and the device times of its two stages in ms.  ``flux_pattern``: a
        ``DeviceCsr`` whose rows hold the union of the Darcy and Fourier div @ flux patterns."""
        return self._system(self.lib.pb_tpsa_thm_system, nd, self._poro_cells(mu, lmbda, alpha, cell_volumes), codes,
                            robin_diag, face_flags, face_areas, flux_pattern.h)

    @staticmethod
    def _poro_cells(mu, lmbda, alpha, cell_volumes) -> dict:
        return {"fourth_order_tensor.mu": mu, "fourth_order_tensor.lmbda": lmbda, "the Biot coefficient": alpha,
                "cell_volumes": cell_volumes}

    def tpsa_poro_rhs(self, n: int, bc_values, body_force=None, angular_source=None, mass_source=None):
        """-R(0) of the mechanics rows of the poromechanics system last assembled on this grid (``pb_tpsa_poro_rhs``),
        0 in the fluid rows, as a CUDA tensor of ``n`` doubles."""
        return self._rhs(self.lib.pb_tpsa_poro_rhs, n, bc_values, body_force, angular_source, mass_source)

    def tpsa_thm_rhs(self, n: int, bc_values, body_force=None, angular_source=None, mass_source=None):
        """-R(0) of the mechanics rows of the thermo-poromechanics system last assembled on this grid
        (``pb_tpsa_thm_rhs``), 0 in the mass and energy rows, as a CUDA tensor of ``n`` doubles."""
        return self._rhs(self.lib.pb_tpsa_thm_rhs, n, bc_values, body_force, angular_source, mass_source)

    def tpsa_poro_fluid_rows(self, A, jf, neg_res, rhs, missing=None) -> None:
        """Write the fluid rows of ``A`` (the matrix of ``tpsa_poro_system``) from the field-ordered fluid Jacobian
        ``jf`` (``DeviceCsr``, columns [p_t | p]) and the fluid entries of ``rhs`` from ``neg_res``, on the current
        stream (``pb_tpsa_poro_fluid_rows``).  ``missing``: int32 CUDA tensor counting entries outside the pattern."""
        self._balance_rows(self.lib.pb_tpsa_poro_fluid_rows, self.nc, A, jf, neg_res, rhs, missing)

    def tpsa_thm_balance_rows(self, A, jf, neg_res, rhs, missing=None) -> None:
        """Write the mass and energy rows of ``A`` (the matrix of ``tpsa_thm_system``) from the field-ordered Jacobian
        ``jf`` (``DeviceCsr``, rows [mass | energy], columns [p_t | p | T]) and their entries of ``rhs`` from
        ``neg_res`` (2 nc), on the current stream (``pb_tpsa_thm_balance_rows``).  ``missing``: int32 CUDA tensor
        counting entries outside the pattern."""
        self._balance_rows(self.lib.pb_tpsa_thm_balance_rows, 2 * self.nc, A, jf, neg_res, rhs, missing)

    def tpsa_contact_system(self, nd: int, mu, lmbda, cell_volumes, codes, robin_diag, face_flags, face_areas,
                            mortars: dict, frames, characteristic_traction: float) -> tuple:
        """The TPSA contact Jacobian with its balance and force rows (``pb_tpsa_contact_system``, layout in
        include/poreb200.h) as a ``DeviceCsr`` and the device times of its two stages in ms.  ``mortars``: per mortar
        cell (all interfaces in order) ``face``, ``cell`` (fracture cell, all fractures in order), ``m2p``, ``p2m``,
        ``sign`` and ``volume``; ``frames``: nd x nd per fracture cell, row-major."""
        face, cell = (np.ascontiguousarray(mortars[k], dtype=np.int32) for k in ("face", "cell"))
        w = [_lib.f64(mortars[k]) for k in ("m2p", "p2m", "sign", "volume")]
        nm, nk = face.size, int(np.asarray(frames).size) // (nd * nd)
        if cell.size != nm or any(a.size != nm for a in w):
            raise ValueError("every mortar array must have one value per mortar cell")
        fr = _lib.f64(frames)
        return self._system(self.lib.pb_tpsa_contact_system, nd, {"fourth_order_tensor.mu": mu,
                                                                  "fourth_order_tensor.lmbda": lmbda,
                                                                  "cell_volumes": cell_volumes},
                            codes, robin_diag, face_flags, face_areas, int(nm), int(nk), _lib.ptr(face, _lib._i32p),
                            _lib.ptr(cell, _lib._i32p), *[_lib.ptr(a, _lib._f64p) for a in w],
                            _lib.ptr(fr, _lib._f64p), float(characteristic_traction))

    def tpsa_contact_rhs(self, n: int, bc_values, body_force=None, angular_source=None, mass_source=None):
        """-R(0) of the balance and force rows of the contact system last assembled on this grid
        (``pb_tpsa_contact_rhs``), 0 in the contact rows, as a CUDA tensor of ``n`` doubles."""
        return self._rhs(self.lib.pb_tpsa_contact_rhs, n, bc_values, body_force, angular_source, mass_source)

    def tpsa_contact_rows(self, A, jc, neg_res, rhs, missing=None) -> None:
        """Write the contact rows of ``A`` (the matrix of ``tpsa_contact_system``) from the Jacobian ``jc`` of the
        [normal | tangential] laws in the variables [t | u_j] (``DeviceCsr``) and their entries of ``rhs`` from
        ``neg_res``, on the current stream (``pb_tpsa_contact_rows``).  ``missing``: int32 CUDA tensor counting entries
        outside the pattern."""
        self._balance_rows(self.lib.pb_tpsa_contact_rows, jc.shape[0], A, jc, neg_res, rhs, missing)

    def _system(self, fn, nd, cells: dict, codes, robin_diag, face_flags, face_areas, *extra) -> tuple:
        """``fn(handle, nd, *cells, codes, robin_diag, face_flags, *extra, &matrix, stage_ms)`` of a
        ``pb_tpsa_*_system`` entry point after checking that every array of ``cells`` (by name) has one value per cell
        and setting the face areas: the matrix as a ``DeviceCsr`` and the device times of its two stages in ms."""
        from .sparse import DeviceCsr
        cells = {name: _lib.f64(a) for name, a in cells.items()}
        for name, a in cells.items():
            if a.shape != (self.nc,):
                raise ValueError(f"{name} must have one value per cell")
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        rob = None if robin_diag is None else _lib.f64(robin_diag)
        flags = np.ascontiguousarray(face_flags, dtype=np.uint8)
        _lib.check(self.lib.pb_facegrid_set_face_areas(self.h, _lib.ptr(_lib.f64(face_areas), _lib._f64p)))
        h = C.c_void_p()
        ms = (C.c_float * 2)()
        _lib.check(fn(self.h, int(nd), *[_lib.ptr(a, _lib._f64p) for a in cells.values()], _lib.ptr(cod, _lib._u8p),
                      _lib.ptr(rob, _lib._f64p), _lib.ptr(flags, _lib._u8p), *extra, C.byref(h),
                      C.cast(ms, _lib._f32p)))
        return DeviceCsr.from_handle(h), [float(ms[0]), float(ms[1])]

    def _rhs(self, fn, n, bc_values, body_force, angular_source, mass_source):
        """``fn(handle, bc_values, body_force, angular_source, mass_source, b)`` of a ``pb_tpsa_*_rhs`` entry point
        (None: zero): b as a CUDA tensor of ``n`` doubles."""
        import torch
        arrs = [None if a is None else _lib.f64(a) for a in (bc_values, body_force, angular_source, mass_source)]
        b = torch.empty(int(n), dtype=torch.float64, device="cuda")
        _lib.check(fn(self.h, *[_lib.ptr(a, _lib._f64p) for a in arrs], C.c_void_p(b.data_ptr())))
        return b

    def _balance_rows(self, fn, n, A, jf, neg_res, rhs, missing):
        import torch
        from .sparse import device_operand
        neg_res = device_operand(neg_res.contiguous(), n, "neg_res")
        rhs = device_operand(rhs, A.shape[0], "rhs")
        mp = 0
        if missing is not None:
            if not (missing.is_cuda and missing.dtype == torch.int32 and missing.numel() == 1):
                raise TypeError("missing: one int32 CUDA element is required")
            mp = missing.data_ptr()
        _lib.check(fn(self.h, A.h, jf.h, C.c_void_p(neg_res.data_ptr()), C.c_void_p(rhs.data_ptr()), C.c_void_p(mp),
                      torch.cuda.current_stream().cuda_stream))


# (rows per face, columns per cell or face) of the 14 TPSA terms in PB_TPSA_* order; "k" marks kron(., I_nd), "r" the
# rotation dimension (nd in 3-D, 1 in 2-D), "d" the dimension.  The first ten terms have cell columns.
_TPSA_BLOCKS = (("d", "k"), ("d", "r"), ("d", 1), ("r", "d"), ("r", "r"), (1, "d"), (1, 1), ("d", "k"), ("d", "r"),
                ("d", 1), ("d", "k"), ("r", "d"), (1, "d"), ("d", "k"))
_TPSA_NCELLTERMS = 10


def _tpsa_block(nd: int, k: int):
    """(rows, columns, kron) of one block of TPSA term k."""
    nr = 3 if nd == 3 else 1
    size = {"d": nd, "r": nr, 1: 1}
    br, bc = _TPSA_BLOCKS[k]
    if bc == "k":
        return nd, nd, True
    return size[br], size[bc], False


def tpsa_value_counts(nd: int, nf: int, nnz: int) -> list:
    """Number of values of each TPSA term (``nnz`` = entries of cell_faces)."""
    counts = []
    for k in range(len(_TPSA_BLOCKS)):
        br, bc, kron = _tpsa_block(nd, k)
        per = br if kron else br * bc
        counts.append(per * (nnz if k < _TPSA_NCELLTERMS else nf))
    return counts



# ------------------------------------------------------------------------------------------
# boundary-condition encoding
# ------------------------------------------------------------------------------------------


def scalar_bc_codes(bc, nf: int) -> np.ndarray:
    """Face codes for MPFA.  Internal (fracture) faces are Neumann (mpfa.py:1452-1454)."""
    internal = np.asarray(getattr(bc, "is_internal", np.zeros(nf, bool)), bool)
    codes = np.zeros(nf, np.uint8)
    codes[np.asarray(bc.is_neu, bool) | internal] = _lib.BC_NEU
    codes[np.asarray(bc.is_dir, bool) & ~internal] = _lib.BC_DIR
    codes[np.asarray(bc.is_rob, bool) & ~internal] = _lib.BC_ROB
    return codes


def face_bc_bits(bc, nf: int) -> np.ndarray:
    """Boundary byte of the per-face kernels (csrc/face_kernels.cuh): effective code in bits 0-1
    (internal faces count as Neumann, tpfa.py:187-188), the raw ``is_dir`` / ``is_neu`` flags in
    bits 2 / 3 (used as such by tpfa.py:221-225 and upwind.py:260-270)."""
    internal = np.asarray(getattr(bc, "is_internal", np.zeros(nf, bool)), bool)
    is_dir, is_neu, is_rob = (np.asarray(getattr(bc, k), bool) for k in ("is_dir", "is_neu", "is_rob"))
    bits = np.zeros(nf, np.uint8)
    bits[is_rob & ~internal] = _lib.BC_ROB
    bits[is_dir & ~internal] = _lib.BC_DIR
    bits[is_neu | internal] = _lib.BC_NEU
    bits |= (is_dir.astype(np.uint8) << 2) | (is_neu.astype(np.uint8) << 3)
    return bits


def vector_bc_codes(bc, nd: int, nf: int):
    if getattr(bc, "bc_type", "vectorial") != "vectorial":
        raise AttributeError("MPSA must be given a vectorial boundary condition")  # mpsa.py:823
    codes = np.zeros((nd, nf), np.uint8)
    codes[np.asarray(bc.is_neu, bool)[:nd]] = _lib.BC_NEU
    codes[np.asarray(bc.is_dir, bool)[:nd]] = _lib.BC_DIR
    codes[np.asarray(bc.is_rob, bool)[:nd]] = _lib.BC_ROB
    robw = None
    if np.any(codes == _lib.BC_ROB):
        rw = np.asarray(bc.robin_weight, float)
        robw = np.ascontiguousarray(rw[:nd, :nd])
    return codes, robw


def vector_bc_basis(bc, nd: int, codes=None):
    """``bc.basis`` (nd, nd, nf) when it is not the identity on some boundary face, else None
    (_fvutils.py:765-945: boundary conditions given in a rotated coordinate system).  The basis acts on the equations
    of boundary sub-faces only, so with the (nd, nf) condition ``codes`` of ``vector_bc_codes`` the test reads the
    flagged faces instead of all of the (nd, nd, nf) array (40 ms at 2 * 10^6 faces, in front of every MPSA call)."""
    basis = getattr(bc, "basis", None)
    if basis is None:
        return None
    b = np.asarray(basis, float)
    if b.ndim != 3:
        return None
    sub = b[:nd, :nd]
    eye = np.eye(nd)[:, :, None]
    if sub.strides[-1] == 0:        # one matrix broadcast over the faces (e.g. a restricted shard condition)
        if np.array_equal(sub[:, :, :1], eye):
            return None
    else:
        probe = sub if codes is None else sub[:, :, np.flatnonzero(np.asarray(codes).any(axis=0))]
        if np.array_equal(probe, np.broadcast_to(eye, probe.shape)):
            return None   # the identity on every (boundary) face: exact test; anything else IS a rotated basis
    return np.ascontiguousarray(b[:nd, :nd])


# ------------------------------------------------------------------------------------------
# discretization classes
# ------------------------------------------------------------------------------------------


def active_indices(sd, params: dict):
    """Cells of the sub-grid to discretize and faces whose rows are (re)computed, from
    ``specified_cells / specified_faces / specified_nodes`` (``_fvutils.find_active_indices``,
    _fvutils.py:308-355, and ``cell_ind_for_partial_update``, :1260-1462).  Cells mode: the faces
    touching a node of the given cells, and every cell touching a node of those faces.  Faces mode
    (split faces): the faces sharing a node with the given ones, and two layers of cells around
    them.  Nodes mode (gradual build-up): the cells touching the given nodes, and the faces all of
    whose nodes are given.  Writes ``active_cells`` / ``active_faces`` into ``params``."""
    nc, nf, nn = sd.num_cells, sd.num_faces, sd.num_nodes
    spec = [params.get(k) for k in ("specified_cells", "specified_faces", "specified_nodes")]
    if all(v is None for v in spec):
        cells, faces = np.arange(nc), np.arange(nf)
        params["active_cells"], params["active_faces"] = cells, faces
        return cells, faces
    fn = abs(sps.csr_matrix(sd.face_nodes)).astype(np.float64)      # nn x nf
    cf = abs(sps.csr_matrix(sd.cell_faces)).astype(np.float64)      # nf x nc
    cn = (fn @ cf).tocsr()                                          # nn x nc

    def mask(n, idx):
        m = np.zeros(n)
        m[np.asarray(idx, dtype=np.int64)] = 1.0
        return m

    active_faces = np.zeros(nf, bool)
    cell_ind = np.zeros(nc, bool)
    if spec[0] is not None:
        vert = (cn @ mask(nc, spec[0])) > 0
        active_faces |= (fn.T @ vert.astype(np.float64)) > 0
        vert |= (fn @ active_faces.astype(np.float64)) > 0
        cell_ind |= (cn.T @ vert.astype(np.float64)) > 0
    if spec[1] is not None:
        pvert = (fn @ mask(nf, spec[1])) > 0
        active_faces |= (fn.T @ pvert.astype(np.float64)) > 0
        anodes = (fn @ active_faces.astype(np.float64)) > 0
        pcells = (cn.T @ anodes.astype(np.float64)) > 0
        anodes |= (cn @ pcells.astype(np.float64)) > 0
        cell_ind |= (cn.T @ anodes.astype(np.float64)) > 0
    if spec[2] is not None:
        vert = mask(nn, spec[2])
        cell_ind |= (cn.T @ vert) > 0
        active_faces |= np.asarray(fn.T @ vert).ravel() == np.asarray(fn.sum(axis=0)).ravel()
    cells, faces = np.flatnonzero(cell_ind), np.flatnonzero(active_faces)
    params["active_cells"], params["active_faces"] = cells, faces
    return cells, faces


def _replace_rows(old, new, keep_entity: np.ndarray):
    """``old`` with the rows of the flagged entities (block rows) replaced by those of ``new``."""
    old = sps.csr_matrix(old)
    new = sps.csr_matrix(new)
    br = new.shape[0] // keep_entity.size
    stay = sps.diags(np.repeat(~keep_entity, br).astype(np.float64))
    return (stay @ old + new).tocsr()


class _Base:
    """numerics/discretization.py:12-121."""

    def __init__(self, keyword: str) -> None:
        self.keyword = keyword
        self.last_timing: dict = {}

    def __repr__(self) -> str:
        """numerics/discretization.py:21-25."""
        return f"Discretization of type {self.__class__.__name__} with keyword {self.keyword}"

    def _key(self) -> str:
        return self.keyword + "_"

    def discretize(self, sd, data: dict) -> None:
        """Full discretization, or -- with ``specified_cells / specified_faces / specified_nodes`` in
        the parameters -- the reference's partial one (mpfa.py:176-201,468-508; biot.py:326-342,
        614-712): the sub-grid of the active cells is discretized as a whole (same kernels), the rows
        of the active faces (and, for Biot's cell-row terms, of the cells next to them) are embedded
        in global numbering, all other rows are zero -- or, with ``update_discretization = True``,
        keep the values already stored.  ``active_cells`` / ``active_faces`` are written back to the
        parameter dictionary as the reference does (_fvutils.py:346-353)."""
        params = data[PARAMETERS][self.keyword]
        mats = data.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        cells, faces = active_indices(sd, params)
        if cells.size == sd.num_cells and faces.size == sd.num_faces:
            mats.update(self._discretize_grid(sd, params))
            return
        from . import shard as _shard
        update = bool(params.get("update_discretization", False))
        keep_faces = np.zeros(sd.num_faces, bool)
        keep_faces[faces] = True
        if update:
            # Cell-row terms (Biot) sum over ALL nodes of a cell, and every cell sharing a node with a
            # modified one changes.  The reference replaces the rows of the cells next to an active face
            # although some of their nodes have cut interaction regions in its sub-grid (biot.py:627-632;
            # "update is not fully tested", biot.py:318-324).  Replacing stored rows must not corrupt
            # them: grow the sub-grid by one ring and replace exactly the rows of the cells all of whose
            # interaction regions are complete in it.
            cn = (abs(sps.csr_matrix(sd.face_nodes)) @ abs(sps.csr_matrix(sd.cell_faces))).tocsr()
            cn.data[:] = 1.0
            inside = np.zeros(sd.num_cells)
            inside[cells] = 1.0
            grown = (cn.T @ ((cn @ inside) > 0).astype(np.float64)) > 0
            complete_node = (cn @ grown.astype(np.float64)) == np.asarray(cn.sum(axis=1)).ravel()
            keep_cells = grown & ((cn.T @ (~complete_node).astype(np.float64)) == 0)
            cells = np.flatnonzero(grown)
        else:
            keep_cells = np.asarray(abs(sps.csr_matrix(sd.cell_faces)).T @ keep_faces.astype(np.float64)).ravel() > 0
        sub = _shard.extract_cells(sd, cells, keep_faces, keep_cells)
        local = _shard.restrict_parameters(params, sub)
        local.setdefault(self._eta_key, determine_eta(sd))
        out = {key: _shard.embed(sub, key, m) for key, m in self._discretize_grid(sub.grid, local).items()}
        if update:
            for key, new in out.items():
                keep = keep_faces if _shard._LAYOUT[key][0] == "face" else keep_cells
                if isinstance(new, dict):
                    mats[key] = {k: _replace_rows(mats[key][k], v, keep) for k, v in new.items()}
                else:
                    mats[key] = _replace_rows(mats[key], new, keep)
        else:
            mats.update(out)

    def update_discretization(self, sd, data: dict) -> None:
        """numerics/discretization.py:54: re-discretize (the partial path of ``discretize`` applies when
        ``specified_cells/faces/nodes`` are set)."""
        self.discretize(sd, data)

    def _check_unsupported(self, params: dict, sd=None) -> None:
        """``partition_arguments`` bound the reference's working set (``_fvutils.py:358-411``); the
        kernels stream over nodes and never materialise the global block-diagonal inverse, so the
        key is accepted and ignored.  Periodic face pairs
        (``_fvutils.py:95-140``) are not merged by the topology plan: refuse rather than discretize
        the pair as two boundaries."""
        if sd is not None and getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("periodic boundaries (sd.periodic_face_map) are not supported")
        return None


class Mpfa(_Base):
    """MPFA-O flux discretization; see module docstring.  Matrix keys as fv_elliptic.py:29-53."""

    def __init__(self, keyword: str) -> None:
        super().__init__(keyword)
        self.flux_matrix_key = "flux"
        self.bound_flux_matrix_key = "bound_flux"
        self.bound_pressure_cell_matrix_key = "bound_pressure_cell"
        self.bound_pressure_face_matrix_key = "bound_pressure_face"
        self.vector_source_matrix_key = "vector_source"
        self.bound_pressure_vector_source_matrix_key = "bound_pressure_vector_source"

    def ndof(self, sd) -> int:
        return sd.num_cells

    _eta_key = "mpfa_eta"

    def _discretize_grid(self, sd, params: dict) -> dict:
        """mpfa.py:65 on the whole of ``sd``.  Reads ``second_order_tensor``, ``bc``, optional
        ``mpfa_eta`` and ``ambient_dimension``; returns the six matrices of mpfa.py:496-508."""
        k = params["second_order_tensor"]
        bc = params["bc"]
        if sd.dim <= 1:
            # mpfa.py:687-722: the scheme reduces to TPFA on a line; a point grid has no faces
            sub = {"bc": bc, "second_order_tensor": k, "ambient_dimension": params.get("ambient_dimension", sd.dim)}
            tp = Tpfa(self.keyword)
            out = tp._discretize_grid(sd, sub)
            self.last_timing = tp.last_timing
            return out
        eta = params.get("mpfa_eta", None)
        if eta is None:
            eta = determine_eta(sd)
        if np.asarray(eta).size != 1:
            raise NotImplementedError("sub-face valued mpfa_eta is not supported")
        amb = int(params.get("ambient_dimension", sd.dim))
        if amb != sd.dim and not (sd.dim == 2 and amb == 3):
            raise NotImplementedError(f"ambient_dimension={amb} for a {sd.dim}-d grid is not supported")
        if np.asarray(bc.is_dir).shape[-1] != sd.num_faces:
            raise NotImplementedError("sub-face boundary conditions are not supported")
        self._check_unsupported(params, sd)
        t0 = time.perf_counter()
        plan = DevicePlan.for_grid(sd)
        codes = scalar_bc_codes(bc, sd.num_faces)
        robw = np.asarray(bc.robin_weight, float) if np.any(codes == _lib.BC_ROB) else None
        t1 = time.perf_counter()
        kvals = k.values
        if plan.rotation is not None:  # fracture plane: mpfa.py:733-754
            kvals = rotate_second_order(kvals, plan.rotation)
        plan.mpfa_upload(kvals, codes, robw, float(np.asarray(eta).ravel()[0]))
        t2 = time.perf_counter()
        ms = plan.mpfa_assemble()
        t3 = time.perf_counter()
        # device-resident results: scipy-compatible matrices whose arrays are fetched on first touch
        out = plan.mpfa_lazy() if hasattr(plan, "mpfa_lazy") else plan.mpfa_download()
        if sd.dim == 2 and (amb == 3 or plan.rotation is not None):
            # vector source back to the ambient space, mpfa.py:423-466 (with ambient_dimension = 2 on a tilted
            # plane the reference keeps the first two ambient components, mpfa.py:459-462)
            rows = (np.eye(3) if plan.rotation is None else plan.rotation)[:2, :amb]
            for key in (self.vector_source_matrix_key, self.bound_pressure_vector_source_matrix_key):
                out[key] = _lifted(plan, out[key], rows, sd.num_cells)
        t4 = time.perf_counter()
        self.last_timing = dict(plan_s=t1 - t0, upload_s=t2 - t1, kernel_ms=ms,
                                assemble_s=t3 - t2, download_s=t4 - t3)
        _log_throughput("Mpfa", self.keyword, sd, ms, t4 - t0, out)
        return out

    def assemble_matrix_rhs(self, sd, data: dict):
        """fv_elliptic.py:67-112: A = div @ flux, b = -div @ bound_flux @ bc_values
        (- div @ vector_source_discr @ vector_source).  When the stored matrices are still device resident
        (``LazyCsr`` not yet touched) the products run on the GPU from exactly those matrices and ``A`` comes back
        as a ``LazyCsr`` backed by the device system (``A.device_csr`` feeds ``porepy_b200.krylov`` directly);
        otherwise the host scipy products of the reference."""
        mats = data[DISCRETIZATION_MATRICES][self.keyword]
        params = data[PARAMETERS][self.keyword]
        flux, bflux = mats[self.flux_matrix_key], mats[self.bound_flux_matrix_key]
        vsd = mats.get(self.vector_source_matrix_key) if "vector_source" in params else None
        if _on_device(flux, bflux) and (vsd is None or _on_device(vsd)) and flux.shape == (sd.num_faces, sd.num_cells):
            plan = flux.plan
            vec = None
            if vsd is not None:
                vec = np.asarray(params["vector_source"], dtype=np.float64)
                rows = vsd.__dict__.get("plane_rows")
                if rows is not None:  # fracture plane: the device values live in the plane's frame
                    vec = (vec.reshape(-1, rows.shape[1]) @ rows.T).ravel()
            a = plan.mpfa_system(flux.device_values)
            b = plan.mpfa_rhs(params["bc_values"], vec, bound_flux=bflux.device_values,
                              vector_source_discr=None if vsd is None else vsd.device_values)
            return _lazy_system(a), b
        div = sd.divergence(dim=1)
        matrix = div @ flux
        rhs = -div @ (bflux @ params["bc_values"])
        if "vector_source" in params:
            rhs -= div @ (mats[self.vector_source_matrix_key] @ params["vector_source"])
        return matrix, rhs

    def assemble_matrix_rhs_device(self, sd, data: dict):
        """(``DeviceCsr``, host rhs) of ``assemble_matrix_rhs``; raises unless the stored matrices are still device
        resident."""
        a, b = self.assemble_matrix_rhs(sd, data)
        if getattr(a, "device_csr", None) is None:
            raise RuntimeError("the discretization matrices are no longer device resident")
        return a.device_csr, b


class Mpsa(_Base):
    """MPSA-W stress discretization; see module docstring.  Matrix keys as mpsa.py:82-95."""

    def __init__(self, keyword: str) -> None:
        super().__init__(keyword)
        self.stress_matrix_key = "stress"
        self.bound_stress_matrix_key = "bound_stress"
        self.bound_displacement_cell_matrix_key = "bound_displacement_cell"
        self.bound_displacement_face_matrix_key = "bound_displacement_face"

    def ndof(self, sd) -> int:
        return sd.dim * sd.num_cells

    def _alphas(self, sd, params):
        return {}

    _eta_key = "mpsa_eta"

    def _discretize_grid(self, sd, params: dict) -> dict:
        """mpsa.py:121 (and biot.py:247 through ``_alphas``) on the whole of ``sd``.  Reads
        ``fourth_order_tensor``, ``bc`` (vectorial), optional ``mpsa_eta``."""
        constit = params["fourth_order_tensor"]
        bc = params["bc"]
        if getattr(bc, "bc_type", "vectorial") != "vectorial":
            raise AttributeError("MPSA must be given a vectorial boundary condition")  # mpsa.py:658
        if sd.dim == 1:
            # mpsa.py:666-697: TPFA with the longitudinal modulus 2 mu + lambda, Neumann everywhere
            if np.any(bc.is_dir):
                raise ValueError("have not considered Dirichlet boundary values here")
            from .params import BoundaryCondition, SecondOrderTensor
            tp = Tpfa("tpfa_elasticity")
            sub = {"bc": BoundaryCondition(sd), "second_order_tensor": SecondOrderTensor(2 * constit.mu + constit.lmbda)}
            t = tp._discretize_grid(sd, sub)
            return {"stress": t["flux"], "bound_stress": t["bound_flux"],
                    "bound_displacement_cell": t["bound_pressure_cell"],
                    "bound_displacement_face": t["bound_pressure_face"]}
        eta = params.get("mpsa_eta", None)
        if eta is None:
            eta = determine_eta(sd)
        hf_eta = params.get("reconstruction_eta", None)
        if hf_eta is not None and hf_eta != eta:
            raise NotImplementedError("reconstruction_eta != mpsa_eta is not supported")
        if np.asarray(bc.is_dir).shape[-1] != sd.num_faces:
            raise NotImplementedError("sub-face boundary conditions are not supported")
        self._check_unsupported(params, sd)
        alphas = self._alphas(sd, params)
        t0 = time.perf_counter()
        plan = DevicePlan.for_grid(sd)
        if plan.rotation is not None:
            # the reference discretizes in the local frame of map_grid without rotating the stiffness
            # back (mpsa.py:2005-2040): frame dependent, and not a use case (mechanics lives on the
            # top-dimensional grid)
            raise NotImplementedError("MPSA on a 2-D grid outside the xy-plane is not supported")
        codes, robw = vector_bc_codes(bc, sd.dim, sd.num_faces)
        t1 = time.perf_counter()
        plan.mpsa_upload(constit.values, codes, robw, float(eta), list(alphas.values()))
        plan.mpsa_set_basis(vector_bc_basis(bc, sd.dim, codes))
        t2 = time.perf_counter()
        ms = plan.mpsa_assemble()
        t3 = time.perf_counter()
        lazy = hasattr(plan, "mpsa_lazy")
        out = plan.mpsa_lazy() if lazy else plan.mpsa_download()
        if alphas:
            coupled = {k: {} for k in ("displacement_divergence", "boundary_displacement_divergence",
                                       "scalar_gradient", "mpsa_consistency",
                                       "bound_displacement_pressure")}
            for q, key in enumerate(alphas):
                for name, m in (plan.biot_lazy(q) if lazy else plan.biot_download(q)).items():
                    coupled[name][key] = m
            out.update(coupled)
        t4 = time.perf_counter()
        self.last_timing = dict(plan_s=t1 - t0, upload_s=t2 - t1, kernel_ms=ms,
                                assemble_s=t3 - t2, download_s=t4 - t3)
        _log_throughput(type(self).__name__, self.keyword, sd, ms, t4 - t0, out)
        return out

    def assemble_matrix_rhs(self, sd, data: dict):
        """mpsa.py:486-529; device path as in ``Mpfa.assemble_matrix_rhs``."""
        mats = data[DISCRETIZATION_MATRICES][self.keyword]
        params = data[PARAMETERS][self.keyword]
        stress, bstress = mats["stress"], mats["bound_stress"]
        if _on_device(stress, bstress) and stress.shape[0] == sd.num_faces * sd.dim:
            plan = stress.plan
            a = plan.mpsa_system(stress.device_values)
            b = plan.mpsa_rhs(params["bc_values"], params["source"], bound_stress=bstress.device_values)
            return _lazy_system(a), b
        div = sd.divergence(dim=sd.dim)
        matrix = div @ stress
        rhs = -div @ (bstress @ params["bc_values"]) + params["source"]
        return matrix, rhs

    def assemble_matrix_rhs_device(self, sd, data: dict):
        """(``DeviceCsr``, host rhs); see ``Mpfa.assemble_matrix_rhs_device``."""
        a, b = self.assemble_matrix_rhs(sd, data)
        if getattr(a, "device_csr", None) is None:
            raise RuntimeError("the discretization matrices are no longer device resident")
        return a.device_csr, b


class Biot(Mpsa):
    """MPSA + Biot coupling terms (biot.py:40; keys :94-111, dict-valued per coupling keyword)."""

    def __init__(self, keyword: str = "mechanics") -> None:
        super().__init__(keyword)
        self.displacement_divergence_matrix_key = "displacement_divergence"
        self.bound_displacement_divergence_matrix_key = "boundary_displacement_divergence"
        self.scalar_gradient_matrix_key = "scalar_gradient"
        self.consistency_matrix_key = "mpsa_consistency"
        self.bound_pressure_matrix_key = "bound_displacement_pressure"

    def _alphas(self, sd, params):
        out = {}
        for key, a in params["scalar_vector_mappings"].items():
            if isinstance(a, (float, int, np.floating, np.integer)):
                v = np.zeros((3, 3, sd.num_cells))
                v[0, 0] = v[1, 1] = v[2, 2] = float(a)  # biot.py:312-321
            else:
                v = np.asarray(a.values, float)
            out[key] = v
        if len(out) > 4:
            raise NotImplementedError("at most 4 coupling tensors per Biot discretization")
        return out

    def assemble_matrix_rhs(self, sd, data: dict):
        """biot.py:125-149."""
        raise NotImplementedError("This class cannot be used for assembly.\nUse the ad version instead")


def _empty_flux_terms(discr, sd, vdim: int) -> dict:
    """The 0-D shortcut of tpfa.py:87-104 (a point grid has no faces)."""
    nc = sd.num_cells
    return {
        discr.flux_matrix_key: sps.csr_matrix((0, nc)),
        discr.bound_flux_matrix_key: sps.csr_matrix((0, 0)),
        discr.bound_pressure_cell_matrix_key: sps.csr_matrix((0, nc)),
        discr.bound_pressure_face_matrix_key: sps.csr_matrix((0, 0)),
        discr.vector_source_matrix_key: sps.csr_matrix((0, nc * max(vdim, 1))),
        discr.bound_pressure_vector_source_matrix_key: sps.csr_matrix((0, nc * max(vdim, 1))),
    }


class Tpfa(Mpfa):
    """Two-point flux approximation (numerics/fv/tpfa.py:18; same keys and ``assemble_matrix_rhs`` as
    MPFA through FVElliptic).  One thread per face on a ``FaceGrid``; grids of any dimension, anywhere in
    space (the reference works on the 3-D coordinates, tpfa.py:160-175)."""

    def discretize(self, sd, data: dict) -> None:
        """tpfa.py:40: always the whole grid -- the reference's TPFA has no partial mode, so
        ``specified_cells/faces/nodes`` (possibly left behind by an MPFA update on the same keyword,
        _fvutils.py:346-353) and ``update_discretization`` are ignored."""
        params = data[PARAMETERS][self.keyword]
        mats = data.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        mats.update(self._discretize_grid(sd, params))

    def _discretize_grid(self, sd, params: dict) -> dict:
        vdim = int(params.get("ambient_dimension", sd.dim))
        if sd.dim == 0:
            return _empty_flux_terms(self, sd, vdim)
        k = params["second_order_tensor"]
        bc = params["bc"]
        self._check_unsupported(params, sd)
        t0 = time.perf_counter()
        fg = FaceGrid.for_grid(sd)
        fc = sps.csr_matrix(sd.cell_faces)
        fc.sort_indices()
        ip, ix = fc.indptr, fc.indices
        vals = fg.tpfa(k.values, face_bc_bits(bc, sd.num_faces), ip, vdim)
        nf, nc = sd.num_faces, sd.num_cells
        boundary = np.diff(ip) == 1
        cols_v = (ix[:, None].astype(np.int64) * vdim + np.arange(vdim)).ravel()
        ipv = ip.astype(np.int64) * vdim
        self.last_timing = dict(total_s=time.perf_counter() - t0)
        return {
            self.flux_matrix_key: sps.csr_matrix((vals[0], ix, ip), shape=(nf, nc)),
            self.bound_flux_matrix_key: sps.diags(np.where(boundary, vals[4], 0.0)).tocsr(),
            self.bound_pressure_cell_matrix_key: sps.csr_matrix((vals[1], ix, ip), shape=(nf, nc)),
            self.bound_pressure_face_matrix_key: sps.diags(vals[5]).tocsr(),
            self.vector_source_matrix_key: sps.csr_matrix((vals[2], cols_v, ipv), shape=(nf, nc * vdim)),
            self.bound_pressure_vector_source_matrix_key: sps.csr_matrix((vals[3], cols_v, ipv),
                                                                         shape=(nf, nc * vdim)),
        }


def _tpsa_patterns(nd: int, nc: int, nf: int, ip: np.ndarray, ix: np.ndarray) -> list:
    """(indptr, indices, shape) of the 14 TPSA terms in the value layouts of ``pb_tpsa`` (include/poreb200.h).  Cell
    terms expand the face x cell pattern with ``block_expand``; kron(., I_nd) terms keep column c*nd + i in row
    f*nd + i; face terms are block diagonal."""
    out, cache = [], {}
    for k in range(len(_TPSA_BLOCKS)):
        br, bc, kron = _tpsa_block(nd, k)
        key = (k < _TPSA_NCELLTERMS, br, bc, kron)
        if key not in cache:
            if k < _TPSA_NCELLTERMS:
                nip, cols = block_expand(ip, ix, br, 1 if kron else bc)
                if kron:
                    rows = np.repeat(np.arange(nf * br, dtype=np.int64), np.diff(nip))
                    cols = cols * nd + rows % nd
                shape = (nf * br, nc * bc)
            else:
                per = 1 if kron else bc
                nip = np.arange(0, nf * br * per + 1, per, dtype=np.int64)
                if kron:
                    cols = np.arange(nf * br, dtype=np.int64)
                else:
                    cols = ((np.arange(nf * br, dtype=np.int64) // br) * bc)[:, None] + np.arange(bc, dtype=np.int64)
                shape = (nf * br, nf * bc)
            dt = _index_dtype(int(nip[-1]), shape[1])
            cache[key] = (nip.astype(dt), cols.reshape(-1).astype(dt), shape)
        out.append(cache[key])
    return out


def tpsa_bc_arrays(bc, nd: int, nf: int):
    """Per-(face, component) codes (nf, nd) and diagonal Robin weights (nf, nd) or None, after the refusals of
    tpsa.py:572-618 (same exceptions and messages)."""
    basis = np.asarray(bc.basis)
    if np.logical_or.reduce((np.any(basis[0, 1:, :] > 0), np.any(basis[1, 0, :] > 0), np.any(basis[1, 2:, :] > 0),
                             np.any(basis[2:, :2, :] > 0), np.any(basis[0, 0, :] != 1),
                             np.any(basis[1, 1, :] != 1))):
        raise NotImplementedError("Have not implemented Robin conditions with a non-trivial basis.")
    if nd == 3 and np.any(basis[2, 2] != 1):
        raise NotImplementedError("Have not implemented Robin conditions with a non-trivial basis.")
    rw = np.asarray(bc.robin_weight)
    if np.logical_or.reduce((np.any(rw[0, 1:, :] > 0), np.any(rw[1, 0, :] > 0), np.any(rw[1, 2:, :] > 0),
                             np.any(rw[2:, :2, :] > 0))):
        raise NotImplementedError("Non-diagonal Robin weights have not been implemnted.")
    is_rob = np.asarray(bc.is_rob, bool)[:nd]
    if not all(np.logical_xor(np.any(is_rob, axis=0), np.logical_not(np.all(is_rob, axis=0)))):
        raise NotImplementedError("Mixing Robin with Dirichlet or Neumann conditions is not implemneted.")
    codes = np.zeros((nf, nd), np.uint8)
    codes[np.asarray(bc.is_neu, bool)[:nd].T] = _lib.BC_NEU
    codes[np.asarray(bc.is_dir, bool)[:nd].T] = _lib.BC_DIR
    codes[is_rob.T] = _lib.BC_ROB
    robin = None
    if is_rob.any():
        robin = np.ascontiguousarray(np.stack([rw[i, i] for i in range(nd)], axis=1), dtype=np.float64)
    return codes, robin


def tpsa_face_inputs(sd, bc, nd: int):
    """(codes, robin, flags) of the TPSA face kernels on ``sd``: ``tpsa_bc_arrays`` of the vectorial ``bc`` and the
    boundary-face flags (nf uint8), after the refusals of ``tpsa_bc_arrays`` and of a 2-D grid whose face normals leave
    the xy-plane."""
    codes, robin = tpsa_bc_arrays(bc, nd, sd.num_faces)
    if nd == 2 and np.any(np.abs(sd.face_normals[2]) > np.maximum(np.abs(sd.face_normals[0]),
                                                                   np.abs(sd.face_normals[1]))):
        # tpsa.py:1053-1054 indexes is_dir (2 rows) with the argmax over all three rows of the normals
        raise IndexError("Tpsa: a face normal of a 2d grid points mostly out of the xy-plane")
    flags = np.zeros(sd.num_faces, np.uint8)
    flags[np.asarray(sd.get_all_boundary_faces(), dtype=np.int64)] = 1
    return codes, robin, flags


class Tpsa(_Base):
    """Two-point stress approximation (numerics/fv/tpsa.py:136, Nordbotten & Keilegavlen): the same constructor,
    matrix keys (:265-331), ``ndof`` and ``discretize`` outputs as the reference, computed by one thread per face on a
    ``FaceGrid`` (csrc/tpsa_face.cuh).  The matrices are scipy CSR with the fixed block pattern of each term; values
    equal the reference's (its explicit zeros are not reproduced).  Always the whole grid: the reference has no
    partial mode."""

    def __init__(self, keyword: str) -> None:
        super().__init__(keyword)
        self.stress_displacement_matrix_key = "stress"
        self.stress_rotation_matrix_key = "stress_rotation"
        self.stress_total_pressure_matrix_key = "stress_total_pressure"
        self.rotation_displacement_matrix_key = "rotation_displacement"
        self.rotation_rotation_matrix_key = "rotation_rotation"
        self.mass_total_pressure_matrix_key = "solid_mass_total_pressure"
        self.mass_displacement_matrix_key = "solid_mass_displacement"
        self.bound_stress_matrix_key = "bound_stress"
        self.bound_rotation_displacement_matrix_key = "bound_rotation_displacement"
        self.bound_mass_displacement_matrix_key = "bound_mass_displacement"
        self.bound_displacement_cell_matrix_key = "bound_displacement_cell"
        self.bound_displacement_face_matrix_key = "bound_displacement_face"
        self.bound_displacement_rotation_cell_matrix_key = "bound_displacement_rotation_cell"
        self.bound_displacement_solid_pressure_cell_matrix_key = "bound_displacement_solid_pressure_cell"

    def _term_keys(self) -> list:
        """Matrix keys in PB_TPSA_* order."""
        return [self.stress_displacement_matrix_key, self.stress_rotation_matrix_key,
                self.stress_total_pressure_matrix_key, self.rotation_displacement_matrix_key,
                self.rotation_rotation_matrix_key, self.mass_displacement_matrix_key,
                self.mass_total_pressure_matrix_key, self.bound_displacement_cell_matrix_key,
                self.bound_displacement_rotation_cell_matrix_key,
                self.bound_displacement_solid_pressure_cell_matrix_key, self.bound_stress_matrix_key,
                self.bound_rotation_displacement_matrix_key, self.bound_mass_displacement_matrix_key,
                self.bound_displacement_face_matrix_key]

    def ndof(self, sd) -> int:
        """tpsa.py:333-348."""
        if sd.dim == 2:
            return sd.num_cells * (2 + sd.dim)
        elif sd.dim == 3:
            return sd.num_cells * (1 + 2 * sd.dim)
        raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")

    def assemble_matrix_rhs(self, sd, sd_data: dict):
        """tpsa.py:350-374: assembly belongs to the multiphysics models."""
        raise NotImplementedError(
            """This class cannot be used for assembly.
            Use a multiphysics model class instead."""
        )

    def discretize(self, sd, data: dict) -> None:
        params = data[PARAMETERS][self.keyword]
        mats = data.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        mats.update(self._discretize_grid(sd, params))

    def _discretize_grid(self, sd, params: dict) -> dict:
        nd, nc, nf = sd.dim, sd.num_cells, sd.num_faces
        if nd not in (2, 3):
            raise NotImplementedError("Tpsa is only implemented for 2d and 3d grids.")
        self._check_unsupported(params, sd)
        mu = params["fourth_order_tensor"].mu
        codes, robin, flags = tpsa_face_inputs(sd, params["bc"], nd)
        t0 = time.perf_counter()
        fg = FaceGrid.for_grid(sd)
        fc = sps.csr_matrix(sd.cell_faces)
        fc.sort_indices()
        ip, ix = fc.indptr, fc.indices
        vals, kernel_ms = fg.tpsa(nd, mu, codes, robin, flags, ip, sd.face_areas)
        t1 = time.perf_counter()
        # the index arrays depend on the topology only: built once per grid, copied per matrix (scipy may edit a
        # matrix's index arrays in place, e.g. eliminate_zeros)
        cached = getattr(sd, "_b200_tpsa_patterns", None)
        if (cached is None or cached[0] != nd or not np.array_equal(cached[1], ip)
                or not np.array_equal(cached[2], ix)):
            cached = (nd, ip.copy(), ix.copy(), _tpsa_patterns(nd, nc, nf, ip, ix))
            try:
                sd._b200_tpsa_patterns = cached
            except AttributeError:
                pass
        mats = {key: sps.csr_matrix((v, pat[1].copy(), pat[0].copy()), shape=pat[2])
                for key, v, pat in zip(self._term_keys(), vals, cached[3])}
        self.last_timing = dict(kernel_ms=kernel_ms, device_s=t1 - t0, total_s=time.perf_counter() - t0)
        return mats


def line_frame(sd, tol: float = 1e-5) -> np.ndarray:
    """Rotation ``R`` (3, 3) whose first row is the direction of a straight 1-D grid (the frame the mixed schemes
    discretize a line in; any orthonormal completion gives the same matrices).  Raises ``ValueError`` when the nodes
    deviate from the line by more than ``tol`` relative to the grid's extent."""
    x = np.asarray(sd.nodes, dtype=np.float64)
    xc = x - x.mean(axis=1, keepdims=True)
    _, v = np.linalg.eigh(xc @ xc.T)          # ascending: v[:, 2] is the line's direction
    t = v[:, 2]
    off = xc - np.outer(t, t @ xc)
    if np.abs(off).max() > tol * max(np.abs(xc).max(), 1e-300):
        raise ValueError("1-D grid is not straight")
    return np.vstack((t, v[:, 1], v[:, 0]))


def dual_frame(sd, tol: float = 1e-5) -> np.ndarray:
    """The rotation that takes a grid into its own frame for MVEM / RT0: identity in 3-D and for 2-D grids in a plane
    z = const, ``line_frame`` for lines.  Other planes (checked by ``plane_frame`` with the same
    ``deviation_from_plane_tol``) are turned about n x e_z until their normal n is e_z, as ``map_geometry.map_grid``
    does, with n the cross product of the longest centred node vector and the one giving the longest product.  MVEM
    needs that very in-plane basis: its stabilization weight |K^-1|_inf is not invariant under in-plane rotations."""
    if sd.dim == 1:
        return line_frame(sd, tol)
    if sd.dim != 2 or plane_frame(sd, tol) is None:
        return np.eye(3)
    v = np.asarray(sd.nodes, dtype=np.float64)
    v = v - v.mean(axis=1, keepdims=True)
    v1 = v[:, np.argmax(np.linalg.norm(v, axis=0))]
    cross = np.cross(v1, v.T).T
    n = cross[:, np.argmax(np.linalg.norm(cross, axis=0))]
    n = n / np.linalg.norm(n)
    axis = np.cross(n, [0.0, 0.0, 1.0])
    if np.allclose(axis, 0.0):   # the reference's test in map_geometry.rotation_matrix
        return np.eye(3)
    axis = axis / np.linalg.norm(axis)
    a = np.arccos(n[2])
    W = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    return np.eye(3) + np.sin(a) * W + (1.0 - np.cos(a)) * (W @ W)


class DualGrid:
    """Device topology of a grid for the mixed schemes (``pb_dual``): cell_faces with the faces of every cell sorted,
    face_nodes, and the FACE x FACE mass pattern, built on the device at the first use and kept here.  Cached on the
    grid object and rebuilt when the topology changes."""

    def __init__(self, sd):
        lib = _lib.load()
        _lib.require_gpu()
        self.lib = lib
        cf = sps.csc_matrix(sd.cell_faces, copy=True)
        cf.sort_indices()
        fn = sps.csc_matrix(sd.face_nodes)
        self.nd, self.nc, self.nf, self.nn = int(sd.dim), sd.num_cells, sd.num_faces, sd.num_nodes
        self.cf_ip, self.cf_ix = cf.indptr.astype(np.int32), cf.indices.astype(np.int32)
        cfd = np.asarray(cf.data).astype(np.int8)
        fnp, fni = fn.indptr.astype(np.int32), fn.indices.astype(np.int32)
        h = C.c_void_p()
        _lib.check(lib.pb_dual_create(self.nd, self.nc, self.nf, self.nn, _lib.ptr(self.cf_ip, _lib._i32p),
                                      _lib.ptr(self.cf_ix, _lib._i32p), _lib.ptr(cfd, _lib._i8p),
                                      _lib.ptr(fnp, _lib._i32p), _lib.ptr(fni, _lib._i32p), C.byref(h)))
        self.h = h
        self.fingerprint = DevicePlan._fingerprint(sd, sd.cell_faces, sd.face_nodes)
        self._mass = None
        self._proj = None
        self.pattern_seconds = 0.0
        self.live, self.current = [], None

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            try:
                self.lib.pb_dual_destroy(h)
            except Exception:
                pass
            self.h = None

    @classmethod
    def for_grid(cls, sd) -> "DualGrid":
        fp = DevicePlan._fingerprint(sd, sd.cell_faces, sd.face_nodes)
        dg = getattr(sd, "_b200_dual", None)
        if dg is None or dg.fingerprint != fp:
            dg = cls(sd)
            try:
                sd._b200_dual = dg
            except AttributeError:
                pass
        return dg

    def mass_pattern(self):
        """(indptr, indices) of the FACE x FACE mass pattern."""
        if self._mass is None:
            t0 = time.perf_counter()
            nnz = C.c_int64(0)
            _lib.check(self.lib.pb_dual_mass_pattern(self.h, C.byref(nnz), None, None))
            ip, ix = np.empty(self.nf + 1, np.int32), np.empty(nnz.value, np.int32)
            _lib.check(self.lib.pb_dual_mass_pattern(self.h, C.byref(nnz), _lib.ptr(ip, _lib._i32p),
                                                     _lib.ptr(ix, _lib._i32p)))
            self._mass = (ip, ix)
            self.pattern_seconds = time.perf_counter() - t0
        return self._mass

    def proj_pattern(self):
        """(indptr, indices) of the (3 nc x nf) flux reconstruction: row 3c + a holds the faces of c."""
        if self._proj is None:
            n = np.diff(self.cf_ip).astype(np.int64)
            start = 3 * self.cf_ip[:-1].astype(np.int64)[:, None] + np.arange(3) * n[:, None]
            ip = np.append(start.ravel(), 3 * int(self.cf_ip[-1]))
            lens = np.repeat(n, 3)
            cell = np.repeat(np.arange(3 * self.nc) // 3, lens)
            off = np.arange(int(ip[-1])) - np.repeat(ip[:-1], lens)
            self._proj = (ip.astype(np.int32), self.cf_ix[self.cf_ip[cell] + off])
        return self._proj

    def discretize(self, method: int, geo, perm, rot):
        """Run the per-cell kernel; the mass values (in ``mass_pattern``) and flux reconstruction values (in
        ``proj_pattern``) stay on the device until ``download``.  Returns the first cell failing the MVEM consistency
        test (-1: none) and the kernel time in ms.  ``geo``: nodes, face normals, face centres, cell centres (each
        (3, n)) and cell volumes, in the frame ``rot``; ``perm`` (3, 3, nc) in that frame."""
        self.mass_pattern()
        arrs = [_lib.f64(a) for a in geo] + [_lib.f64(perm), _lib.f64(rot)]
        bad, ms = C.c_int64(-1), C.c_float(0.0)
        _lib.check(self.lib.pb_dual_discretize(self.h, int(method), *[_lib.ptr(a, _lib._f64p) for a in arrs], None,
                                               None, C.byref(bad), C.byref(ms)))
        return int(bad.value), float(ms.value)

    def download(self):
        """Mass and flux reconstruction values of the last ``discretize``."""
        mass, proj = np.empty(self.mass_pattern()[1].size), np.empty(3 * int(self.cf_ip[-1]))
        _lib.check(self.lib.pb_dual_download(self.h, _lib.ptr(mass, _lib._f64p), _lib.ptr(proj, _lib._f64p)))
        return mass, proj

    def system(self, codes, robin_weight, face_areas, bc_values, vector_source=None):
        """The saddle-point system of the last ``discretize`` assembled on the device (``pb_dual_system``): a
        ``DeviceCsr``, the right-hand side and |mass|_inf."""
        from .sparse import DeviceCsr
        arrs = [_lib.f64(a) for a in (robin_weight, face_areas, bc_values)]
        vs = None if vector_source is None else _lib.f64(vector_source)
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        rhs, norm, h = np.empty(self.nf + self.nc), C.c_double(0.0), C.c_void_p()
        _lib.check(self.lib.pb_dual_system(self.h, _lib.ptr(cod, _lib._u8p), *[_lib.ptr(a, _lib._f64p) for a in arrs],
                                           _lib.ptr(vs, _lib._f64p), C.byref(h), _lib.ptr(rhs, _lib._f64p),
                                           C.byref(norm)))
        return DeviceCsr.from_handle(h), rhs, float(norm.value)

    @staticmethod
    def _geo_ptrs(geo):
        """Geometry pointers of the hybrid entry points: nodes, face normals, face centres, cell centres, cell volumes,
        perm, rot and aperture, or eight NULLs (the geometry of the last ``discretize``)."""
        if geo is None:
            return [None] * 8, []
        arrs = [_lib.f64(a) for a in geo]
        return [_lib.ptr(a, _lib._f64p) for a in arrs], arrs

    def hybrid_system(self, mode: int, geo, codes, robin_weight, face_areas, values):
        """The hybridized face system (``pb_dual_hybrid_system``): a ``DeviceCsr`` in the mass pattern, its right-hand
        side, the first cell failing the MVEM consistency test (-1: none) and the kernel time in ms."""
        from .sparse import DeviceCsr
        ptrs, keep = self._geo_ptrs(geo)
        arrs = [_lib.f64(a) for a in (robin_weight, face_areas, values)]
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        rhs, h, bad, ms = np.empty(self.nf), C.c_void_p(), C.c_int64(-1), C.c_float(0.0)
        _lib.check(self.lib.pb_dual_hybrid_system(self.h, int(mode), *ptrs, _lib.ptr(cod, _lib._u8p),
                                                  *[_lib.ptr(a, _lib._f64p) for a in arrs], C.byref(h),
                                                  _lib.ptr(rhs, _lib._f64p), C.byref(bad), C.byref(ms)))
        return DeviceCsr.from_handle(h), rhs, int(bad.value), float(ms.value)

    def hybrid_recover(self, mode: int, geo, codes, values, lam):
        """[u; p] from the face pressures ``lam`` (``pb_dual_hybrid_recover``) and the kernel time in ms."""
        ptrs, keep = self._geo_ptrs(geo)
        cod = np.ascontiguousarray(codes, dtype=np.uint8)
        vals, lam = _lib.f64(values), _lib.f64(lam)
        up, ms = np.empty(self.nf + self.nc), C.c_float(0.0)
        _lib.check(self.lib.pb_dual_hybrid_recover(self.h, int(mode), *ptrs, _lib.ptr(cod, _lib._u8p),
                                                   _lib.ptr(vals, _lib._f64p), _lib.ptr(lam, _lib._f64p),
                                                   _lib.ptr(up, _lib._f64p), C.byref(ms)))
        return up, float(ms.value)


def dual_bc_codes(sd, bc) -> np.ndarray:
    """PB_BC_* per face for the mixed schemes: Dirichlet, Neumann and Robin faces that are not internal."""
    internal = np.asarray(bc.is_internal, bool)
    codes = np.zeros(sd.num_faces, np.uint8)
    codes[np.asarray(bc.is_dir, bool) & ~internal] = _lib.BC_DIR
    codes[np.asarray(bc.is_rob, bool) & ~internal] = _lib.BC_ROB
    codes[np.asarray(bc.is_neu, bool) & ~internal] = _lib.BC_NEU
    return codes


def _to_host(x) -> np.ndarray:
    """A solver's solution (torch tensor on any device, or array) as a float64 NumPy array."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=np.float64)


class _DualElliptic(_Base):
    """Mixed (dual) discretizations of Darcy flow (numerics/vem/dual_elliptic.py ``DualElliptic``): the same
    constructor, matrix keys (``mass``, ``div``, ``vector_proj``), ``ndof`` and helpers.  ``discretize`` computes the
    local matrices of every cell on the GPU (csrc/dual_cell.cuh), one thread per (cell, face); the matrices are scipy
    CSR.  Always the whole grid: the reference has no partial mode."""

    _method = -1

    def __init__(self, keyword: str, name: str = "") -> None:
        super().__init__(keyword)
        self.name = name or type(self).__name__
        self.mass_matrix_key = "mass"
        self.div_matrix_key = "div"
        self.vector_proj_key = "vector_proj"
        self.vector_source_key = "vector_source"

    def ndof(self, sd) -> int:
        return sd.num_cells + sd.num_faces

    def discretize(self, sd, data: dict) -> None:
        mats = data.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        if sd.dim == 0:   # mvem.py / rt0.py: identity mass, empty divergence and projection
            mats[self.mass_matrix_key] = sps.dia_matrix(([1], 0), (sd.num_faces, sd.num_faces))
            mats[self.div_matrix_key] = sps.csr_matrix((sd.num_faces, sd.num_cells))
            mats[self.vector_proj_key] = sps.csr_matrix((3, 0))
            return
        params = data[PARAMETERS][self.keyword]
        if sd.dim < 3 and data.get("is_tangential", False):
            raise NotImplementedError(f"{self.name}: is_tangential=True (a tensor in the map_grid frame) is not supported")
        self._check_unsupported(params, sd)
        if self._method == _lib.DUAL_RT0:
            n = np.diff(sps.csc_matrix(sd.cell_faces).indptr)
            if np.any(n != sd.dim + 1):
                c = int(np.flatnonzero(n != sd.dim + 1)[0])
                raise ValueError(f"RT0 needs simplices: cell {c} has {n[c]} faces")
        t0 = time.perf_counter()
        rot = dual_frame(sd, data.get("deviation_from_plane_tol", 1e-5))
        geo = [rot @ np.asarray(a, dtype=np.float64) for a in (sd.nodes, sd.face_normals, sd.face_centers,
                                                                 sd.cell_centers)]
        geo.append(sd.cell_volumes)
        perm = rotate_second_order(params["second_order_tensor"].values, rot)
        dg = DualGrid.for_grid(sd)
        first = dg._mass is None
        for m in dg.live:   # the device values are about to be overwritten: fetch those still referenced
            if m.__dict__.get("_lazy_data") is None:
                m.data
        bad, ms = dg.discretize(self._method, geo, perm, rot)
        if bad >= 0:   # mvem.py massHdiv: assert np.allclose(G, F @ D)
            raise AssertionError(f"MVEM: the consistency test G == F D fails in cell {bad}")
        t1 = time.perf_counter()
        mip, mix = dg.mass_pattern()
        pip, pix = dg.proj_pattern()
        nf, nc = sd.num_faces, sd.num_cells
        from .sparse import LazyCsr
        cache = {}

        def values():
            if "v" not in cache:
                cache["v"] = dg.download()
            return cache["v"]
        mass = LazyCsr.lazy((nf, nf), mix.size, lambda: values()[0], lambda: mix.copy(), lambda: mip.copy())
        proj = LazyCsr.lazy((3 * nc, nf), pix.size, lambda: values()[1], lambda: pix.copy(), lambda: pip.copy())
        div = -sps.csc_matrix(sd.cell_faces).T.tocsr()
        dg.live = [mass, proj]
        dg.current = (mass, proj, div)
        out = {self.mass_matrix_key: mass, self.div_matrix_key: div, self.vector_proj_key: proj}
        mats.update(out)
        self.last_timing = dict(kernel_ms=ms, pattern_s=dg.pattern_seconds if first else 0.0, device_s=t1 - t0,
                                total_s=time.perf_counter() - t0)
        _log_throughput(self.name, self.keyword, sd, ms, self.last_timing["total_s"], out)

    def assemble_matrix(self, sd, data: dict) -> sps.csr_matrix:
        """dual_elliptic.py ``assemble_matrix``: [[mass, div^T], [div, 0]]."""
        mats = data[DISCRETIZATION_MATRICES][self.keyword]
        div = mats[self.div_matrix_key]
        return sps.bmat([[mats[self.mass_matrix_key], div.T], [div, None]], format="csr")

    def assemble_neumann_robin(self, sd, data: dict, M, bc_weight: bool = False):
        """dual_elliptic.py ``assemble_neumann_robin``: Neumann rows (not internal) cleared with |mass|_inf on the
        diagonal (1 without ``bc_weight``), 1 / (robin_weight area) added on Robin diagonals."""
        mass = data[DISCRETIZATION_MATRICES][self.keyword][self.mass_matrix_key]
        norm = 1.0
        if mass.shape[0] and bc_weight:
            norm = sps.linalg.norm(mass, np.inf)
        bc = data[PARAMETERS][self.keyword]["bc"]
        internal = np.asarray(bc.is_internal, bool)
        is_neu = np.flatnonzero(np.asarray(bc.is_neu, bool) & ~internal)
        M = sps.csr_matrix(M)
        if is_neu.size:
            for row in is_neu:
                M.data[M.indptr[row]:M.indptr[row + 1]] = 0.0
            d = M.diagonal()
            d[is_neu] = norm
            M.setdiag(d)
        is_rob = np.flatnonzero(np.asarray(bc.is_rob, bool) & ~internal)
        if is_rob.size:
            rob = np.zeros(self.ndof(sd))
            rob[is_rob] = 1.0 / (np.asarray(bc.robin_weight)[is_rob] * sd.face_areas[is_rob])
            M = M + sps.dia_matrix((rob, 0), shape=(rob.size, rob.size))
        return M, norm

    def assemble_rhs(self, sd, data: dict, bc_weight: float = 1.0) -> np.ndarray:
        """dual_elliptic.py ``assemble_rhs``: proj^T vector_source, Dirichlet and Robin terms with the face sign,
        Neumann values times ``bc_weight``."""
        params = data[PARAMETERS][self.keyword]
        proj = data[DISCRETIZATION_MATRICES][self.keyword][self.vector_proj_key]
        rhs = np.zeros(self.ndof(sd))
        if sd.dim == 0:
            return rhs
        bc, bc_val = params["bc"], params["bc_values"]
        assert not bool(bc is None) != bool(bc_val is None)
        vs = params.get("vector_source", np.zeros(proj.shape[0]))
        rhs[:sd.num_faces] += proj.T @ vs
        if bc is None:
            return rhs
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("Periodic boundary conditions are not implemented for DualElliptic")
        internal = np.asarray(bc.is_internal, bool)
        is_neu = np.flatnonzero(np.asarray(bc.is_neu, bool) & ~internal)
        is_dir = np.flatnonzero(np.asarray(bc.is_dir, bool) & ~internal)
        is_rob = np.flatnonzero(np.asarray(bc.is_rob, bool) & ~internal)
        cf = sps.csc_matrix(sd.cell_faces).tocoo()
        sign = np.zeros(sd.num_faces)
        faces, first = np.unique(cf.row, return_index=True)
        sign[faces] = cf.data[first]
        bc_val = np.asarray(bc_val, dtype=np.float64)
        rhs[is_dir] += -sign[is_dir] * bc_val[is_dir]
        rhs[is_rob] += -sign[is_rob] * bc_val[is_rob] / np.asarray(bc.robin_weight)[is_rob]
        rhs[is_neu] = sign[is_neu] * bc_weight * bc_val[is_neu]
        return rhs

    def assemble_matrix_rhs(self, sd, data: dict):
        """dual_elliptic.py ``assemble_matrix_rhs``: the saddle-point matrix (faces first, then cells) with the
        Neumann / Robin rows, and the right-hand side scaled by the same |mass|_inf.  While the stored matrices are
        the device-resident ones of the last ``discretize`` (``LazyCsr`` not yet touched), the system is assembled on
        the GPU from exactly those values (``pb_dual_system``) and ``A`` comes back as a ``LazyCsr`` backed by the
        device system (``A.device_csr``); otherwise the host formulas of the reference."""
        params = data[PARAMETERS][self.keyword]
        dg = self._resident(sd, data)
        if dg is not None and getattr(dg, "h", None) is not None and params.get("bc") is not None:
            bc = params["bc"]
            if getattr(sd, "periodic_face_map", None) is not None:
                raise NotImplementedError("Periodic boundary conditions are not implemented for DualElliptic")
            vs = params.get("vector_source")
            a, rhs, _ = dg.system(dual_bc_codes(sd, bc),
                                  np.broadcast_to(np.asarray(bc.robin_weight, float), (sd.num_faces,)),
                                  sd.face_areas, params["bc_values"], vs)
            return _lazy_system(a), rhs
        M = self.assemble_matrix(sd, data)
        M, norm = self.assemble_neumann_robin(sd, data, M, bc_weight=True)
        return M, self.assemble_rhs(sd, data, norm)

    def _resident(self, sd, data: dict):
        """The ``DualGrid`` whose device values are this keyword's stored matrices (the ``LazyCsr`` of the last
        ``discretize``, untouched by the host), or None."""
        mats = data.get(DISCRETIZATION_MATRICES, {}).get(self.keyword, {})
        dg = getattr(sd, "_b200_dual", None)
        cur = None if dg is None else dg.current
        if (sd.dim > 0 and cur is not None and cur[0] is mats.get(self.mass_matrix_key)
                and cur[1] is mats.get(self.vector_proj_key) and cur[2] is mats.get(self.div_matrix_key)
                and not cur[0].on_host and not cur[1].on_host):
            return dg
        return None

    def solve(self, sd, data: dict, b, tol: float = 1e-10, maxiter: int = 5000, linear_solver=None) -> np.ndarray:
        """[u; p] solving the saddle-point system ``A x = b`` of ``assemble_matrix_rhs`` for any right-hand side ``b``
        (e.g. the returned one with a source added to the cell rows), by hybridization on the device: every cell's
        local system is condensed onto one pressure per face (csrc/dual_hybrid.cuh), the symmetric face system is
        solved by ``linear_solver(H, rhs)`` (default: ``krylov.bicgstab_solver(tol, maxiter)``, Jacobi-preconditioned
        BiCGStab on the ``DeviceCsr`` H), and u and p are recovered cell by cell.  No matrix leaves the device.

        Faces with a given pressure (Dirichlet, and boundary faces without a condition) are fixed in the face system;
        Neumann faces prescribe the flux b_f / |mass|_inf of their saddle-point row; Robin faces keep their
        1 / (robin_weight area) as a local term.  Needs the device-resident discretization (the condition under which
        ``assemble_matrix_rhs`` assembles on the device) and at least one Dirichlet or Robin face, else ``ValueError``.
        ``last_solve``: iterations, relative residual of the face system, kernel times (ms) and wall time (s)."""
        t0 = time.perf_counter()
        params = data[PARAMETERS][self.keyword]
        dg = self._resident(sd, data)
        if dg is None:
            raise ValueError(f"{self.name}.solve needs the device-resident discretization of the last discretize(); "
                             "the stored mass / vector_proj / div matrices were downloaded or replaced")
        bc = params.get("bc")
        if bc is None:
            raise ValueError(f"{self.name}.solve needs boundary conditions (params['bc'])")
        if getattr(sd, "periodic_face_map", None) is not None:
            raise NotImplementedError("Periodic boundary conditions are not implemented for DualElliptic")
        codes = dual_bc_codes(sd, bc)
        one_cell = np.diff(sps.csr_matrix(sd.cell_faces).indptr) == 1
        fixed = (codes == _lib.BC_DIR) | ((codes == _lib.BC_INTERIOR) & one_cell)
        if not fixed.any() and not (codes == _lib.BC_ROB).any():
            raise ValueError(f"{self.name}.solve: no Dirichlet and no Robin face, the pressure is determined only up "
                             "to a constant and the face system is singular")
        b = _lib.f64(b)
        if b.shape != (self.ndof(sd),):
            raise ValueError(f"b must have {self.ndof(sd)} entries")
        rw = np.broadcast_to(np.asarray(bc.robin_weight, float), (sd.num_faces,))
        H, rhs, _, ms_c = dg.hybrid_system(_lib.DUAL_HYBRID_SADDLE, None, codes, rw, sd.face_areas, b)
        if linear_solver is None:
            from .krylov import bicgstab_solver
            linear_solver = bicgstab_solver(tol, maxiter)
        t1 = time.perf_counter()
        lam = _to_host(linear_solver(H, rhs))
        t2 = time.perf_counter()
        up, ms_r = dg.hybrid_recover(_lib.DUAL_HYBRID_SADDLE, None, codes, b, lam)
        info = getattr(linear_solver, "last_info", None) or {}
        res = np.linalg.norm(rhs - _to_host(H @ lam)) / max(np.linalg.norm(rhs), 1e-300)
        self.last_solve = dict(iterations=info.get("iterations"), converged=info.get("converged"),
                               face_residual=float(res), condense_ms=ms_c, recover_ms=ms_r, solve_s=t2 - t1,
                               wall_s=time.perf_counter() - t0, face_unknowns=sd.num_faces, face_nnz=int(H.nnz))
        return up

    def project_flux(self, sd, u: np.ndarray, data: dict) -> np.ndarray:
        """dual_elliptic.py ``project_flux``: one 3-vector per cell, (3, nc)."""
        if sd.dim == 0:
            return np.zeros(3).reshape((3, 1))
        proj = data[DISCRETIZATION_MATRICES][self.keyword][self.vector_proj_key]
        return (proj @ u).reshape((3, -1), order="F")

    def extract_flux(self, sd, solution_array: np.ndarray, data: dict) -> np.ndarray:
        return solution_array[:sd.num_faces]

    def extract_pressure(self, sd, solution_array: np.ndarray, data: dict) -> np.ndarray:
        return solution_array[sd.num_faces:]


class MVEM(_DualElliptic):
    """Lowest-order mixed virtual element method (numerics/vem/mvem.py ``MVEM``)."""

    _method = _lib.DUAL_MVEM

    def __init__(self, keyword: str) -> None:
        super().__init__(keyword, "MVEM")


class RT0(_DualElliptic):
    """Lowest-order Raviart-Thomas element on simplices (numerics/fem/rt0.py ``RT0``)."""

    _method = _lib.DUAL_RT0

    def __init__(self, keyword: str) -> None:
        super().__init__(keyword, "RT0")


class HybridDualVEM:
    """Hybridized mixed virtual element method (numerics/vem/hybrid.py ``HybridDualVEM``): the same constructor,
    ``ndof`` (one pressure per face) and ``matrix_rhs``.  Every cell's MVEM saddle system is condensed onto its face
    pressures on the GPU, one warp per cell (csrc/dual_hybrid.cuh); H comes back as scipy CSR.  The local matrix is
    built as hybrid.py builds it: ``second_order_tensor`` as given (not rotated), the geometry in the frame of
    ``map_geometry.map_grid``, outward normals and unit signs, cell volume and normals scaled by ``aperture``.

    ``compute_up`` restates the reference's formulas on the device, p = S (f - B^T A^-1 C lambda) and
    u = -sgn A^-1 (B p + C lambda), with the parameters ``matrix_rhs`` reads (``second_order_tensor``, ``source``,
    ``aperture`` under ``data["parameters"][keyword]``).  The reference's own ``compute_up`` reads ``data["param"]``
    and calls ``pp.DualVEM``, neither of which exists any more.  Each u_f is taken from the face's first cell (the
    reference keeps the last one; the two agree to the accuracy of lambda).

    Mapping to the saddle-point system of ``MVEM.assemble_matrix_rhs`` (aperture 1, a tensor that needs no rotation):
    Dirichlet faces carry the same pressures bc_values in both; a Neumann value here is the flux per unit area along
    the face normal, u_f = bc_values area, where MVEM prescribes u_f = s bc_values (s: the sign of the face in its
    first cell); and the source f here, the net outflow of a cell, enters MVEM's right-hand side as -f in the cell
    rows (the source convention of the MVEM tutorial)."""

    def __init__(self, keyword: str = "flow") -> None:
        self.keyword = keyword

    def ndof(self, g) -> int:
        return g.num_faces

    def _inputs(self, g, data: dict):
        params = data[PARAMETERS][self.keyword]
        rot = dual_frame(g, data.get("deviation_from_plane_tol", 1e-5))
        geo = [rot @ np.asarray(a, dtype=np.float64) for a in (g.nodes, g.face_normals, g.face_centers,
                                                                g.cell_centers)]
        geo += [g.cell_volumes, np.asarray(params["second_order_tensor"].values, dtype=np.float64), rot,
                np.broadcast_to(np.asarray(params["aperture"], dtype=np.float64), (g.num_cells,))]
        bc = params["bc"]
        codes = np.zeros(g.num_faces, np.uint8)
        if bc is not None:
            codes[np.asarray(bc.is_dir, bool)] = _lib.BC_DIR
            codes[np.asarray(bc.is_neu, bool)] = _lib.BC_NEU
        bc_val = params.get("bc_values")
        bc_val = np.zeros(g.num_faces) if bc_val is None else np.asarray(bc_val, dtype=np.float64)
        f = np.broadcast_to(np.asarray(params["source"], dtype=np.float64), (g.num_cells,))
        return geo, codes, np.concatenate((bc_val, f))

    def matrix_rhs(self, g, data: dict):
        """hybrid.py ``matrix_rhs``: the face matrix H (Dirichlet rows cleared, |H|_inf before the boundary
        conditions on their diagonal) and its right-hand side."""
        if g.dim == 0:
            return sps.identity(self.ndof(g), format="csr"), np.zeros(1)
        t0 = time.perf_counter()
        geo, codes, values = self._inputs(g, data)
        dg = DualGrid.for_grid(g)
        H, rhs, bad, ms = dg.hybrid_system(_lib.DUAL_HYBRID_VEM, geo, codes, np.zeros(g.num_faces), g.face_areas,
                                           values)
        if bad >= 0:   # mvem.py massHdiv: assert np.allclose(G, F @ D)
            raise AssertionError(f"HybridDualVEM: the consistency test G == F D fails in cell {bad}")
        self.last_timing = dict(kernel_ms=ms, total_s=time.perf_counter() - t0)
        return H.to_scipy(), rhs

    def compute_up(self, g, solution, data: dict):
        """u (per face) and p (per cell) from the face pressures ``solution`` (see the class docstring)."""
        if g.dim == 0:
            return 0, solution[0]
        geo, codes, values = self._inputs(g, data)
        up, _ = DualGrid.for_grid(g).hybrid_recover(_lib.DUAL_HYBRID_VEM, geo, codes, values, solution)
        return up[:g.num_faces], up[g.num_faces:]


class Upwind(_Base):
    """First-order upwinding of an advective flux (numerics/fv/upwind.py:13).  ``discretize`` reads
    ``bc`` and the face fluxes under ``flux_array_key`` (default ``"darcy_flux"``) and writes the
    upwind matrix and the two boundary matrices; ``assemble_matrix_rhs`` as upwind.py:57-148."""

    def __init__(self, keyword: str = "transport") -> None:
        super().__init__(keyword)
        self.upwind_matrix_key = "transport"
        self.bound_transport_dir_matrix_key = "rhs_dir"
        self.bound_transport_neu_matrix_key = "rhs_neu"
        self._flux_array_key = "darcy_flux"

    @property
    def flux_array_key(self) -> str:
        return self._flux_array_key

    @flux_array_key.setter
    def flux_array_key(self, value: str) -> None:
        self._flux_array_key = value

    def ndof(self, sd) -> int:
        return sd.num_cells

    def discretize(self, sd, data: dict) -> None:
        params = data[PARAMETERS][self.keyword]
        mats = data.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        bc = params.get("bc")
        if bc is None:  # upwind.py:244-247: Dirichlet on the boundary
            from .params import BoundaryCondition
            bc = BoundaryCondition(sd, sd.get_boundary_faces(), "dir")
        nf, nc = sd.num_faces, sd.num_cells
        ncomp = int(params.get("num_components", 1))
        if nf == 0:  # point grids: upwind.py:226-236
            mats[self.upwind_matrix_key] = sps.csr_matrix((0, nc * ncomp))
            mats[self.bound_transport_neu_matrix_key] = sps.csr_matrix((0, 0))
            mats[self.bound_transport_dir_matrix_key] = sps.csr_matrix((0, 0))
            return
        fg = FaceGrid.for_grid(sd)
        bits = face_bc_bits(bc, nf)
        up, neu, dr = fg.upwind(params[self._flux_array_key], bits)
        # A boundary face that is neither Dirichlet nor Neumann (Robin / unflagged) with inflow has no upstream
        # cell: the reference ends up with column index -1 and scipy raises (upwind.py:272-281).  Fail as loudly.
        single = np.diff(sps.csr_matrix(sd.cell_faces).indptr) == 1
        orphan = single & (up < 0) & ((bits & 12) == 0)
        if orphan.any():
            raise ValueError(f"upwind: boundary face {int(np.flatnonzero(orphan)[0])} has inflow but neither a "
                             "Dirichlet nor a Neumann condition")
        rows = np.flatnonzero(up >= 0)
        m = sps.csr_matrix((np.ones(rows.size), (rows, up[rows])), shape=(nf, nc))
        eye = sps.eye(ncomp)
        mats[self.upwind_matrix_key] = sps.kron(m, eye).tocsr()
        mats[self.bound_transport_neu_matrix_key] = sps.kron(sps.diags(neu), eye).tocsr()
        mats[self.bound_transport_dir_matrix_key] = sps.kron(sps.diags(dr), eye).tocsr()

    def assemble_matrix_rhs(self, sd, data: dict):
        """upwind.py:57-148: ``div @ diag(q) @ upwind`` and the boundary right-hand side."""
        mats = data[DISCRETIZATION_MATRICES][self.keyword]
        params = data[PARAMETERS][self.keyword]
        q = sps.diags(np.asarray(params[self._flux_array_key], float))
        div = sd.divergence(dim=1)
        if div.shape[1] != mats[self.upwind_matrix_key].shape[0]:
            raise ValueError("Dimension mismatch: upwinding with several components is only supported in Ad mode")
        matrix = div @ q @ mats[self.upwind_matrix_key]
        rhs = div @ ((mats[self.bound_transport_neu_matrix_key] + mats[self.bound_transport_dir_matrix_key] @ q)
                     @ params["bc_values"])
        return matrix, rhs


def interface_upwind_masks(interface_flux):
    """(sign, upstream-is-primary, upstream-is-secondary) per mortar cell through ``pb_upwind_coupling`` (one thread per
    entry).  A separate function so that the CPU tests can substitute the host formulas."""
    lam = _lib.f64(interface_flux)
    lib = _lib.load()
    _lib.require_gpu()
    n = int(lam.size)
    sgn, up1, up2 = np.empty(n), np.empty(n), np.empty(n)
    _lib.check(lib.pb_upwind_coupling(n, _lib.ptr(lam, _lib._f64p), _lib.ptr(sgn, _lib._f64p),
                                      _lib.ptr(up1, _lib._f64p), _lib.ptr(up2, _lib._f64p)))
    return sgn, up1, up2


class UpwindCoupling:
    """Upwinding of an advective flux across the interface between a subdomain and a lower-dimensional one
    (numerics/fv/upwind.py:377).  ``discretize`` writes the reference's six matrices to
    ``data_intf["discretization_matrices"][keyword]``; ``assemble_matrix_rhs`` as upwind.py:530-680."""

    def __init__(self, keyword: str) -> None:
        self.keyword = keyword
        self.trace_primary_matrix_key = "trace"
        self.inv_trace_primary_matrix_key = "inv_trace"
        self.upwind_primary_matrix_key = "upwind_primary"
        self.upwind_secondary_matrix_key = "upwind_secondary"
        self.flux_matrix_key = "flux"
        self.mortar_discr_matrix_key = "mortar_discr"
        self._flux_array_key = "darcy_flux"

    def key(self) -> str:
        return self.keyword + "_"

    def discretization_key(self):
        return self.key() + DISCRETIZATION_MATRICES

    @property
    def flux_array_key(self) -> str:
        return self._flux_array_key

    @flux_array_key.setter
    def flux_array_key(self, value: str) -> None:
        self._flux_array_key = value

    def ndof(self, intf) -> int:
        return intf.num_cells

    def discretize(self, sd_primary, sd_secondary, intf, data_primary, data_secondary, data_intf) -> None:
        if sd_primary.dim - sd_secondary.dim not in [1, 2]:
            raise ValueError("Implementation is only valid for grids one dimension apart.")
        mats = data_intf.setdefault(DISCRETIZATION_MATRICES, {}).setdefault(self.keyword, {})
        sgn, up1, up2 = interface_upwind_masks(data_intf[PARAMETERS][self.keyword][self._flux_array_key])
        inv_trace = abs(sd_primary.divergence(dim=1))
        mats[self.inv_trace_primary_matrix_key] = inv_trace
        mats[self.trace_primary_matrix_key] = inv_trace.T
        mats[self.upwind_primary_matrix_key] = sps.diags(up1)
        mats[self.upwind_secondary_matrix_key] = sps.diags(up2)
        mats[self.flux_matrix_key] = sps.diags(sgn)
        mats[self.mortar_discr_matrix_key] = sps.eye(intf.num_cells)

    def assemble_matrix_rhs(self, sd_primary, sd_secondary, intf, data_primary, data_secondary, data_intf, matrix):
        """upwind.py:530-680: the 3 x 3 block contribution of the coupling condition (right-hand side zero)."""
        m = data_intf[DISCRETIZATION_MATRICES][self.keyword]
        dof = np.array([matrix[0, 0].shape[1], matrix[1, 1].shape[1], intf.num_cells])
        cc = np.array([sps.coo_matrix((i, j)) for i in dof for j in dof]).reshape((3, 3))
        lam = np.abs(data_intf[PARAMETERS][self.keyword][self._flux_array_key])
        scaling = sps.dia_matrix((lam, 0), shape=(intf.num_cells, intf.num_cells))
        cc[0, 2] = m[self.inv_trace_primary_matrix_key] @ intf.mortar_to_primary_int()
        cc[1, 2] = -intf.mortar_to_secondary_int()
        cc[2, 0] = (scaling @ m[self.flux_matrix_key] @ m[self.upwind_primary_matrix_key]
                    @ intf.primary_to_mortar_avg() @ m[self.trace_primary_matrix_key])
        cc[2, 1] = scaling @ m[self.flux_matrix_key] @ m[self.upwind_secondary_matrix_key] @ intf.secondary_to_mortar_avg()
        cc[2, 2] = -m[self.mortar_discr_matrix_key]
        if sd_primary == sd_secondary:
            cc = np.array([np.sum(cc, axis=(0, 1))])
        rhs = np.array([np.zeros(dof[0]), np.zeros(dof[1]), np.zeros(dof[2])], dtype=object)
        if rhs.ndim == 2:
            rhs = rhs.ravel()
        matrix += cc
        return matrix, rhs
