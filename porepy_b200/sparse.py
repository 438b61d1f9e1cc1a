"""Device-resident CSR matrix with the SpMV the Newton residual / Krylov loop needs.

Replaces the scipy ``M @ val`` of ``AdArray.__rmatmul__`` (reference
src/porepy/numerics/ad/forward_mode.py:565-595) for matrices kept in HBM."""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sps

from . import _lib


def device_operand(t, n: int, what: str):
    """``t`` if the library may read it through ``t.data_ptr()``: a contiguous float64 CUDA tensor of ``n`` elements.
    A view (strided, expanded), another dtype or a host tensor would be read as if it were that, so it is refused."""
    import torch
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float64 and t.is_contiguous()):
        raise TypeError(f"{what}: a contiguous float64 CUDA tensor is required")
    if t.numel() != n:
        raise ValueError("dimension mismatch")
    return t


class DeviceCsr:
    def __init__(self, a):
        lib = _lib.load()
        _lib.require_gpu()
        a = sps.csr_matrix(a)
        a.sort_indices()
        if a.nnz >= 2**31:
            raise ValueError("matrix too large for int32 indices")
        self.shape = a.shape
        self.nnz = int(a.nnz)
        ip = a.indptr.astype(np.int32)
        ix = a.indices.astype(np.int32)
        da = np.ascontiguousarray(a.data, np.float64)
        h = C.c_void_p()
        _lib.check(lib.pb_csr_create(a.shape[0], a.shape[1], a.nnz, _lib.ptr(ip, _lib._i32p),
                                     _lib.ptr(ix, _lib._i32p), _lib.ptr(da, _lib._f64p), C.byref(h)))
        self.h = h
        self.lib = lib

    @classmethod
    def from_handle(cls, h) -> "DeviceCsr":
        """Wrap a matrix that was assembled on the device (e.g. ``DevicePlan.mpfa_system``)."""
        lib = _lib.load()
        self = cls.__new__(cls)
        nr, ncl, nz = C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(lib.pb_csr_shape(h, C.byref(nr), C.byref(ncl), C.byref(nz)))
        self.shape, self.nnz, self.h, self.lib = (nr.value, ncl.value), nz.value, h, lib
        return self

    def truncate_rows(self, nrows: int) -> "DeviceCsr":
        """Keep the first ``nrows`` rows (in place; the own rows of a shard's system come first)."""
        _lib.check(self.lib.pb_csr_truncate_rows(self.h, int(nrows)))
        self.shape = (int(nrows), self.shape[1])
        return self

    def diagonal(self) -> np.ndarray:
        d = np.empty(min(self.shape))
        _lib.check(self.lib.pb_csr_diagonal(self.h, _lib.ptr(d, _lib._f64p)))
        return d

    def block_diagonal_inverse(self, bs: int, nblocks: int | None = None, stream: int = 0):
        """Inverses of the first ``nblocks`` bs x bs diagonal blocks (default: all), as a flat torch CUDA tensor of
        nblocks*bs*bs doubles (row-major blocks): the block-Jacobi preconditioner of ``krylov.bicgstab``."""
        import torch
        nb = min(self.shape) // bs if nblocks is None else int(nblocks)
        out = torch.empty(nb * bs * bs, dtype=torch.float64, device="cuda")
        _lib.check(self.lib.pb_csr_block_diag_inv_dev(self.h, int(bs), nb, C.c_void_p(out.data_ptr()),
                                                      stream or torch.cuda.current_stream().cuda_stream))
        return out

    def checksum(self):
        """(sum, sum of squares) of the stored values: a device reduction."""
        a, b = C.c_double(), C.c_double()
        _lib.check(self.lib.pb_csr_checksum(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def to_scipy(self) -> sps.csr_matrix:
        ip = np.empty(self.shape[0] + 1, np.int32)
        ix = np.empty(max(self.nnz, 1), np.int32)
        da = np.empty(max(self.nnz, 1), np.float64)
        _lib.check(self.lib.pb_csr_download(self.h, _lib.ptr(ip, _lib._i32p), _lib.ptr(ix, _lib._i32p),
                                            _lib.ptr(da, _lib._f64p)))
        nnz = int(ip[-1])   # after truncate_rows the row-pointer prefix addresses fewer entries
        return sps.csr_matrix((da[:nnz], ix[:nnz], ip), shape=self.shape)

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            try:
                self.lib.pb_csr_destroy(h)
            except Exception:
                pass
            self.h = None

    # ---- device-side sparse algebra (csrc/sparse_ops.cu): the operations of the AD Jacobian chain
    @staticmethod
    def _new(lib, h) -> "DeviceCsr":
        return DeviceCsr.from_handle(h)

    def matmul(self, other: "DeviceCsr") -> "DeviceCsr":
        """C = A @ B (SpGEMM on the device; ``M @ jac`` of forward_mode.py:565-595)."""
        h = C.c_void_p()
        _lib.check(self.lib.pb_csr_spgemm(self.h, other.h, C.byref(h)))
        return DeviceCsr.from_handle(h)

    def axpby(self, alpha: float, other: "DeviceCsr", beta: float) -> "DeviceCsr":
        """alpha * self + beta * other on the union pattern."""
        h = C.c_void_p()
        _lib.check(self.lib.pb_csr_axpby(float(alpha), self.h, float(beta), other.h, C.byref(h)))
        return DeviceCsr.from_handle(h)

    def scaled(self, d, by_cols: bool = False) -> "DeviceCsr":
        """diag(d) @ self (``_diagvec_mul_jac``, forward_mode.py:613-616) or self @ diag(d); ``d``: contiguous float64
        CUDA tensor."""
        d = device_operand(d, self.shape[1 if by_cols else 0], "DeviceCsr.scaled")
        h = C.c_void_p()
        _lib.check(self.lib.pb_csr_scale_dev(self.h, C.c_void_p(d.data_ptr()), int(by_cols), C.byref(h)))
        return DeviceCsr.from_handle(h)

    @staticmethod
    def bmat(blocks) -> "DeviceCsr":
        """Block matrix from a 2-D list of ``DeviceCsr`` / ``None`` (zero blocks); every block row / column needs at
        least one matrix to fix its size."""
        lib = _lib.load()
        nbr, nbc = len(blocks), len(blocks[0])
        rs, cs = [None] * nbr, [None] * nbc
        for i, row in enumerate(blocks):
            if len(row) != nbc:
                raise ValueError("ragged block list")
            for j, b in enumerate(row):
                if b is not None:
                    if rs[i] not in (None, b.shape[0]) or cs[j] not in (None, b.shape[1]):
                        raise ValueError("block shape mismatch")
                    rs[i], cs[j] = b.shape[0], b.shape[1]
        if None in rs or None in cs:
            raise ValueError("a block row / column holds only zero blocks")
        arr = (C.c_void_p * (nbr * nbc))(*[None if b is None else b.h for row in blocks for b in row])
        rsz = np.asarray(rs, dtype=np.int64)
        csz = np.asarray(cs, dtype=np.int64)
        h = C.c_void_p()
        _lib.check(lib.pb_csr_bmat(nbr, nbc, arr, _lib.ptr(rsz, _lib._i64p), _lib.ptr(csz, _lib._i64p), C.byref(h)))
        return DeviceCsr.from_handle(h)

    @staticmethod
    def block_diag(mats) -> "DeviceCsr":
        """``MergedOperator.parse``'s concatenation of per-subdomain matrices (ad_utils.py:650-664)."""
        n = len(mats)
        return DeviceCsr.bmat([[mats[i] if i == j else None for j in range(n)] for i in range(n)])

    @staticmethod
    def vstack(mats) -> "DeviceCsr":
        """``EquationSystem.assemble``'s stacking of the equation blocks (equation_system.py:1695-1713)."""
        return DeviceCsr.bmat([[m] for m in mats])

    @staticmethod
    def hstack(mats) -> "DeviceCsr":
        return DeviceCsr.bmat([list(mats)])

    @staticmethod
    def identity(n: int) -> "DeviceCsr":
        return DeviceCsr(sps.identity(n, format="csr"))

    def __add__(self, other):
        return self.axpby(1.0, other, 1.0) if isinstance(other, DeviceCsr) else NotImplemented

    def __sub__(self, other):
        return self.axpby(1.0, other, -1.0) if isinstance(other, DeviceCsr) else NotImplemented

    def __neg__(self):
        return self.axpby(-1.0, self, 0.0)

    def __mul__(self, a):
        if isinstance(a, (int, float, np.floating, np.integer)):
            return self.axpby(float(a), self, 0.0)
        return NotImplemented

    __rmul__ = __mul__

    def __matmul__(self, x):
        if isinstance(x, DeviceCsr):
            return self.matmul(x)
        if hasattr(x, "__rmatmul__") and type(x).__name__ == "DeviceAdArray":
            return x.__rmatmul__(self)
        if hasattr(x, "data_ptr"):       # CUDA tensor: y = A x on the device (a strided view is copied first)
            import torch
            x = device_operand(x.contiguous() if torch.is_tensor(x) else x, self.shape[1], "DeviceCsr @ tensor")
            if self.shape[0] == 0 or self.shape[1] == 0:
                return torch.zeros(self.shape[0], dtype=torch.float64, device=x.device)
            y = torch.empty(self.shape[0], dtype=torch.float64, device=x.device)
            self.spmv_device(x.data_ptr(), y.data_ptr(), torch.cuda.current_stream().cuda_stream)
            return y
        x = _lib.f64(x)
        if x.shape != (self.shape[1],):
            raise ValueError("dimension mismatch")
        y = np.empty(self.shape[0])
        _lib.check(self.lib.pb_csr_spmv(self.h, _lib.ptr(x, _lib._f64p), _lib.ptr(y, _lib._f64p)))
        return y

    def spmv_device(self, x_ptr: int, y_ptr: int, stream: int = 0) -> None:
        """y = A x on raw device pointers (e.g. ``torch.Tensor.data_ptr()``)."""
        _lib.check(self.lib.pb_csr_spmv_dev(self.h, C.c_void_p(x_ptr), C.c_void_p(y_ptr), stream))

    def bench(self, reps: int = 50) -> float:
        """Mean device milliseconds per SpMV (CUDA events on the launching stream)."""
        ms = C.c_float()
        _lib.check(self.lib.pb_csr_spmv_bench(self.h, reps, C.byref(ms)))
        return float(ms.value)

    def algorithmic_bytes(self) -> int:
        """12 B per non-zero + 20 B per row (SURVEY.md §8d)."""
        return 12 * self.nnz + 20 * self.shape[0]


# ------------------------------------------------------------------------------------------
# device-resident discretization matrices behind the scipy interface
# ------------------------------------------------------------------------------------------


class DeviceValues:
    """Value array of one output matrix, detached from the plan and kept in HBM (``pb_values``)."""

    def __init__(self, h, lib):
        self.h, self.lib = h, lib
        self.size = int(lib.pb_values_size(h))

    def download(self) -> np.ndarray:
        out = _lib.pinned_empty(self.size)
        _lib.check(self.lib.pb_values_download(self.h, _lib.ptr(out, _lib._f64p)))
        return out

    def checksum(self):
        s, q = C.c_double(), C.c_double()
        _lib.check(self.lib.pb_values_checksum(self.h, C.byref(s), C.byref(q)))
        return s.value, q.value

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            try:
                self.lib.pb_values_destroy(h)
            except Exception:
                pass
            self.h = None


def _lazy_field(name):
    slot, loader = "_lazy_" + name, "_load_" + name

    def get(self):
        d = self.__dict__
        v = d.get(slot)
        if v is None:
            ld = d.get(loader)
            if ld is None:
                raise AttributeError(name)
            v = ld()
            d[slot] = v
            d[loader] = None
            LazyCsr.downloads[name] += int(getattr(v, "nbytes", 0))
        return v

    def put(self, v):
        self.__dict__[slot] = v
        self.__dict__[loader] = None
    return property(get, put)


class LazyCsr(sps.csr_matrix):
    """A ``scipy.sparse.csr_matrix`` whose ``data`` / ``indices`` / ``indptr`` arrays are fetched from the device on
    first touch.  ``discretize()`` stores these in ``data[pp.DISCRETIZATION_MATRICES]``: the drop-in contract of the
    reference (scipy-sparse outputs: ``.shape``, ``@``, slicing, ``sps.block_diag`` ... -- it IS a ``csr_matrix``) is
    kept, but only the matrices a caller actually uses cross PCIe, and ``assemble_matrix_rhs`` of the same classes
    builds the system from the device copies without any download.  ``LazyCsr.downloads`` counts the bytes fetched."""

    downloads = {"data": 0, "indices": 0, "indptr": 0}
    data = _lazy_field("data")
    indices = _lazy_field("indices")
    indptr = _lazy_field("indptr")

    @classmethod
    def lazy(cls, shape, nnz, load_data, load_indices, load_indptr, device_values=None, device_csr=None, plan=None):
        zero = np.broadcast_to(np.float64(0.0), (0,))
        self = cls((zero, np.zeros(0, np.int32), np.zeros(int(shape[0]) + 1, np.int32)), shape=shape, copy=False)
        d = self.__dict__
        d["_lazy_data"] = d["_lazy_indices"] = d["_lazy_indptr"] = None
        d["_load_data"], d["_load_indices"], d["_load_indptr"] = load_data, load_indices, load_indptr
        d["_structural_nnz"] = int(nnz)
        d["device_values"], d["device_csr"], d["plan"] = device_values, device_csr, plan
        d["pattern_key"] = None
        self.has_sorted_indices = True
        self.has_canonical_format = True
        return self

    @property
    def on_host(self) -> bool:
        """True once the values have been downloaded (or the matrix was built from host arrays)."""
        return self.__dict__.get("_lazy_data") is not None

    @property
    def dtype(self):
        return np.dtype(np.float64) if not self.on_host else self.data.dtype

    @property
    def nnz(self):
        n = self.__dict__.get("_structural_nnz")
        return n if (n is not None and self.__dict__.get("_lazy_indptr") is None) else int(self.indptr[-1])

    def _getnnz(self, axis=None):
        if axis is None:
            return self.nnz
        return super()._getnnz(axis)

    def getnnz(self, axis=None):
        return self._getnnz(axis)

    def __repr__(self):
        where = "host" if self.on_host else "device"
        return f"<{self.shape[0]}x{self.shape[1]} LazyCsr, {self.nnz} stored elements, values on the {where}>"


def materialize(obj):
    """Force every ``LazyCsr`` in a matrix dictionary (or a single matrix) to the host; returns the bytes fetched."""
    before = sum(LazyCsr.downloads.values())
    if isinstance(obj, dict):
        for v in obj.values():
            materialize(v)
    elif isinstance(obj, LazyCsr):
        obj.data, obj.indices, obj.indptr  # noqa: B018  (property access triggers the download)
    return sum(LazyCsr.downloads.values()) - before
