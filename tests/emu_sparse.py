"""Host stand-in for ``porepy_b200.sparse.DeviceCsr`` (scipy + CPU torch tensors) with the same interface, so that the
AD chain of ``porepy_b200.ad`` and the equation builders on top of it (``porepy_b200.mdflow``) run in the build container.
Test infrastructure only: the product never imports it."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps
import torch


class HostCsr:
    def __init__(self, a):
        self.m = sps.csr_matrix(a, dtype=np.float64)
        self.m.sort_indices()
        self.shape = self.m.shape

    @property
    def nnz(self):
        return int(self.m.nnz)

    def to_scipy(self):
        return self.m.copy()

    def diagonal(self):
        return self.m.diagonal()

    def matmul(self, other):
        if not isinstance(other, HostCsr) or other.shape[0] != self.shape[1]:
            raise ValueError("matmul: inner dimensions differ")
        return HostCsr(self.m @ other.m)

    def axpby(self, alpha, other, beta):
        if not isinstance(other, HostCsr) or other.shape != self.shape:
            raise ValueError("axpby: operands must be matrices of the same shape")      # pb_csr_axpby refuses as well
        return HostCsr(float(alpha) * self.m + float(beta) * other.m)

    def scaled(self, d, by_cols=False):
        # the device routine reads ``d.data_ptr()``: a contiguous float64 torch tensor of the right length, nothing else
        if not (torch.is_tensor(d) and d.dtype == torch.float64 and d.is_contiguous()):
            raise TypeError("scaled: a contiguous float64 tensor is required (DeviceCsr.scaled takes its data_ptr)")
        if d.numel() != self.shape[1 if by_cols else 0]:
            raise ValueError("dimension mismatch")
        d = d.cpu().numpy()
        return HostCsr(self.m @ sps.diags(d) if by_cols else sps.diags(d) @ self.m)

    @staticmethod
    def bmat(blocks):
        # same argument checks as DeviceCsr.bmat (porepy_b200/sparse.py)
        nbr, nbc = len(blocks), len(blocks[0])
        rs, cs = [None] * nbr, [None] * nbc
        for i, row in enumerate(blocks):
            if len(row) != nbc:
                raise ValueError("ragged block list")
            for j, b in enumerate(row):
                if b is not None:
                    if not isinstance(b, HostCsr):
                        raise TypeError("bmat: blocks must be device matrices or None")
                    if rs[i] not in (None, b.shape[0]) or cs[j] not in (None, b.shape[1]):
                        raise ValueError("block shape mismatch")
                    rs[i], cs[j] = b.shape[0], b.shape[1]
        if None in rs or None in cs:
            raise ValueError("a block row / column holds only zero blocks")
        return HostCsr(sps.bmat([[None if b is None else b.m for b in row] for row in blocks], format="csr"))

    @staticmethod
    def block_diag(mats):
        return HostCsr(sps.block_diag([m.m for m in mats], format="csr"))

    @staticmethod
    def vstack(mats):
        return HostCsr(sps.vstack([m.m for m in mats], format="csr"))

    @staticmethod
    def hstack(mats):
        return HostCsr(sps.hstack([m.m for m in mats], format="csr"))

    @staticmethod
    def identity(n):
        return HostCsr(sps.identity(n, format="csr"))

    def __add__(self, o):
        return self.axpby(1.0, o, 1.0) if isinstance(o, HostCsr) else NotImplemented

    def __sub__(self, o):
        return self.axpby(1.0, o, -1.0) if isinstance(o, HostCsr) else NotImplemented

    def __neg__(self):
        return HostCsr(-self.m)

    def __mul__(self, a):
        if isinstance(a, (int, float, np.floating, np.integer)):
            return HostCsr(float(a) * self.m)
        return NotImplemented

    __rmul__ = __mul__

    def __matmul__(self, x):
        if isinstance(x, HostCsr):
            return self.matmul(x)
        if type(x).__name__ == "DeviceAdArray":
            return x.__rmatmul__(self)
        if torch.is_tensor(x):
            # DeviceCsr @ tensor copies a strided view, but refuses what the kernel cannot read as float64
            if x.dtype != torch.float64:
                raise TypeError("a float64 tensor is required")
            if x.numel() != self.shape[1]:
                raise ValueError("dimension mismatch")
            return torch.as_tensor(self.m @ x.cpu().numpy())
        x = np.asarray(x, float)
        if x.shape != (self.shape[1],):
            raise ValueError("dimension mismatch")
        return self.m @ x


def install(monkeypatch):
    """Route ``porepy_b200.ad`` to the host stand-in."""
    from porepy_b200 import ad

    def as_csr(m):
        if isinstance(m, HostCsr):
            return m
        return HostCsr(sps.csr_matrix(m))

    def vec(v, device=None):
        return v.to(dtype=torch.float64) if torch.is_tensor(v) else torch.as_tensor(np.ascontiguousarray(v, dtype=np.float64))
    monkeypatch.setattr(ad, "DeviceCsr", HostCsr)
    monkeypatch.setattr(ad, "as_device_csr", as_csr)
    monkeypatch.setattr(ad, "device_vector", vec)


def _bench(self, reps=1):
    return 1.0


def _algorithmic_bytes(self):
    return 12 * self.nnz + 20 * self.shape[0]


HostCsr.bench = _bench
HostCsr.algorithmic_bytes = _algorithmic_bytes
