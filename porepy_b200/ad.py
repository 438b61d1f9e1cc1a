"""Forward-mode AD on the device: the Jacobian chain of PorePy's operator evaluation with values and Jacobians
that never leave HBM (SURVEY.md 8a rows a21-a23, 8f rank 2).

Mirrors, on ``DeviceCsr`` matrices and CUDA vectors, what the reference does with scipy on the host at every operator
evaluation:

* ``AdArray``                      numerics/ad/forward_mode.py:25   -> ``DeviceAdArray`` (``val``: CUDA float64 tensor,
  ``jac``: ``DeviceCsr``); ``__rmatmul__`` = SpMV + SpGEMM (:565-595), elementwise products through
  ``_diagvec_mul_jac`` (:613-616), sums, negation, scalar factors
* ``initAdArrays``                 numerics/ad/forward_mode.py      -> ``variables``: identity blocks of the global dof
* ``MergedOperator.parse``         numerics/ad/ad_utils.py:597-664  -> ``merged``: block-diagonal concatenation of the
  per-subdomain discretization matrices, taken straight from the device-resident ``LazyCsr`` outputs of ``discretize``
* ``EquationSystem.assemble``      numerics/ad/equation_system.py:1579-1713 -> ``assemble``: vstack of the equation
  blocks, global Jacobian and right-hand side ``-residual``

torch is plumbing here (device vectors and their elementwise kernels); the sparse kernels are csrc/sparse_ops.cu.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps

from .sparse import DeviceCsr, LazyCsr


def as_device_csr(m) -> DeviceCsr:
    """``DeviceCsr`` view of a matrix: device-resident discretization outputs and systems are used where they are
    (no host round trip); host scipy matrices (divergence, projections, ...) are uploaded."""
    if isinstance(m, DeviceCsr):
        return m
    if isinstance(m, LazyCsr) and not m.on_host:
        if m.device_csr is not None:
            return m.device_csr
        if m.device_values is not None and m.plan is not None and m.__dict__.get("pattern_key") is not None:
            return m.plan.output_csr(m.device_values, *m.pattern_key)
    return DeviceCsr(sps.csr_matrix(m))


def device_vector(v, device=None):
    """``v`` as a contiguous float64 CUDA tensor (the kernels read it through its data pointer): views, other dtypes
    and host tensors are copied."""
    import torch
    if torch.is_tensor(v):
        dev = device or (v.device if v.is_cuda else torch.device("cuda", torch.cuda.current_device()))
        return v.to(device=dev, dtype=torch.float64).contiguous()
    dev = device or torch.device("cuda", torch.cuda.current_device())
    return torch.as_tensor(np.ascontiguousarray(v, dtype=np.float64), device=dev)


class DeviceAdArray:
    """Value + Jacobian pair on the device (``AdArray``, numerics/ad/forward_mode.py:25)."""

    def __init__(self, val, jac: DeviceCsr):
        self.val = device_vector(val)
        self.jac = jac
        if jac.shape[0] != self.val.numel():
            raise ValueError("value and Jacobian have different numbers of rows")

    # ---- linear combinations
    def __add__(self, other):
        if isinstance(other, DeviceAdArray):
            return DeviceAdArray(self.val + other.val, self.jac.axpby(1.0, other.jac, 1.0))
        return DeviceAdArray(self.val + _plain(other, self.val), self.jac)

    __radd__ = __add__

    def __sub__(self, other):
        if isinstance(other, DeviceAdArray):
            return DeviceAdArray(self.val - other.val, self.jac.axpby(1.0, other.jac, -1.0))
        return DeviceAdArray(self.val - _plain(other, self.val), self.jac)

    def __rsub__(self, other):
        return (-self) + other

    def __neg__(self):
        return DeviceAdArray(-self.val, -self.jac)

    # ---- products (forward_mode.py:__mul__: scalars, arrays elementwise, AdArrays by the product rule)
    def __mul__(self, other):
        if isinstance(other, DeviceAdArray):
            jac = self.jac.scaled(other.val).axpby(1.0, other.jac.scaled(self.val), 1.0)
            return DeviceAdArray(self.val * other.val, jac)
        if isinstance(other, (int, float, np.floating, np.integer)):
            return DeviceAdArray(self.val * float(other), self.jac * float(other))
        d = _plain(other, self.val)
        return DeviceAdArray(self.val * d, self.jac.scaled(d))

    __rmul__ = __mul__

    def __truediv__(self, other):
        if isinstance(other, (int, float, np.floating, np.integer)):
            return self * (1.0 / float(other))
        if isinstance(other, DeviceAdArray):
            inv = 1.0 / other.val
            return self * DeviceAdArray(inv, other.jac.scaled(-inv * inv))
        return self * (1.0 / _plain(other, self.val))

    def __rmatmul__(self, matrix):
        """``matrix @ self``: SpMV of the value and SpGEMM of the Jacobian (forward_mode.py:565-595)."""
        m = as_device_csr(matrix)
        if m.shape[1] != self.jac.shape[0]:
            raise ValueError("Dimension mismatch between sparse matrix and AdArray during matrix multiplication.")
        return DeviceAdArray(m @ self.val, m.matmul(self.jac))

    def exp(self):
        e = self.val.exp()
        return DeviceAdArray(e, self.jac.scaled(e))

    def reciprocal(self):
        """``1 / self`` (the ``one / x`` of the reference's harmonic means, constitutive_laws.py:1567-1581)."""
        inv = 1.0 / self.val
        return DeviceAdArray(inv, self.jac.scaled(-inv * inv))

    def __rtruediv__(self, other):
        return self.reciprocal() * other

    def host(self):
        """(val, jac) as NumPy / scipy (tests)."""
        return self.val.cpu().numpy(), self.jac.to_scipy()


def _plain(other, like):
    import torch
    if isinstance(other, (int, float, np.floating, np.integer)):
        return float(other)
    if torch.is_tensor(other):          # views and other dtypes: ``scaled`` reads a contiguous float64 buffer
        return other.to(device=like.device, dtype=torch.float64).contiguous()
    return torch.as_tensor(np.asarray(other, dtype=np.float64), device=like.device)


def variables(values) -> list:
    """One ``DeviceAdArray`` per variable block with the identity in its own columns of the global dof numbering
    (``initAdArrays``)."""
    sizes = [int(np.asarray(v).size) if not hasattr(v, "numel") else int(v.numel()) for v in values]
    eyes = [DeviceCsr.identity(n) for n in sizes]
    zero = {}

    def zeros(r, c):
        if (r, c) not in zero:
            zero[(r, c)] = DeviceCsr(sps.csr_matrix((r, c)))
        return zero[(r, c)]
    out = []
    for i, v in enumerate(values):
        row = [eyes[i] if j == i else zeros(sizes[i], sizes[j]) for j in range(len(values))]
        out.append(DeviceAdArray(v, DeviceCsr.hstack(row)))
    return out


def merged(matrices) -> DeviceCsr:
    """``MergedOperator.parse`` (ad_utils.py:597-664): the block-diagonal concatenation of one discretization matrix per
    subdomain, built on the device from device-resident operands."""
    mats = [as_device_csr(m) for m in matrices]
    return mats[0] if len(mats) == 1 else DeviceCsr.block_diag(mats)


def assemble(equations):
    """``EquationSystem.assemble`` (equation_system.py:1579-1713): stack the equation blocks; returns the global
    Jacobian (``DeviceCsr``) and the right-hand side ``-residual`` (CUDA tensor)."""
    import torch
    jac = equations[0].jac if len(equations) == 1 else DeviceCsr.vstack([e.jac for e in equations])
    return jac, -torch.cat([e.val for e in equations])
