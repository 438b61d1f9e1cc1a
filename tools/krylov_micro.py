"""Where a fused BiCGStab iteration spends its time (one GPU, bench-size flow system): the SpMV at its
autotuned lanes per row, the three vector kernels, the SpMV with dot-product epilogue, one graph-replayed block.   python tools/krylov_micro.py"""
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import porepy_b200 as pb  # noqa: E402
from porepy_b200 import _lib  # noqa: E402
from porepy_b200 import krylov as kr  # noqa: E402

lib = _lib.load()
w = sys.argv[1] if len(sys.argv) > 1 else "tet1m"
kind, dims, _ = bench.WORKLOADS[w]
g = bench.make_grid(kind, dims)
k, bc, C4, vbc = bench.make_params(g)
bv = np.zeros(g.num_faces)
bf = g.get_all_boundary_faces()
bv[bf[g.face_centers[0, bf] < 1e-10]] = 1.0
d = pb.initialize_data({}, "flow", {"second_order_tensor": k, "bc": bc, "bc_values": bv})
m = pb.Mpfa("flow")
m.discretize(g, d)
A, b = m.assemble_matrix_rhs(g, d)
a_dev = A.device_csr
host = a_dev.to_scipy()
print("rows", host.shape[0], "nnz", host.nnz, "autotuned lanes per row", lib.pb_csr_lanes_per_row(a_dev.h), flush=True)

n = host.shape[0]
dev = torch.device("cuda")
vec = lambda: torch.randn(n, dtype=torch.float64, device=dev)  # noqa: E731
x, r, rhat, p, v, s, t, ph, sh = (vec() for _ in range(9))
minv = torch.rand(n, dtype=torch.float64, device=dev) + 0.5
scal = torch.ones(14, dtype=torch.float64, device=dev)
scal[11] = 0.0   # not DONE
scal[13] = 0.0   # tol^2 = 0: never frozen
P = lambda a: C.c_void_p(a.data_ptr())  # noqa: E731
S = lambda i: C.c_void_p(scal.data_ptr() + 8 * i)  # noqa: E731
st = torch.cuda.current_stream().cuda_stream


def timed(name, fn, reps=100):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    print(f"{name:28s} {e0.elapsed_time(e1) / reps:.4f} ms", flush=True)


def reset():
    scal.fill_(1.0)
    scal[11] = 0.0
    scal[13] = 0.0


timed("kry_p (Jacobi)", lambda: (reset(), lib.pb_kry_p(n, P(r), P(p), P(v), P(minv), P(ph), P(scal), 0, 1, st)))
timed("kry_s (Jacobi)", lambda: (reset(), lib.pb_kry_s(n, P(r), P(v), P(minv), P(s), P(sh), P(scal), 0, 1, st)))
timed("kry_xr", lambda: (reset(), lib.pb_kry_xr(n, P(x), P(ph), P(sh), P(s), P(t), P(r), P(rhat), P(scal), 0, 1, st)))
timed("reset only (2 tiny torch ops)", reset)
timed("spmv", lambda: lib.pb_csr_spmv_dev(a_dev.h, P(ph), P(v), st))
timed("spmv + 1 dot", lambda: lib.pb_csr_spmv_dots_dev(a_dev.h, P(ph), P(v), P(rhat), S(0), None, None, st))
timed("spmv + 2 dots", lambda: lib.pb_csr_spmv_dots_dev(a_dev.h, P(sh), P(t), P(s), S(1), None, S(2), st))
# a full solve, graph and plain launches
loc = kr.LocalSystem(0, 1, np.arange(n), np.zeros(0, np.int64), a_dev, [0], [np.zeros(0, np.int64)])
diag = torch.as_tensor(a_dev.diagonal(), device=dev)
for graph in ("1", "0"):
    os.environ["POREB200_KRYLOV_GRAPH"] = graph
    for rep in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xs, info = kr.solve_local(loc, b, diag_own=diag, tol=1e-8, maxiter=3000)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    print(f"solve graph={graph}: {dt:.4f} s  {info['iterations']} it  {1e3 * dt / info['iterations']:.3f} ms/it  "
          f"host syncs {info['host_syncs']}  converged {info['converged']}", flush=True)
