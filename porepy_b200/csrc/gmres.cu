// gmres.cu -- restarted GMRES(m), right-preconditioned by a grouped block-Jacobi: the device solver of the Newton updates
// of the fractured contact models (contact.py, fractured_poromech.py, fractured_thm.py), whose Jacobians have zero
// diagonals in the complementarity and force-balance rows.  BiCGStab breaks down on several of them; GMRES with the
// grouped preconditioner does not.
//
// Preconditioner.  Groups g = (R_g, C_g) of rows and columns, |R_g| = |C_g| = s_g <= 32, that partition all rows and all
// columns; M^-1 y is z[C_g] = J[R_g, C_g]^-1 y[R_g].  group_inv_kernel gathers and inverts one block per warp
// (group_block.cuh, shared with the host build in tests/emu); group_apply_kernel runs one thread per output entry.
//
// GMRES.  Right preconditioning, so the minimised residual is the true |b - A x|.  Arnoldi step j (V_{j+1} is the work
// vector w):  z = M^-1 V_j;  w = A z (pb_csr_spmv_dev);  h = V^T w (one pass over the j+1 basis vectors);  w -= V h
// fused with the dots of the second classical Gram-Schmidt pass;  w -= V h2 fused with |w|^2;  one warp applies the
// Givens rotations and updates the residual estimate |g_{j+1}|;  V_{j+1} = w / h_{j+1,j}.  Every reduction writes
// per-block partials that one kernel sums in a fixed order (no floating-point atomics), so two solves of the same
// system are bit-identical.  All scalars (Hessenberg matrix, rotations, g, y) live in a device buffer; the DONE flag is
// sticky within a cycle and turns the remaining steps into no-ops, so a whole cycle of m steps can be captured once as
// a CUDA graph and replayed.  The cycle end solves the small triangular system, adds M^-1 (V y) to x (one extra apply
// instead of storing Z) and recomputes the true residual b - A x, which starts the next cycle; the host reads the scalar
// buffer once per cycle and decides on that true residual.
#include "plan.hpp"
#include "group_block.cuh"

#include <climits>

#define GM_BB 0      // |b|^2
#define GM_DONE 1    // sticky within a cycle
#define GM_STEPS 2   // Arnoldi steps of the current cycle
#define GM_TOLB 3    // tol |b|
#define GM_RES2 4    // |b - A x|^2 at the last cycle end
#define GM_BETA 5    // |r| at the start of the cycle
#define GM_LUCKY 6   // an invariant Krylov subspace was reached (h_{j+1,j} = 0 to round-off)
#define GM_BAD 7     // a singular Hessenberg column or a value that is not finite
#define GM_EST 8     // |g_{j+1}|: residual estimate of the current cycle
#define GM_TOTAL 9   // Arnoldi steps of all cycles
#define GM_HDR 16
#define GM_MAX_RESTART 128
#define GM_THREADS 256

namespace {

struct GmLayout {   // offsets in the scalar buffer
    int m;
    __host__ __device__ int h(int i, int j) const { return GM_HDR + j * (m + 1) + i; }   // H[i][j], m + 1 rows
    __host__ __device__ int cs() const { return GM_HDR + m * (m + 1); }
    __host__ __device__ int sn() const { return cs() + m; }
    __host__ __device__ int g() const { return sn() + m; }        // m + 1
    __host__ __device__ int y() const { return g() + m + 1; }     // m
    __host__ __device__ int red() const { return y() + m; }       // m + 2: the last reduction
    __host__ __device__ int size() const { return red() + m + 2; }
};

// deterministic block sum (fixed shuffle tree, then warp 0 over the warp sums); the result is valid in thread 0
__device__ double block_sum(double v) {
    __shared__ double part[GM_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) part[w] = v;
    __syncthreads();
    v = 0.0;
    if (w == 0) {
        v = lane < (int)(blockDim.x >> 5) ? part[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    return v;
}

// partial[b][i] = sum over this block's rows of V_i . w   (i < cnt)
__device__ void block_dots(int64_t n, const double *__restrict__ V, int cnt, const double *__restrict__ w,
                           double *__restrict__ partial, int stride) {
    for (int i = 0; i < cnt; ++i) {
        const double *vi = V + (int64_t)i * n;
        double acc = 0.0;
        for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
            acc += vi[r] * w[r];
        acc = block_sum(acc);
        if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * stride + i] = acc;
    }
}

// ---------------------------------------------------------------- grouped block-Jacobi
constexpr int kInvWarps = 4;

__global__ void group_inv_kernel(int64_t ng, const int32_t *__restrict__ ip, const int32_t *__restrict__ ix,
                                 const double *__restrict__ data, const int64_t *__restrict__ gptr,
                                 const int32_t *__restrict__ grows, const int32_t *__restrict__ gcols,
                                 const int64_t *__restrict__ inv_off, int smax, double *__restrict__ inv,
                                 int32_t *__restrict__ status) {
    extern __shared__ double sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double *A = sm + (size_t)wid * 2 * smax * smax, *E = A + (size_t)smax * smax;
    for (int64_t g = (int64_t)blockIdx.x * kInvWarps + wid; g < ng; g += (int64_t)gridDim.x * kInvWarps) {
        const int64_t base = gptr[g];
        const int s = (int)(gptr[g + 1] - base);
        if (lane < s) {
            pb::group_gather_row(ip, ix, data, grows[base + lane], gcols + base, s, A + lane * s);
            pb::group_identity_row(E, s, lane);
        }
        __syncwarp();
        bool ok = true;
        for (int k = 0; k < s; ++k) {
            const int p = pb::group_pivot(A, s, k);    // every lane finds the same pivot
            if (p < 0) { ok = false; break; }
            __syncwarp();
            if (lane < s) pb::group_swap_col(A, E, s, k, p, lane);
            __syncwarp();
            if (lane < s && lane != k) pb::group_eliminate_row(A, E, s, k, lane);
            __syncwarp();
            if (lane == k) pb::group_scale_row(A, E, s, k);
            __syncwarp();
        }
        if (ok) {
            bool finite = true;
            if (lane < s)
                for (int j = 0; j < s; ++j) finite = finite && isfinite(E[lane * s + j]);
            ok = __all_sync(0xffffffffu, finite);
        }
        if (!ok) {
            if (lane == 0) atomicMin(status, (int32_t)g);
        } else if (lane < s) {
            double *out = inv + inv_off[g] + (int64_t)lane * s;
            for (int j = 0; j < s; ++j) out[j] = E[lane * s + j];
        }
        __syncwarp();
    }
}

// z[C_g] = B_g^-1 y[R_g] (acc: z[C_g] +=); one thread per entry of the grouped order; skipped once DONE is set (scal)
__global__ void group_apply_kernel(int64_t n, const int32_t *__restrict__ grp_of, const int64_t *__restrict__ gptr,
                                   const int32_t *__restrict__ grows, const int32_t *__restrict__ gcols,
                                   const int64_t *__restrict__ inv_off, const double *__restrict__ inv,
                                   const double *__restrict__ y, double *__restrict__ z, int acc,
                                   const double *__restrict__ scal) {
    if (scal && scal[GM_DONE] != 0.0) return;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
        const int32_t g = grp_of[q];
        const int64_t base = gptr[g];
        const int s = (int)(gptr[g + 1] - base), i = (int)(q - base);
        const double *b = inv + inv_off[g] + (int64_t)i * s;
        double v = 0.0;
        for (int j = 0; j < s; ++j) v += b[j] * y[grows[base + j]];
        if (acc) z[gcols[q]] += v; else z[gcols[q]] = v;
    }
}

// ---------------------------------------------------------------- GMRES vector kernels
// x = 0, V_0 = b, partial |b|^2
__global__ void gm_init_kernel(int64_t n, const double *__restrict__ b, double *__restrict__ x, double *__restrict__ v0,
                               double *__restrict__ partial, int stride) {
    double acc = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const double bi = b[r];
        x[r] = 0.0;
        v0[r] = bi;
        acc += bi * bi;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * stride] = acc;
}

// V_j *= 1 / scal[slot] (V_0 by beta at the cycle start, V_{j+1} by h_{j+1,j})
__global__ void gm_scale_kernel(int64_t n, double *__restrict__ v, const double *__restrict__ scal, int slot) {
    if (scal[GM_DONE] != 0.0) return;
    const double d = scal[slot];
    if (!(d != 0.0)) return;
    const double inv = 1.0 / d;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) v[r] *= inv;
}

// partial[b][0..cnt) = V^T w, partial[b][cnt] = |w|^2
__global__ void gm_dots_kernel(int64_t n, const double *__restrict__ V, int cnt, const double *__restrict__ w,
                               double *__restrict__ partial, int stride, const double *__restrict__ scal) {
    if (scal[GM_DONE] != 0.0) return;
    block_dots(n, V, cnt, w, partial, stride);
    double acc = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
        acc += w[r] * w[r];
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * stride + cnt] = acc;
}

// w -= V c (c: the last reduction), partial[b][cnt] = |w|^2; dots: partial[b][0..cnt) = V^T w (next CGS pass)
__global__ void gm_update_kernel(int64_t n, const double *__restrict__ V, int cnt, double *__restrict__ w,
                                 double *__restrict__ partial, int stride, int dots, const double *__restrict__ scal,
                                 int m) {
    __shared__ double c[GM_MAX_RESTART + 1];
    if (scal[GM_DONE] != 0.0) return;
    const GmLayout L{m};
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) c[i] = scal[L.red() + i];
    __syncthreads();
    double nrm = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        double wr = w[r];
        for (int i = 0; i < cnt; ++i) wr -= V[(int64_t)i * n + r] * c[i];
        w[r] = wr;
        nrm += wr * wr;
    }
    nrm = block_sum(nrm);
    if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * stride + cnt] = nrm;
    if (dots) block_dots(n, V, cnt, w, partial, stride);   // this thread's own rows: its writes are visible
}

// red[i] = sum_b partial[b][i] (i < cnt, fixed order: lane-strided sums, then a shuffle tree; one warp per entry);
// column j of H: H[i][j] = red[i] (acc = 0) or += red[i] (acc = 1) for i < nh
__global__ void gm_reduce_kernel(int nblk, const double *__restrict__ partial, int stride, int cnt, int nh, int j,
                                 int acc, double *__restrict__ scal, int m) {
    if (scal[GM_DONE] != 0.0) return;
    const GmLayout L{m};
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int i = w; i < cnt; i += nw) {
        double v = 0.0;
        for (int b = lane; b < nblk; b += 32) v += partial[(int64_t)b * stride + i];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) {
            scal[L.red() + i] = v;
            if (i < nh) {
                if (acc) scal[L.h(i, j)] += v; else scal[L.h(i, j)] = v;
            }
        }
    }
}

__device__ double warp_sum_partials(int nblk, const double *__restrict__ partial, int stride, int slot) {
    const int lane = threadIdx.x & 31;
    double v = 0.0;
    for (int b = lane; b < nblk; b += 32) v += partial[(int64_t)b * stride + slot];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One warp: h_{j+1,j} = |w| from the partials, the previous rotations on column j, the new rotation, g and the
// estimate; DONE on convergence of the estimate, on a lucky breakdown or on a breakdown.
__global__ void gm_givens_kernel(int nblk, const double *__restrict__ partial, int stride, int j,
                                 double *__restrict__ scal, int m) {
    if (scal[GM_DONE] != 0.0) return;
    const GmLayout L{m};
    const double ww = warp_sum_partials(nblk, partial, stride, j + 1);
    if (threadIdx.x != 0) return;
    const double hn = sqrt(ww), w0 = sqrt(scal[L.red() + j + 1]);   // |w| after and before the orthogonalisation
    double *cs = scal + L.cs(), *sn = scal + L.sn(), *g = scal + L.g();
    for (int i = 0; i < j; ++i) {
        const double a = scal[L.h(i, j)], b = scal[L.h(i + 1, j)];
        scal[L.h(i, j)] = cs[i] * a + sn[i] * b;
        scal[L.h(i + 1, j)] = -sn[i] * a + cs[i] * b;
    }
    scal[L.h(j + 1, j)] = hn;
    const double a = scal[L.h(j, j)];
    const double r = hypot(a, hn);
    if (!(r > 0.0) || !isfinite(r) || !isfinite(w0)) {   // singular column or overflow: keep the previous steps
        scal[GM_BAD] = 1.0;
        scal[GM_DONE] = 1.0;
        return;
    }
    cs[j] = a / r;
    sn[j] = hn / r;
    scal[L.h(j, j)] = r;
    g[j + 1] = -sn[j] * g[j];
    g[j] = cs[j] * g[j];
    scal[GM_EST] = fabs(g[j + 1]);
    scal[GM_STEPS] += 1.0;
    scal[GM_TOTAL] += 1.0;
    const bool lucky = hn <= 1e-14 * w0;
    if (lucky) scal[GM_LUCKY] = 1.0;
    if (lucky || scal[GM_EST] <= scal[GM_TOLB]) scal[GM_DONE] = 1.0;
}

// One warp (lane 0): y = R^-1 g over the k = STEPS columns of the cycle
__global__ void gm_solve_kernel(double *__restrict__ scal, int m) {
    if (threadIdx.x != 0) return;
    const GmLayout L{m};
    const int k = (int)scal[GM_STEPS];
    double *y = scal + L.y();
    const double *g = scal + L.g();
    for (int i = k - 1; i >= 0; --i) {
        double v = g[i];
        for (int l = i + 1; l < k; ++l) v -= scal[L.h(i, l)] * y[l];
        y[i] = v / scal[L.h(i, i)];
    }
}

// u = V y (acc: u += V y) over the k = STEPS columns of the cycle
__global__ void gm_combine_kernel(int64_t n, const double *__restrict__ V, double *__restrict__ u, int acc,
                                  const double *__restrict__ scal, int m) {
    const GmLayout L{m};
    const int k = (int)scal[GM_STEPS];
    const double *y = scal + L.y();
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        double v = 0.0;
        for (int i = 0; i < k; ++i) v += V[(int64_t)i * n + r] * y[i];
        u[r] = acc ? u[r] + v : v;
    }
}

// V_0 = b - V_0 (V_0 holds A x), partial |V_0|^2
__global__ void gm_residual_kernel(int64_t n, const double *__restrict__ b, double *__restrict__ v0,
                                   double *__restrict__ partial, int stride) {
    double acc = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const double v = b[r] - v0[r];
        v0[r] = v;
        acc += v * v;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[(int64_t)blockIdx.x * stride] = acc;
}

// One warp: the true residual of the cycle end starts the next cycle (first: it is |b|, which sets the tolerance)
__global__ void gm_restart_kernel(int nblk, const double *__restrict__ partial, int stride, double *__restrict__ scal,
                                  int m, int first, double tol) {
    const GmLayout L{m};
    const double rr = warp_sum_partials(nblk, partial, stride, 0);
    if (threadIdx.x != 0) return;
    if (first) {
        scal[GM_BB] = rr;
        scal[GM_TOLB] = tol * sqrt(rr);
    }
    if (!isfinite(rr)) scal[GM_BAD] = 1.0;
    scal[GM_RES2] = rr;
    scal[GM_BETA] = sqrt(rr);
    scal[GM_EST] = sqrt(rr);
    scal[GM_STEPS] = 0.0;
    scal[GM_DONE] = 0.0;
    double *g = scal + L.g();
    g[0] = sqrt(rr);
    for (int i = 1; i <= m; ++i) g[i] = 0.0;
}

bool gm_args_ok(int64_t n, int m, int nblk) { return n > 0 && m >= 1 && m <= GM_MAX_RESTART && nblk >= 1 && nblk <= 4096; }

// z = M^-1 y (acc: z +=) with the group arrays; no preconditioner: z = y, or z += y
int apply_prec(int64_t n, const int32_t *grp_of, const int64_t *gptr, const int32_t *grows, const int32_t *gcols,
               const int64_t *inv_off, const double *inv, const double *y, double *z, int acc, const double *scal,
               cudaStream_t st) {
    group_apply_kernel<<<grid_stride_blocks(n, GM_THREADS, 8), GM_THREADS, 0, st>>>(n, grp_of, gptr, grows, gcols,
                                                                                    inv_off, inv, y, z, acc, scal);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

}  // namespace

extern "C" int pb_group_inv_dev(const pb_csr *a, int64_t ngroups, const int64_t *gptr, const int32_t *grows,
                                const int32_t *gcols, const int64_t *inv_off, int smax, double *inv_out,
                                int32_t *status_dev, uint64_t stream) {
    if (!a || !gptr || !grows || !gcols || !inv_off || !inv_out || !status_dev)
        return pb_fail_(PB_EINVAL, "pb_group_inv_dev: null pointer");
    if (ngroups < 0 || smax < 1 || smax > pb::kGroupMax)
        return pb_fail_(PB_EINVAL, "pb_group_inv_dev: group sizes must be 1 .. 32");
    if (ngroups == 0) return PB_OK;
    const CsrView v = pb_csr_view_(a);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)kInvWarps * 2 * smax * smax * sizeof(double);
    CUDA_TRY(cudaFuncSetAttribute(group_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaMemsetAsync(status_dev, 0x7f, sizeof(int32_t), st));
    group_inv_kernel<<<grid_stride_blocks(ngroups, kInvWarps, 16), 32 * kInvWarps, smem, st>>>(
        ngroups, v.indptr, v.indices, v.data, gptr, grows, gcols, inv_off, smax, inv_out, status_dev);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    int32_t bad = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(&bad, status_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad < ngroups)
        return pb_fail_(PB_ESINGULAR, "group " + std::to_string(bad) + " of the block-Jacobi preconditioner has a zero "
                                      "or non-finite pivot");
    return PB_OK;
}

extern "C" int pb_group_apply_dev(int64_t n, const int32_t *grp_of, const int64_t *gptr, const int32_t *grows,
                                  const int32_t *gcols, const int64_t *inv_off, const double *inv, const double *y,
                                  double *z, int accumulate, uint64_t stream) {
    if (!grp_of || !gptr || !grows || !gcols || !inv_off || !inv || !y || !z)
        return pb_fail_(PB_EINVAL, "pb_group_apply_dev: null pointer");
    if (n <= 0) return PB_OK;
    return apply_prec(n, grp_of, gptr, grows, gcols, inv_off, inv, y, z, accumulate != 0, nullptr, (cudaStream_t)stream);
}

extern "C" int64_t pb_gmres_scal_size(int m) { return m >= 1 && m <= GM_MAX_RESTART ? GmLayout{m}.size() : -1; }

extern "C" int pb_gmres_init(int64_t n, int m, const double *b, double *x, double *V, double *partial, int nblk,
                             double *scal, double tol, uint64_t stream) {
    if (!b || !x || !V || !partial || !scal) return pb_fail_(PB_EINVAL, "pb_gmres_init: null pointer");
    if (!gm_args_ok(n, m, nblk)) return pb_fail_(PB_EINVAL, "pb_gmres_init: need n > 0, 1 <= m <= 128, 1 <= nblk <= 4096");
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaMemsetAsync(scal, 0, GmLayout{m}.size() * sizeof(double), st));
    gm_init_kernel<<<nblk, GM_THREADS, 0, st>>>(n, b, x, V, partial, m + 2);
    gm_restart_kernel<<<1, 32, 0, st>>>(nblk, partial, m + 2, scal, m, 1, tol);
    pb_count_launch_();
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

extern "C" int pb_gmres_step(pb_csr *a, int64_t n, int m, int j, double *V, double *z, double *partial, int nblk,
                             double *scal, const int32_t *grp_of, const int64_t *gptr, const int32_t *grows,
                             const int32_t *gcols, const int64_t *inv_off, const double *inv, uint64_t stream) {
    if (!a || !V || !z || !partial || !scal) return pb_fail_(PB_EINVAL, "pb_gmres_step: null pointer");
    if (!gm_args_ok(n, m, nblk) || j < 0 || j >= m) return pb_fail_(PB_EINVAL, "pb_gmres_step: bad size or step");
    cudaStream_t st = (cudaStream_t)stream;
    const int stride = m + 2, cnt = j + 1;
    double *vj = V + (int64_t)j * n, *w = V + (int64_t)(j + 1) * n;
    if (j == 0) {
        gm_scale_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, scal, GM_BETA);
        pb_count_launch_();
    }
    const double *x_in = vj;
    if (inv) {
        int rc = apply_prec(n, grp_of, gptr, grows, gcols, inv_off, inv, vj, z, 0, scal, st);
        if (rc) return rc;
        x_in = z;
    }
    int rc = pb_csr_spmv_dev(a, x_in, w, stream);
    if (rc) return rc;
    gm_dots_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, cnt, w, partial, stride, scal);
    gm_reduce_kernel<<<1, 1024, 0, st>>>(nblk, partial, stride, cnt + 1, cnt, j, 0, scal, m);
    gm_update_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, cnt, w, partial, stride, 1, scal, m);
    gm_reduce_kernel<<<1, 1024, 0, st>>>(nblk, partial, stride, cnt, cnt, j, 1, scal, m);
    gm_update_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, cnt, w, partial, stride, 0, scal, m);
    gm_givens_kernel<<<1, 32, 0, st>>>(nblk, partial, stride, j, scal, m);
    gm_scale_kernel<<<nblk, GM_THREADS, 0, st>>>(n, w, scal, GmLayout{m}.h(j + 1, j));
    for (int k = 0; k < 7; ++k) pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

extern "C" int pb_gmres_cycle_end(pb_csr *a, int64_t n, int m, const double *b, double *x, double *V, double *z,
                                  double *partial, int nblk, double *scal, const int32_t *grp_of, const int64_t *gptr,
                                  const int32_t *grows, const int32_t *gcols, const int64_t *inv_off, const double *inv,
                                  uint64_t stream) {
    if (!a || !b || !x || !V || !z || !partial || !scal) return pb_fail_(PB_EINVAL, "pb_gmres_cycle_end: null pointer");
    if (!gm_args_ok(n, m, nblk)) return pb_fail_(PB_EINVAL, "pb_gmres_cycle_end: bad size");
    cudaStream_t st = (cudaStream_t)stream;
    gm_solve_kernel<<<1, 32, 0, st>>>(scal, m);
    pb_count_launch_();
    if (inv) {
        gm_combine_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, z, 0, scal, m);
        pb_count_launch_();
        int rc = apply_prec(n, grp_of, gptr, grows, gcols, inv_off, inv, z, x, 1, nullptr, st);
        if (rc) return rc;
    } else {
        gm_combine_kernel<<<nblk, GM_THREADS, 0, st>>>(n, V, x, 1, scal, m);
        pb_count_launch_();
    }
    int rc = pb_csr_spmv_dev(a, x, V, stream);
    if (rc) return rc;
    gm_residual_kernel<<<nblk, GM_THREADS, 0, st>>>(n, b, V, partial, m + 2);
    gm_restart_kernel<<<1, 32, 0, st>>>(nblk, partial, m + 2, scal, m, 0, 0.0);
    pb_count_launch_();
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
