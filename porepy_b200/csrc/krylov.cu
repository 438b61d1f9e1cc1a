// krylov.cu -- fused vector kernels of the Jacobi-preconditioned BiCGStab that replaces the reference's direct
// solve (SolutionStrategy.solve_linear_system, models/solution_strategy.py:830-884; SURVEY.md 8f rank 1).
//
// One iteration = 3 fused vector kernels + 2 SpMVs whose epilogue accumulates the dot products the recurrence
// needs.  Every scalar of the recurrence (rho, alpha, omega, beta, the residual norm) lives in a small DEVICE
// buffer: kernels read the scalars they need from it, so the host never synchronises inside the loop (it polls
// the buffer every few iterations).  Under torch.distributed the Python layer all-reduces contiguous slices of
// that buffer between the kernels (NCCL, on the same stream) and exchanges the ghost entries before each SpMV.
//
// Scalar buffer (doubles): two parity groups of 5  [RHATV, TS, TT, RR, RHO]  at offsets 0 and 5, then
// [BB, DONE, ITER] at 10..12.  Iteration `it` accumulates into group it&1 (RR, RHO of the NEXT iteration into group
// (it+1)&1) and reads alpha / omega / rho of the previous iteration from the other group; the s-update kernel
// zeroes the other group once its last reader (the p-update of the same iteration) has finished.
//   rho_new = RHO[cur], rho_old = RHO[prv], alpha_prev = RHO[prv] / RHATV[prv], omega_prev = TS[prv] / TT[prv]
//   alpha   = RHO[cur] / RHATV[cur],         omega = TS[cur] / TT[cur]
// DONE is sticky: once the residual norm (all-reduced, identical on all ranks) is below tol * |b| the vector kernels
// stop updating, so polling every k iterations cannot run the recurrence into a 0/0 breakdown.
#include "plan.hpp"

#define KS_RHATV 0
#define KS_TS 1
#define KS_TT 2
#define KS_RR 3
#define KS_RHO 4
#define KS_GROUP 5
#define KS_BB 10
#define KS_DONE 11
#define KS_ITER 12
#define KS_TOL2 13

__device__ __forceinline__ void block_add(double v, double *slot) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __shared__ double part[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) part[w] = v;
    __syncthreads();
    if (w == 0) {
        v = lane < (blockDim.x >> 5) ? part[lane] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) atomicAdd(slot, v);
    }
    __syncthreads();
}

// r = b (x = 0), rhat = r, p = v = 0; BB = RR[0] = RHO[0] = (b, b) accumulated (all-reduce them afterwards)
__global__ void kry_init_kernel(int64_t n, const double *__restrict__ b, double *__restrict__ x, double *__restrict__ r,
                                double *__restrict__ rhat, double *__restrict__ p, double *__restrict__ v,
                                double *__restrict__ scal) {
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double bi = b[i];
        x[i] = 0.0; r[i] = bi; rhat[i] = bi; p[i] = 0.0; v[i] = 0.0;
        acc += bi * bi;
    }
    block_add(acc, scal + KS_BB);
}

// Preconditioner application z = M^-1 y on one block of BS consecutive entries: BS == 1 -- minv holds the inverse
// diagonal (Jacobi); BS > 1 -- minv holds the inverted BS x BS diagonal blocks, row-major (block Jacobi: the nd
// displacement components of a cell in the mechanics system A = div_nd @ stress, the nd + nr + 1 unknowns [u, r, p]
// of a cell in the TPSA system, BS = 4 in 2-D and 7 in 3-D, the nd + nr + 2 unknowns [u, r, p_t, p] of a cell in the
// TPSA poromechanics system, BS = 5 and 8, or the nd + nr + 3 unknowns [u, r, p_t, p, T] of a cell in the TPSA
// thermo-poromechanics system, BS = 6 and 9).
template <int BS>
__device__ __forceinline__ void apply_minv(const double *__restrict__ minv, int64_t b, const double (&y)[BS], double (&z)[BS]) {
    if (!minv) {
#pragma unroll
        for (int i = 0; i < BS; ++i) z[i] = y[i];
    } else if (BS == 1) {
        z[0] = minv[b] * y[0];
    } else {
        const double *m = minv + b * (BS * BS);
#pragma unroll
        for (int i = 0; i < BS; ++i) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j < BS; ++j) acc += m[i * BS + j] * y[j];
            z[i] = acc;
        }
    }
}

// p = r + beta (p - omega_prev v),  ph = M^-1 p      [minv may be null]
template <int BS>
__global__ void kry_p_kernel(int64_t n, const double *__restrict__ r, double *__restrict__ p,
                             const double *__restrict__ v, const double *__restrict__ minv, double *__restrict__ ph,
                             double *__restrict__ scal, int cur) {
    const double *gc = scal + cur * KS_GROUP, *gp = scal + (cur ^ 1) * KS_GROUP;
    const bool frozen = scal[KS_DONE] != 0.0 || !(gc[KS_RR] > scal[KS_TOL2] * scal[KS_BB]);
    if (!frozen) {
        const double alpha_prev = gp[KS_RHO] / gp[KS_RHATV], omega_prev = gp[KS_TS] / gp[KS_TT];
        const double beta = (gc[KS_RHO] / gp[KS_RHO]) * (alpha_prev / omega_prev);
        for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n / BS; b += (int64_t)gridDim.x * blockDim.x) {
            double pv[BS], z[BS];
#pragma unroll
            for (int i = 0; i < BS; ++i) {
                const int64_t q = b * BS + i;
                pv[i] = r[q] + beta * (p[q] - omega_prev * v[q]);
                p[q] = pv[i];
            }
            apply_minv<BS>(minv, b, pv, z);
#pragma unroll
            for (int i = 0; i < BS; ++i) ph[b * BS + i] = z[i];
        }
    }
    __syncthreads();
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        // the last block to be SCHEDULED is not the last to finish; DONE / ITER are only read by LATER kernels
        if (frozen) scal[KS_DONE] = 1.0; else scal[KS_ITER] += 1.0;
    }
}

// s = r - alpha v,  sh = M^-1 s;  zero the other parity group (its last reader was this iteration's p-update)
template <int BS>
__global__ void kry_s_kernel(int64_t n, const double *__restrict__ r, const double *__restrict__ v,
                             const double *__restrict__ minv, double *__restrict__ s, double *__restrict__ sh,
                             double *__restrict__ scal, int cur) {
    const double *gc = scal + cur * KS_GROUP;
    if (scal[KS_DONE] == 0.0) {
        const double alpha = gc[KS_RHO] / gc[KS_RHATV];
        for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n / BS; b += (int64_t)gridDim.x * blockDim.x) {
            double sv[BS], z[BS];
#pragma unroll
            for (int i = 0; i < BS; ++i) {
                const int64_t q = b * BS + i;
                sv[i] = r[q] - alpha * v[q];
                s[q] = sv[i];
            }
            apply_minv<BS>(minv, b, sv, z);
#pragma unroll
            for (int i = 0; i < BS; ++i) sh[b * BS + i] = z[i];
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < KS_GROUP) scal[(cur ^ 1) * KS_GROUP + threadIdx.x] = 0.0;
}

// x += alpha ph + omega sh,  r = s - omega t;  RR[next] += (r, r),  RHO[next] += (rhat, r)
__global__ void kry_xr_kernel(int64_t n, double *__restrict__ x, const double *__restrict__ ph,
                              const double *__restrict__ sh, const double *__restrict__ s, const double *__restrict__ t,
                              double *__restrict__ r, const double *__restrict__ rhat, double *__restrict__ scal, int cur,
                              int carry) {
    const double *gc = scal + cur * KS_GROUP;
    double *gn = scal + (cur ^ 1) * KS_GROUP;
    double rr = 0.0, rho = 0.0;
    if (scal[KS_DONE] != 0.0) {
        // frozen: the residual norm is carried to the next parity group (by ONE rank: the slices are sum-reduced)
        if (carry && blockIdx.x == 0 && threadIdx.x == 0) { rr = gc[KS_RR]; rho = gc[KS_RHO]; }
    } else {
        const double alpha = gc[KS_RHO] / gc[KS_RHATV], omega = gc[KS_TS] / gc[KS_TT];
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
            x[i] += alpha * ph[i] + omega * sh[i];
            const double ri = s[i] - omega * t[i];
            r[i] = ri;
            rr += ri * ri;
            rho += rhat[i] * ri;
        }
    }
    block_add(rr, gn + KS_RR);
    block_add(rho, gn + KS_RHO);
}

extern "C" int pb_kry_init(int64_t n, const double *b, double *x, double *r, double *rhat, double *p, double *v,
                           double *scal, double tol, uint64_t stream) {
    if (!b || !x || !r || !rhat || !p || !v || !scal) return pb_fail_(PB_EINVAL, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    double h[14] = {0.0, 0.0, 0.0, 0.0, 0.0,  /* group 0: accumulators of iteration 0 (RR, RHO seeded from BB) */
                    1.0, 1.0, 1.0, 0.0, 1.0,  /* group 1 = "previous" of iteration 0: alpha = omega = rho = 1 */
                    0.0, 0.0, 0.0, tol * tol};
    CUDA_TRY(cudaMemcpyAsync(scal, h, sizeof(h), cudaMemcpyHostToDevice, st));
    kry_init_kernel<<<grid_stride_blocks(n, 256, 8), 256, 0, st>>>(n, b, x, r, rhat, p, v, scal);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
// after the all-reduce of BB: RR[0] = RHO[0] = BB (r = rhat = b)
__global__ void kry_seed_kernel(double *scal) { scal[KS_RR] = scal[KS_BB]; scal[KS_RHO] = scal[KS_BB]; }
extern "C" int pb_kry_seed(double *scal, uint64_t stream) {
    kry_seed_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(scal);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
static bool kry_block_size_ok(int bs) { return bs >= 1 && bs <= 9; }

// bs: size of the diagonal blocks of the preconditioner (1 = Jacobi, 2 / 3 / 4 / 5 / 7 / 8 = block Jacobi; n must be a
// multiple)
extern "C" int pb_kry_p(int64_t n, const double *r, double *p, const double *v, const double *minv, double *ph,
                        double *scal, int cur, int bs, uint64_t stream) {
    if (!kry_block_size_ok(bs) || n % bs)
        return pb_fail_(PB_EINVAL, "pb_kry_p: block size must be 1, 2, 3, 4, 5, 7 or 8 and divide n");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_stride_blocks(n / bs, 256, 8);
    if (bs == 1) kry_p_kernel<1><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 2) kry_p_kernel<2><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 3) kry_p_kernel<3><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 4) kry_p_kernel<4><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 5) kry_p_kernel<5><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 6) kry_p_kernel<6><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 7) kry_p_kernel<7><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else if (bs == 8) kry_p_kernel<8><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    else kry_p_kernel<9><<<grid, 256, 0, st>>>(n, r, p, v, minv, ph, scal, cur & 1);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
extern "C" int pb_kry_s(int64_t n, const double *r, const double *v, const double *minv, double *s, double *sh,
                        double *scal, int cur, int bs, uint64_t stream) {
    if (!kry_block_size_ok(bs) || n % bs)
        return pb_fail_(PB_EINVAL, "pb_kry_s: block size must be 1, 2, 3, 4, 5, 7 or 8 and divide n");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_stride_blocks(n / bs, 256, 8);
    if (bs == 1) kry_s_kernel<1><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 2) kry_s_kernel<2><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 3) kry_s_kernel<3><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 4) kry_s_kernel<4><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 5) kry_s_kernel<5><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 6) kry_s_kernel<6><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 7) kry_s_kernel<7><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else if (bs == 8) kry_s_kernel<8><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    else kry_s_kernel<9><<<grid, 256, 0, st>>>(n, r, v, minv, s, sh, scal, cur & 1);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

// Inverses of the bs x bs diagonal blocks of a CSR matrix (rows / columns bs*b .. bs*b+bs-1), row-major, to a DEVICE
// array of nblocks*bs*bs doubles: the block-Jacobi preconditioner of the mechanics systems (one block per cell).
// A singular block is replaced by the inverse of its diagonal (identity where that is zero, too).
template <int BS>
__global__ void block_diag_inv_kernel(int64_t nb, const int32_t *__restrict__ ip, const int32_t *__restrict__ ix,
                                      const double *__restrict__ data, double *__restrict__ out) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t)gridDim.x * blockDim.x) {
        double D[BS][BS], E[BS][BS];
#pragma unroll
        for (int i = 0; i < BS; ++i) {
#pragma unroll
            for (int j = 0; j < BS; ++j) { D[i][j] = 0.0; E[i][j] = i == j ? 1.0 : 0.0; }
            const int64_t row = b * BS + i;
            for (int q = ip[row]; q < ip[row + 1]; ++q) {
                const int64_t c = (int64_t)ix[q] - b * BS;
                if (c >= 0 && c < BS) {
#pragma unroll
                    for (int j = 0; j < BS; ++j) if (c == j) D[i][j] += data[q];
                }
            }
        }
        double dg[BS];
#pragma unroll
        for (int i = 0; i < BS; ++i) dg[i] = D[i][i];
        bool ok = true;
#pragma unroll
        for (int k = 0; k < BS; ++k) {   // Gauss-Jordan with partial pivoting, fully unrolled (BS <= 7)
            int piv = k;
            double best = fabs(D[k][k]);
#pragma unroll
            for (int i = k + 1; i < BS; ++i) if (fabs(D[i][k]) > best) { best = fabs(D[i][k]); piv = i; }
            if (!(best > 0.0)) { ok = false; break; }
#pragma unroll
            for (int i = k + 1; i < BS; ++i)
                if (i == piv) {
#pragma unroll
                    for (int j = 0; j < BS; ++j) {
                        double t = D[k][j]; D[k][j] = D[i][j]; D[i][j] = t;
                        t = E[k][j]; E[k][j] = E[i][j]; E[i][j] = t;
                    }
                }
            const double inv = 1.0 / D[k][k];
#pragma unroll
            for (int j = 0; j < BS; ++j) { D[k][j] *= inv; E[k][j] *= inv; }
#pragma unroll
            for (int i = 0; i < BS; ++i) {
                if (i == k) continue;
                const double f = D[i][k];
#pragma unroll
                for (int j = 0; j < BS; ++j) { D[i][j] -= f * D[k][j]; E[i][j] -= f * E[k][j]; }
            }
        }
#pragma unroll
        for (int i = 0; i < BS; ++i)
#pragma unroll
            for (int j = 0; j < BS; ++j)
                out[(b * BS + i) * BS + j] = ok ? E[i][j] : (i == j ? (dg[i] != 0.0 ? 1.0 / dg[i] : 1.0) : 0.0);
    }
}

// BS = 6, 8, 9: the same inverse and fallback, Gauss-Jordan in place (the pivot rows are recorded and the columns of
// the result swapped back at the end), so one block instead of two stays in registers (9 x 9: 232 registers, no spills).
template <int BS>
__global__ void block_diag_inv_inplace_kernel(int64_t nb, const int32_t *__restrict__ ip, const int32_t *__restrict__ ix,
                                              const double *__restrict__ data, double *__restrict__ out) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t)gridDim.x * blockDim.x) {
        double D[BS][BS];
#pragma unroll
        for (int i = 0; i < BS; ++i) {
#pragma unroll
            for (int j = 0; j < BS; ++j) D[i][j] = 0.0;
            const int64_t row = b * BS + i;
            for (int q = ip[row]; q < ip[row + 1]; ++q) {
                const int64_t c = (int64_t)ix[q] - b * BS;
                if (c >= 0 && c < BS) {
#pragma unroll
                    for (int j = 0; j < BS; ++j) if (c == j) D[i][j] += data[q];
                }
            }
        }
        double dg[BS];
        int perm[BS];
#pragma unroll
        for (int i = 0; i < BS; ++i) { dg[i] = D[i][i]; perm[i] = i; }
        bool ok = true;
#pragma unroll
        for (int k = 0; k < BS; ++k) {
            int piv = k;
            double best = fabs(D[k][k]);
#pragma unroll
            for (int i = k + 1; i < BS; ++i) if (fabs(D[i][k]) > best) { best = fabs(D[i][k]); piv = i; }
            ok = ok && best > 0.0;   // no early exit: the loop stays unrolled and D in registers
            if (!ok) continue;
            perm[k] = piv;
#pragma unroll
            for (int i = k + 1; i < BS; ++i)
                if (i == piv) {
#pragma unroll
                    for (int j = 0; j < BS; ++j) { const double t = D[k][j]; D[k][j] = D[i][j]; D[i][j] = t; }
                }
            const double inv = 1.0 / D[k][k];
            D[k][k] = 1.0;
#pragma unroll
            for (int j = 0; j < BS; ++j) D[k][j] *= inv;
#pragma unroll
            for (int i = 0; i < BS; ++i) {
                if (i == k) continue;
                const double f = D[i][k];
                D[i][k] = 0.0;
#pragma unroll
                for (int j = 0; j < BS; ++j) D[i][j] -= f * D[k][j];
            }
        }
        // row swap k <-> perm[k] of the block is column swap k <-> perm[k] of its inverse, undone in reverse order:
        // column j of D goes to column pos[j] (a scattered store instead of register moves indexed by perm)
        int pos[BS];
#pragma unroll
        for (int j = 0; j < BS; ++j) pos[j] = j;
#pragma unroll
        for (int k = BS - 1; k >= 0; --k)
#pragma unroll
            for (int j = 0; j < BS; ++j) pos[j] = pos[j] == k ? perm[k] : (pos[j] == perm[k] ? k : pos[j]);
#pragma unroll
        for (int i = 0; i < BS; ++i)
#pragma unroll
            for (int j = 0; j < BS; ++j) {
                if (ok) out[(b * BS + i) * BS + pos[j]] = D[i][j];
                else out[(b * BS + i) * BS + j] = i == j ? (dg[i] != 0.0 ? 1.0 / dg[i] : 1.0) : 0.0;
            }
    }
}

extern "C" int pb_csr_block_diag_inv_dev(const pb_csr *a, int bs, int64_t nblocks, double *out_dev, uint64_t stream) {
    if (!a || !out_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const CsrView v = pb_csr_view_(a);
    if (!kry_block_size_ok(bs) || nblocks < 0 || nblocks * bs > v.nrows)
        return pb_fail_(PB_EINVAL, "pb_csr_block_diag_inv_dev: bad block size / count");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_stride_blocks(nblocks, 256, 8);
    if (bs == 1) block_diag_inv_kernel<1><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 2) block_diag_inv_kernel<2><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 3) block_diag_inv_kernel<3><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 4) block_diag_inv_kernel<4><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 5) block_diag_inv_kernel<5><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 6) block_diag_inv_inplace_kernel<6><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 7) block_diag_inv_kernel<7><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else if (bs == 8) block_diag_inv_inplace_kernel<8><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    else block_diag_inv_inplace_kernel<9><<<grid, 256, 0, st>>>(nblocks, v.indptr, v.indices, v.data, out_dev);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
extern "C" int pb_kry_xr(int64_t n, double *x, const double *ph, const double *sh, const double *s, const double *t,
                         double *r, const double *rhat, double *scal, int cur, int carry, uint64_t stream) {
    kry_xr_kernel<<<grid_stride_blocks(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(n, x, ph, sh, s, t, r, rhat, scal,
                                                                                   cur & 1, carry);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
