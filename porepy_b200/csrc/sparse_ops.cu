// sparse_ops.cu -- device-side sparse algebra of the forward-mode AD Jacobian chain (SURVEY.md 8a rows a21-a23 / 8f
// rank 2): what the reference does with scipy on the host for every operator evaluation,
//   M @ jac            SpGEMM            AdArray.__rmatmul__        numerics/ad/forward_mode.py:565-595
//   diag(v) @ jac      row scaling       AdArray._diagvec_mul_jac   numerics/ad/forward_mode.py:613-616
//   jac_a + jac_b      sparse add        AdArray.__add__ / __sub__  numerics/ad/forward_mode.py
//   block_diag(mats)   MergedOperator.parse (csr_matrix_from_sparse_blocks)   numerics/ad/ad_utils.py:597-664
//   vstack(blocks)     EquationSystem.assemble                      numerics/ad/equation_system.py:1695-1713
// on pb_csr matrices that never leave HBM.  FP64 values, int32 indices, sorted rows (canonical CSR, like scipy's).
#include "csr_build.cuh"

// The two passes of every operation here, on the legacy default stream: count(counts) launches the pass that writes
// the length of each of the nrows rows of C (and may refuse), the lengths are scanned into C's row offsets, and
// fill(C) launches the pass that writes C's entries.  `what` names the result in the overflow message.
template <class Count, class Fill>
static int csr_two_pass(int64_t nrows, int64_t ncols, const char *what, Count count, Fill fill, pb_csr **out) {
    DevBuf counts, ip;
    CUDA_TRY(counts.ensure((size_t)nrows * sizeof(int32_t)));
    CUDA_TRY(ip.ensure((size_t)(nrows + 1) * sizeof(int32_t)));
    pb_count_launch_();
    int rc = count(counts.as<int32_t>());
    if (rc) return rc;
    int64_t nnz = 0;
    rc = pb_scan_offsets_(counts.as<int32_t>(), ip.as<int32_t>(), nrows, 0, &nnz);
    if (rc) return rc;
    if (nnz >= 0x7fffffffll) return pb_fail_(PB_ENOTIMPL, std::string(what) + " exceeds int32 indices");
    CsrPtr c;
    rc = pb_csr_alloc_(nrows, ncols, nnz, c);
    if (rc) return rc;
    const CsrView C = pb_csr_view_(c.get());
    CUDA_TRY(cudaMemcpy(C.indptr, ip.p, (size_t)(nrows + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice));
    fill(C);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaDeviceSynchronize());
    *out = c.release();
    return PB_OK;
}

// ---- SpGEMM: one warp per row of A, hash table in shared memory -------------------------------------------------
// upper bound of the products of row r: sum over its entries of the length of the matching row of B
__global__ void spgemm_bound_kernel(int64_t nrows, const int32_t *__restrict__ aip, const int32_t *__restrict__ aix,
                                    const int32_t *__restrict__ bip, int *max_bound) {
    int mx = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        long long s = 0;
        for (int q = aip[r]; q < aip[r + 1]; ++q) s += bip[aix[q] + 1] - bip[aix[q]];
        mx = max(mx, (int)(s < 0x7fffffffll ? s : 0x7fffffffll));
    }
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) atomicMax(max_bound, mx);
}

template <int PASS>
__global__ void spgemm_kernel(int64_t nrows, const int32_t *__restrict__ aip, const int32_t *__restrict__ aix,
                              const double *__restrict__ ada, const int32_t *__restrict__ bip,
                              const int32_t *__restrict__ bix, const double *__restrict__ bda, int tsize,
                              int32_t *__restrict__ counts, const int32_t *__restrict__ cip, int32_t *__restrict__ cix,
                              double *__restrict__ cda, int *overflow) {
    extern __shared__ unsigned char so_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    int32_t *keys = (int32_t *)so_smem + (size_t)wib * tsize;
    double *vals = (double *)(so_smem + (size_t)wpb * tsize * sizeof(int32_t)) + (size_t)wib * tsize;
    const unsigned mask = (unsigned)tsize - 1u;
    for (int64_t r = (int64_t)blockIdx.x * wpb + wib; r < nrows; r += (int64_t)gridDim.x * wpb) {
        for (int i = lane; i < tsize; i += 32) { keys[i] = -1; if (PASS == 1) vals[i] = 0.0; }
        __syncwarp();
        for (int qa = aip[r]; qa < aip[r + 1]; ++qa) {
            const int k = aix[qa];
            const double av = PASS == 1 ? ada[qa] : 0.0;
            for (int qb = bip[k] + lane; qb < bip[k + 1]; qb += 32) {
                const int col = bix[qb];
                unsigned h = ((unsigned)col * 2654435761u) & mask;
                for (int probe = 0;; ++probe) {
                    const int old = atomicCAS(&keys[h], -1, col);
                    if (old == -1 || old == col) {
                        if (PASS == 1) atomicAdd(&vals[h], av * bda[qb]);
                        break;
                    }
                    h = (h + 1u) & mask;
                    if (probe > tsize) { atomicExch(overflow, 1); break; }
                }
            }
            __syncwarp();
        }
        // compaction (PASS 0: count only)
        int off = 0;
        const int64_t base = PASS == 1 ? cip[r] : 0;
        for (int i0 = 0; i0 < tsize; i0 += 32) {
            const int kk = keys[i0 + lane];
            const unsigned m = __ballot_sync(0xffffffffu, kk != -1);
            if (PASS == 1 && kk != -1) {
                const int pos = off + __popc(m & ((1u << lane) - 1u));
                cix[base + pos] = kk;
                cda[base + pos] = vals[i0 + lane];
            }
            off += __popc(m);
        }
        if (PASS == 0) { if (lane == 0) counts[r] = off; __syncwarp(); continue; }
        __syncwarp();
        // sort the row by column: bitonic network on (key, value) pairs staged in the (now free) table
        const int len = off;
        int P = 1;
        while (P < len) P <<= 1;
        for (int i = lane; i < P; i += 32) {
            keys[i] = i < len ? cix[base + i] : 0x7fffffff;
            vals[i] = i < len ? cda[base + i] : 0.0;
        }
        __syncwarp();
        warp_bitonic_sort(P, [&](int i, int l, bool asc) {
            if (warp_cas(keys, i, l, asc)) { const double t = vals[i]; vals[i] = vals[l]; vals[l] = t; }
        });
        for (int i = lane; i < len; i += 32) { cix[base + i] = keys[i]; cda[base + i] = vals[i]; }
        __syncwarp();
    }
}

extern "C" int pb_csr_spgemm(const pb_csr *a_, const pb_csr *b_, pb_csr **out) {
    if (!a_ || !b_ || !out) return pb_fail_(PB_EINVAL, "null pointer");
    const CsrView A = pb_csr_view_(a_), B = pb_csr_view_(b_);
    if (A.ncols != B.nrows) return pb_fail_(PB_EINVAL, "dimension mismatch in sparse product");
    DevBuf flag;
    CUDA_TRY(flag.ensure(2 * sizeof(int)));
    CUDA_TRY(cudaMemset(flag.p, 0, 2 * sizeof(int)));
    spgemm_bound_kernel<<<grid_stride_blocks(A.nrows, 256, 8), 256>>>(A.nrows, A.indptr, A.indices, B.indptr,
                                                                      flag.as<int>() + 1);
    pb_count_launch_();
    int hb[2] = {0, 0};
    CUDA_TRY(cudaMemcpy(hb, flag.p, sizeof(hb), cudaMemcpyDeviceToHost));
    long long want = std::min<long long>(2ll * hb[1], 2ll * (long long)B.ncols);
    int tsize = 64;
    while (tsize < want && tsize < 8192) tsize <<= 1;
    if ((long long)tsize < std::min<long long>((long long)hb[1], (long long)B.ncols) + 8)
        return pb_fail_(PB_ENOTIMPL, "sparse product: a row has more than 8184 candidate entries");
    const int wpb = tsize <= 2048 ? 4 : (tsize <= 4096 ? 4 : 2);
    const size_t smem = (size_t)wpb * tsize * (sizeof(int32_t) + sizeof(double));
    CUDA_TRY(cudaFuncSetAttribute(spgemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaFuncSetAttribute(spgemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = grid_stride_blocks(A.nrows, wpb, 4);
    return csr_two_pass(
        A.nrows, B.ncols, "sparse product",
        [&](int32_t *counts) {
            spgemm_kernel<0><<<grid, wpb * 32, smem>>>(A.nrows, A.indptr, A.indices, A.data, B.indptr, B.indices, B.data,
                                                       tsize, counts, nullptr, nullptr, nullptr, flag.as<int>());
            CUDA_TRY(cudaMemcpy(hb, flag.p, sizeof(int), cudaMemcpyDeviceToHost));
            if (hb[0]) return pb_fail_(PB_ECUDA, "sparse product: hash table overflow");
            return PB_OK;
        },
        [&](const CsrView &C) {
            spgemm_kernel<1><<<grid, wpb * 32, smem>>>(A.nrows, A.indptr, A.indices, A.data, B.indptr, B.indices, B.data,
                                                       tsize, nullptr, C.indptr, C.indices, C.data, flag.as<int>());
        },
        out);
}

// ---- C = alpha A + beta B on the union pattern (sorted-row merge; one thread per row) ---------------------------
template <int PASS>
__global__ void axpby_kernel(int64_t nrows, double alpha, const int32_t *__restrict__ aip, const int32_t *__restrict__ aix,
                             const double *__restrict__ ada, double beta, const int32_t *__restrict__ bip,
                             const int32_t *__restrict__ bix, const double *__restrict__ bda,
                             int32_t *__restrict__ counts, const int32_t *__restrict__ cip, int32_t *__restrict__ cix,
                             double *__restrict__ cda) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int qa = aip[r], ea = aip[r + 1], qb = bip[r], eb = bip[r + 1], n = 0;
        const int64_t base = PASS == 1 ? cip[r] : 0;
        while (qa < ea || qb < eb) {
            const int ca = qa < ea ? aix[qa] : 0x7fffffff, cb = qb < eb ? bix[qb] : 0x7fffffff;
            const int col = ca < cb ? ca : cb;
            if (PASS == 1) {
                double v = 0.0;
                if (ca == col) v += alpha * ada[qa];
                if (cb == col) v += beta * bda[qb];
                cix[base + n] = col;
                cda[base + n] = v;
            }
            qa += ca == col; qb += cb == col; ++n;
        }
        if (PASS == 0) counts[r] = n;
    }
}

extern "C" int pb_csr_axpby(double alpha, const pb_csr *a_, double beta, const pb_csr *b_, pb_csr **out) {
    if (!a_ || !b_ || !out) return pb_fail_(PB_EINVAL, "null pointer");
    const CsrView A = pb_csr_view_(a_), B = pb_csr_view_(b_);
    if (A.nrows != B.nrows || A.ncols != B.ncols) return pb_fail_(PB_EINVAL, "dimension mismatch in sparse sum");
    const int grid = grid_stride_blocks(A.nrows, 128, 16);
    return csr_two_pass(
        A.nrows, A.ncols, "sparse sum",
        [&](int32_t *counts) {
            axpby_kernel<0><<<grid, 128>>>(A.nrows, alpha, A.indptr, A.indices, A.data, beta, B.indptr, B.indices, B.data,
                                           counts, nullptr, nullptr, nullptr);
            return PB_OK;
        },
        [&](const CsrView &C) {
            axpby_kernel<1><<<grid, 128>>>(A.nrows, alpha, A.indptr, A.indices, A.data, beta, B.indptr, B.indices, B.data,
                                           nullptr, C.indptr, C.indices, C.data);
        },
        out);
}

// ---- diag(d) @ A and A @ diag(d): same pattern, scaled values (d: DEVICE vector) -------------------------------
__global__ void scale_kernel(int64_t nrows, const int32_t *__restrict__ ip, const int32_t *__restrict__ ix,
                             const double *__restrict__ in, const double *__restrict__ d, int by_cols,
                             double *__restrict__ outv) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        const double dr = by_cols ? 1.0 : d[r];
        for (int q = ip[r] + lane; q < ip[r + 1]; q += 32) outv[q] = in[q] * (by_cols ? d[ix[q]] : dr);
    }
}

extern "C" int pb_csr_scale_dev(const pb_csr *a_, const double *d_dev, int by_cols, pb_csr **out) {
    if (!a_ || !d_dev || !out) return pb_fail_(PB_EINVAL, "null pointer");
    const CsrView A = pb_csr_view_(a_);
    long long nnz = 0;
    CUDA_TRY(cudaMemcpy(&nnz, A.indptr + A.nrows, sizeof(int32_t), cudaMemcpyDeviceToHost));
    nnz &= 0xffffffffll;
    CsrPtr c;
    int rc = pb_csr_alloc_(A.nrows, A.ncols, nnz, c);
    if (rc) return rc;
    const CsrView C = pb_csr_view_(c.get());
    CUDA_TRY(cudaMemcpy(C.indptr, A.indptr, (size_t)(A.nrows + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice));
    if (nnz) CUDA_TRY(cudaMemcpy(C.indices, A.indices, (size_t)nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice));
    scale_kernel<<<grid_stride_blocks(A.nrows * 32, 256, 16), 256>>>(A.nrows, A.indptr, A.indices, A.data, d_dev,
                                                                     by_cols, C.data);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaDeviceSynchronize());
    *out = c.release();
    return PB_OK;
}

// ---- block matrix: nbr x nbc grid of blocks (NULL = zero block) -> one CSR ------------------------------------
// replaces MergedOperator.parse's block-diagonal concatenation (ad_utils.py:650-664) and the vstack of
// EquationSystem.assemble (equation_system.py:1695-1713)
struct BlockDesc { const int32_t *ip, *ix; const double *da; };
template <int PASS>
__global__ void bmat_kernel(int nbr, int nbc, const BlockDesc *__restrict__ blocks, const int64_t *__restrict__ row_off,
                            const int64_t *__restrict__ col_off, int64_t nrows, int32_t *__restrict__ counts,
                            const int32_t *__restrict__ cip, int32_t *__restrict__ cix, double *__restrict__ cda) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int br = 0;
        while (br + 1 < nbr && r >= row_off[br + 1]) ++br;
        const int64_t lr = r - row_off[br];
        int n = 0;
        const int64_t base = PASS == 1 ? cip[r] : 0;
        for (int bc = 0; bc < nbc; ++bc) {
            const BlockDesc b = blocks[br * nbc + bc];
            if (!b.ip) continue;
            for (int q = b.ip[lr]; q < b.ip[lr + 1]; ++q) {
                if (PASS == 1) { cix[base + n] = (int32_t)(b.ix[q] + col_off[bc]); cda[base + n] = b.da[q]; }
                ++n;
            }
        }
        if (PASS == 0) counts[r] = n;
    }
}

extern "C" int pb_csr_bmat(int nbr, int nbc, const pb_csr *const *blocks, const int64_t *row_sizes,
                           const int64_t *col_sizes, pb_csr **out) {
    if (nbr < 1 || nbc < 1 || !blocks || !row_sizes || !col_sizes || !out) return pb_fail_(PB_EINVAL, "bad arguments");
    std::vector<BlockDesc> hb((size_t)nbr * nbc);
    std::vector<int64_t> ro(nbr + 1, 0), co(nbc + 1, 0);
    for (int i = 0; i < nbr; ++i) ro[i + 1] = ro[i] + row_sizes[i];
    for (int j = 0; j < nbc; ++j) co[j + 1] = co[j] + col_sizes[j];
    for (int i = 0; i < nbr; ++i)
        for (int j = 0; j < nbc; ++j) {
            const pb_csr *b = blocks[(size_t)i * nbc + j];
            if (!b) { hb[(size_t)i * nbc + j] = BlockDesc{nullptr, nullptr, nullptr}; continue; }
            const CsrView V = pb_csr_view_(b);
            if (V.nrows != row_sizes[i] || V.ncols != col_sizes[j]) return pb_fail_(PB_EINVAL, "block shape mismatch");
            hb[(size_t)i * nbc + j] = BlockDesc{V.indptr, V.indices, V.data};
        }
    if (co[nbc] >= 0x7fffffffll) return pb_fail_(PB_ENOTIMPL, "block matrix exceeds int32 column indices");
    const int64_t nrows = ro[nbr];
    DevBuf dblocks, drow, dcol;
    CUDA_TRY(dblocks.upload(hb, 0));
    CUDA_TRY(drow.upload(ro, 0));
    CUDA_TRY(dcol.upload(co, 0));
    const int grid = grid_stride_blocks(nrows, 128, 16);
    return csr_two_pass(
        nrows, co[nbc], "block matrix",
        [&](int32_t *counts) {
            bmat_kernel<0><<<grid, 128>>>(nbr, nbc, dblocks.as<BlockDesc>(), drow.as<int64_t>(), dcol.as<int64_t>(), nrows,
                                          counts, nullptr, nullptr, nullptr);
            return PB_OK;
        },
        [&](const CsrView &C) {
            bmat_kernel<1><<<grid, 128>>>(nbr, nbc, dblocks.as<BlockDesc>(), drow.as<int64_t>(), dcol.as<int64_t>(), nrows,
                                          nullptr, C.indptr, C.indices, C.data);
        },
        out);
}
