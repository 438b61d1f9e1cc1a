// spmv.cu -- CSR SpMV / residual kernel on device-resident matrices (HBM-bandwidth bound).
//
// Replaces the scipy `M @ val` of AdArray.__rmatmul__ (numerics/ad/forward_mode.py:565-595)
// and the SpMV chain of a residual-only EquationSystem.assemble
// (numerics/ad/equation_system.py:1579-1713).  fp64 values, int32 column indices, as scipy
// stores the reference's matrices.
//
// Algorithmic traffic per SpMV (SURVEY.md §8d): 12 B per non-zero (value + column index)
// + 20 B per row (row pointer 4, y write 8, x read 8).  A group of TPR lanes (power of two,
// chosen from the mean row length) owns one row: the lanes read consecutive (value, index)
// pairs (coalesced 64/128-byte segments), gather x through the read-only path, and reduce
// with shuffles.  Grid-stride over rows, grid sized to a multiple of the SMs of the device.
#include <cuda_runtime.h>

#include <atomic>
#include <string>

#include "plan.hpp"
#include <map>
#include <mutex>
#include <tuple>


struct pb_csr {
    int64_t nrows = 0, ncols = 0, nnz = 0;
    int32_t *indptr = nullptr, *indices = nullptr;
    double *data = nullptr, *x = nullptr, *y = nullptr;
    DevBuf b_indptr, b_indices, b_data, b_x, b_y;   // owners of the arrays above (pooled device blocks)
    cudaError_t alloc() {
        cudaError_t e;
        if ((e = b_indptr.ensure((size_t)(nrows + 1) * sizeof(int32_t))) != cudaSuccess) return e;
        if ((e = b_indices.ensure((size_t)(nnz ? nnz : 1) * sizeof(int32_t))) != cudaSuccess) return e;
        if ((e = b_data.ensure((size_t)(nnz ? nnz : 1) * sizeof(double))) != cudaSuccess) return e;
        if ((e = b_x.ensure((size_t)(ncols ? ncols : 1) * sizeof(double))) != cudaSuccess) return e;
        if ((e = b_y.ensure((size_t)(nrows ? nrows : 1) * sizeof(double))) != cudaSuccess) return e;
        indptr = b_indptr.as<int32_t>(); indices = b_indices.as<int32_t>();
        data = b_data.as<double>(); x = b_x.as<double>(); y = b_y.as<double>();
        return cudaSuccess;
    }
    int tpr = 8;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
};

template <int TPR>
__global__ void __launch_bounds__(256)
    csr_spmv_kernel(int64_t nrows, const int32_t *__restrict__ indptr,
                    const int32_t *__restrict__ indices, const double *__restrict__ data,
                    const double *__restrict__ x, double *__restrict__ y) {
    const int lane = threadIdx.x & (TPR - 1);
    const int gw = (threadIdx.x & 31) / TPR;           // row group inside the warp
    const int64_t group = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / TPR;
    const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) / TPR;
    // the trip count is WARP-uniform (it depends on the warp's first row only): the full-mask shuffles below are
    // executed by all 32 lanes; groups past the last row carry an empty range
    for (int64_t r0 = group - gw; r0 < nrows; r0 += ngroups) {
        const int64_t r = r0 + gw;
        const bool valid = r < nrows;
        const int b = valid ? __ldg(indptr + r) : 0, e = valid ? __ldg(indptr + r + 1) : 0;
        double acc = 0.0;
        for (int q = b + lane; q < e; q += TPR) acc += __ldg(data + q) * __ldg(x + __ldg(indices + q));
#pragma unroll
        for (int o = TPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, TPR);
        if (lane == 0 && valid) y[r] = acc;
    }
}

// y = A x with the dot products of the Krylov recurrence in the epilogue: d1 += (w1, y), d2 += (w2, y)
// (w2 == y gives |y|^2); one atomic per warp.  Skipped rows never exist: every row is written.
template <int TPR>
__global__ void __launch_bounds__(256)
    csr_spmv_dots_kernel(int64_t nrows, const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                         const double *__restrict__ data, const double *__restrict__ x, double *__restrict__ y,
                         const double *__restrict__ w1, double *d1, const double *__restrict__ w2, int w2_is_y,
                         double *d2) {
    const int lane = threadIdx.x & (TPR - 1);
    const int gw = (threadIdx.x & 31) / TPR;
    const int64_t group = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / TPR;
    const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) / TPR;
    double a1 = 0.0, a2 = 0.0;
    // warp-uniform trip count (see csr_spmv_kernel): with a per-group bound, the groups of one warp that run out of
    // rows first would meet the full-mask shuffles of the epilogue while the others are still inside the loop --
    // undefined, and in practice a row's partial sum leaks into the dot products (seen as a BiCGStab that stalls
    // when the row count of a shard puts the boundary inside a warp)
    for (int64_t r0 = group - gw; r0 < nrows; r0 += ngroups) {
        const int64_t r = r0 + gw;
        const bool valid = r < nrows;
        const int b = valid ? __ldg(indptr + r) : 0, e = valid ? __ldg(indptr + r + 1) : 0;
        double acc = 0.0;
        for (int q = b + lane; q < e; q += TPR) acc += __ldg(data + q) * __ldg(x + __ldg(indices + q));
#pragma unroll
        for (int o = TPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, TPR);
        if (lane == 0 && valid) {
            y[r] = acc;
            if (d1) a1 += w1[r] * acc;
            if (d2) a2 += (w2_is_y ? acc : w2[r]) * acc;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    }
    // one atomic per CTA and dot product (38 k same-address atomics of a one-per-warp epilogue cost 0.05-0.08 ms,
    // a quarter of the SpMV itself: tools/krylov_micro.py)
    __shared__ double part[2][8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { part[0][w] = a1; part[1][w] = a2; }
    __syncthreads();
    if (threadIdx.x < 16) {
        double v = part[threadIdx.x >> 3][threadIdx.x & 7];
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0x0000ffffu, v, o, 8);
        if (threadIdx.x == 0 && d1 && v != 0.0) atomicAdd(d1, v);
        if (threadIdx.x == 8 && d2 && v != 0.0) atomicAdd(d2, v);
    }
}

static int launch_spmv_dots(pb_csr *a, const double *x, double *y, const double *w1, double *d1, const double *w2,
                            int w2_is_y, double *d2, cudaStream_t st) {
    const int block = 256;
    const int64_t groups_per_block = block / a->tpr;
    int64_t need = (a->nrows + groups_per_block - 1) / groups_per_block;
    int64_t cap = (int64_t)pb_sm_count() * 8 * 4;
    int grid = (int)(need < cap ? (need < 1 ? 1 : need) : cap);
#define PB_SPMV_DOTS(T) csr_spmv_dots_kernel<T><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y, w1, d1, w2, w2_is_y, d2)
    switch (a->tpr) {
        case 2: PB_SPMV_DOTS(2); break;
        case 4: PB_SPMV_DOTS(4); break;
        case 8: PB_SPMV_DOTS(8); break;
        case 16: PB_SPMV_DOTS(16); break;
        default: PB_SPMV_DOTS(32); break;
    }
#undef PB_SPMV_DOTS
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

static int launch_spmv(pb_csr *a, const double *x, double *y, cudaStream_t st) {
    const int block = 256;
    const int64_t groups_per_block = block / a->tpr;
    int64_t need = (a->nrows + groups_per_block - 1) / groups_per_block;
    int64_t cap = (int64_t)pb_sm_count() * 8 * 4;  // 8 resident CTAs of 256 threads per SM, 4 waves
    int grid = (int)(need < cap ? (need < 1 ? 1 : need) : cap);
    switch (a->tpr) {
        case 2: csr_spmv_kernel<2><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y); break;
        case 4: csr_spmv_kernel<4><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y); break;
        case 8: csr_spmv_kernel<8><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y); break;
        case 16: csr_spmv_kernel<16><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y); break;
        default: csr_spmv_kernel<32><<<grid, block, 0, st>>>(a->nrows, a->indptr, a->indices, a->data, x, y); break;
    }
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

// pick the lanes-per-row that is fastest for THIS matrix (a few launches, once per matrix; the timing does not
// depend on the values, so device-assembled matrices are tuned before they are filled)
static void autotune_tpr(pb_csr *a) {
    const double mean = a->nrows ? (double)a->nnz / (double)a->nrows : 0.0;
    a->tpr = mean <= 3 ? 2 : mean <= 6 ? 4 : mean <= 24 ? 8 : mean <= 48 ? 16 : 32;
    if (a->nnz <= (1 << 20) || mean > 96.0) return;   // long rows: a full warp per row
    // A re-discretization of the same grid (every Newton iteration, every e2e step) recreates a matrix of the same shape:
    // reuse the choice instead of timing 30-40 launches again (6.6 ms per flow system at 10^6 tetrahedra)
    static std::mutex tune_mu;
    static std::map<std::tuple<int64_t, int64_t, int64_t>, int> tuned;
    const auto key = std::make_tuple(a->nrows, a->ncols, a->nnz);
    {
        std::lock_guard<std::mutex> lk(tune_mu);
        auto it = tuned.find(key);
        if (it != tuned.end()) { a->tpr = it->second; return; }
    }
    cudaMemsetAsync(a->x, 0, (a->ncols ? a->ncols : 1) * sizeof(double), a->stream);
    float best = 1e30f;
    int best_tpr = a->tpr;
    const int cands[4] = {4, 8, 16, 32};
    for (int ci = 0; ci < 4; ++ci) {
        if (cands[ci] * 12 < mean || cands[ci] > 8 * mean) continue;  // implausible for this row length
        a->tpr = cands[ci];
        float ms = 1e30f;
        if (launch_spmv(a, a->x, a->y, a->stream) != PB_OK) break;
        cudaEventRecord(a->e0, a->stream);
        for (int i = 0; i < 10; ++i) launch_spmv(a, a->x, a->y, a->stream);
        cudaEventRecord(a->e1, a->stream);
        if (cudaEventSynchronize(a->e1) == cudaSuccess) cudaEventElapsedTime(&ms, a->e0, a->e1);
        if (ms < best) { best = ms; best_tpr = cands[ci]; }
    }
    a->tpr = best_tpr;
    std::lock_guard<std::mutex> lk(tune_mu);
    tuned[key] = best_tpr;
}

extern "C" void pb_csr_destroy(pb_csr *a) {
    if (!a) return;
    if (a->e0) cudaEventDestroy(a->e0);
    if (a->e1) cudaEventDestroy(a->e1);
    if (a->stream) cudaStreamDestroy(a->stream);
    delete a;
}

extern "C" int pb_csr_create(int64_t nrows, int64_t ncols, int64_t nnz, const int32_t *indptr,
                             const int32_t *indices, const double *data, pb_csr **out) {
    if (!out || !indptr || (nnz > 0 && (!indices || !data)) || nrows < 0 || ncols < 0)
        return pb_fail_(PB_EINVAL, "bad CSR arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1)
        return pb_fail_(PB_ECUDA, "no CUDA device: libporeb200 has no CPU path");
    pb_csr *a = new pb_csr;
    a->nrows = nrows; a->ncols = ncols; a->nnz = nnz;
    auto bail = [&](cudaError_t e) {
        std::string m = cudaGetErrorString(e);
        pb_csr_destroy(a);
        return pb_fail_(PB_ECUDA, m);
    };
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e0)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e1)) != cudaSuccess) return bail(e);
    if ((e = a->alloc()) != cudaSuccess) return bail(e);
    if ((e = cudaMemcpy(a->indptr, indptr, (nrows + 1) * sizeof(int32_t), cudaMemcpyHostToDevice)) != cudaSuccess) return bail(e);
    if (nnz) {
        if ((e = cudaMemcpy(a->indices, indices, nnz * sizeof(int32_t), cudaMemcpyHostToDevice)) != cudaSuccess) return bail(e);
        if ((e = cudaMemcpy(a->data, data, nnz * sizeof(double), cudaMemcpyHostToDevice)) != cudaSuccess) return bail(e);
    }
    double mean = nrows ? (double)nnz / (double)nrows : 0.0;
    a->tpr = mean <= 3 ? 2 : mean <= 6 ? 4 : mean <= 24 ? 8 : mean <= 48 ? 16 : 32;
    autotune_tpr(a);
    *out = a;
    return PB_OK;
}

extern "C" int pb_csr_lanes_per_row(const pb_csr *a) { return a ? a->tpr : -1; }

extern "C" int pb_csr_shape(const pb_csr *a, int64_t *nrows, int64_t *ncols, int64_t *nnz) {
    if (!a) return pb_fail_(PB_EINVAL, "null matrix");
    if (nrows) *nrows = a->nrows;
    if (ncols) *ncols = a->ncols;
    if (nnz) *nnz = a->nnz;
    return PB_OK;
}

int pb_checksum_dev_(const double *v, int64_t n, double *sum, double *sumsq);  // api.cu
extern "C" int pb_csr_checksum(pb_csr *a, double *sum, double *sumsq) {
    if (!a) return pb_fail_(PB_EINVAL, "null matrix");
    CUDA_TRY(cudaDeviceSynchronize());
    int64_t nnz = a->nnz;
    return pb_checksum_dev_(a->data, nnz, sum, sumsq);
}

__global__ void csr_diagonal_kernel(int64_t nrows, const int32_t *__restrict__ ip, const int32_t *__restrict__ ix,
                                    const double *__restrict__ data, double *__restrict__ diag) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        double d = 0.0;
        for (int q = ip[r]; q < ip[r + 1]; ++q)
            if (ix[q] == r) d += data[q];
        diag[r] = d;
    }
}

// diagonal of the matrix (Jacobi preconditioner), to a host array of nrows doubles
extern "C" int pb_csr_diagonal(pb_csr *a, double *diag) {
    if (!a || !diag) return pb_fail_(PB_EINVAL, "null pointer");
    const int64_t n = a->nrows < a->ncols ? a->nrows : a->ncols;
    DevBuf tmp;                       // pooled: no cudaMalloc / cudaFree pair (a device sync each) per call
    CUDA_TRY(tmp.ensure((size_t)(n ? n : 1) * sizeof(double)));
    double *d = tmp.as<double>();
    const int grid = (int)(n / 256 + 1 < pb_sm_count() * 16 ? n / 256 + 1 : pb_sm_count() * 16);
    csr_diagonal_kernel<<<grid, 256, 0, a->stream>>>(n, a->indptr, a->indices, a->data, d);
    pb_count_launch_();
    cudaError_t e = cudaMemcpyAsync(diag, d, n * sizeof(double), cudaMemcpyDeviceToHost, a->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(a->stream);
    if (e != cudaSuccess) return pb_fail_(PB_ECUDA, cudaGetErrorString(e));
    return PB_OK;
}

extern "C" int pb_csr_truncate_rows(pb_csr *a, int64_t nrows) {
    if (!a || nrows < 0 || nrows > a->nrows) return pb_fail_(PB_EINVAL, "bad row count");
    a->nrows = nrows;  // the row-pointer prefix is a valid CSR; nnz keeps the allocated size
    return PB_OK;
}

extern "C" int pb_csr_download(pb_csr *a, int32_t *indptr, int32_t *indices, double *data) {
    if (!a || !indptr || !indices || !data) return pb_fail_(PB_EINVAL, "null pointer");
    CUDA_TRY(cudaMemcpy(indptr, a->indptr, (a->nrows + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (a->nnz) {
        CUDA_TRY(cudaMemcpy(indices, a->indices, a->nnz * sizeof(int32_t), cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(data, a->data, a->nnz * sizeof(double), cudaMemcpyDeviceToHost));
    }
    return PB_OK;
}

// matrix whose pattern is copied from device arrays and whose values the caller fills (api.cu)
int pb_csr_from_device_pattern_(int64_t nrows, int64_t ncols, int64_t nnz, const int32_t *indptr_dev,
                                const int32_t *indices_dev, pb_csr **out) {
    pb_csr *a = new pb_csr;
    a->nrows = nrows; a->ncols = ncols; a->nnz = nnz;
    auto bail = [&](cudaError_t e) {
        std::string m = cudaGetErrorString(e);
        pb_csr_destroy(a);
        return pb_fail_(PB_ECUDA, m);
    };
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e0)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e1)) != cudaSuccess) return bail(e);
    if ((e = a->alloc()) != cudaSuccess) return bail(e);
    if ((e = cudaMemcpy(a->indptr, indptr_dev, (nrows + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice)) != cudaSuccess) return bail(e);
    if (nnz && (e = cudaMemcpy(a->indices, indices_dev, nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice)) != cudaSuccess) return bail(e);
    if ((e = cudaMemset(a->data, 0, (nnz ? nnz : 1) * sizeof(double))) != cudaSuccess) return bail(e);
    // the copies and the memset above ran on the legacy default stream, which does NOT order against the callers'
    // non-blocking streams (the assembly kernels accumulate into `data` right after this returns)
    if ((e = cudaStreamSynchronize(0)) != cudaSuccess) return bail(e);
    autotune_tpr(a);
    *out = a;
    return PB_OK;
}
double *pb_csr_data_(pb_csr *a) { return a->data; }

// an empty matrix of the given sizes (sparse_ops.cu fills indptr / indices / data)
int pb_csr_alloc_(int64_t nrows, int64_t ncols, int64_t nnz, pb_csr **out) {
    pb_csr *a = new pb_csr;
    a->nrows = nrows; a->ncols = ncols; a->nnz = nnz;
    auto bail = [&](cudaError_t e) {
        std::string m = cudaGetErrorString(e);
        pb_csr_destroy(a);
        return pb_fail_(PB_ECUDA, m);
    };
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e0)) != cudaSuccess) return bail(e);
    if ((e = cudaEventCreate(&a->e1)) != cudaSuccess) return bail(e);
    if ((e = a->alloc()) != cudaSuccess) return bail(e);
    const double mean = nrows ? (double)nnz / (double)nrows : 0.0;
    a->tpr = mean <= 3 ? 2 : mean <= 6 ? 4 : mean <= 24 ? 8 : mean <= 48 ? 16 : 32;
    *out = a;
    return PB_OK;
}
int32_t *pb_csr_indptr_(pb_csr *a) { return a->indptr; }
int32_t *pb_csr_indices_(pb_csr *a) { return a->indices; }
struct CsrView { int64_t nrows, ncols, nnz; int32_t *indptr, *indices; double *data; };
CsrView pb_csr_view_(const pb_csr *a) { return CsrView{a->nrows, a->ncols, a->nnz, a->indptr, a->indices, a->data}; }

extern "C" int pb_csr_spmv(pb_csr *a, const double *x, double *y) {
    if (!a || !x || !y) return pb_fail_(PB_EINVAL, "null pointer");
    CUDA_TRY(cudaMemcpyAsync(a->x, x, a->ncols * sizeof(double), cudaMemcpyHostToDevice, a->stream));
    int rc = launch_spmv(a, a->x, a->y, a->stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(y, a->y, a->nrows * sizeof(double), cudaMemcpyDeviceToHost, a->stream));
    CUDA_TRY(cudaStreamSynchronize(a->stream));
    return PB_OK;
}

extern "C" int pb_csr_spmv_dev(pb_csr *a, const double *x_dev, double *y_dev, uint64_t stream) {
    if (!a || !x_dev || !y_dev) return pb_fail_(PB_EINVAL, "null pointer");
    return launch_spmv(a, x_dev, y_dev, (cudaStream_t)stream);
}

// y = A x on device pointers, plus d1 += (w1, y) and d2 += (w2, y) (w2 == NULL with d2 != NULL: d2 += (y, y));
// d1 / d2 are device addresses (slots of the Krylov scalar buffer) or NULL
extern "C" int pb_csr_spmv_dots_dev(pb_csr *a, const double *x_dev, double *y_dev, const double *w1, double *d1,
                                    const double *w2, double *d2, uint64_t stream) {
    if (!a || !x_dev || !y_dev) return pb_fail_(PB_EINVAL, "null pointer");
    if (d1 && !w1) return pb_fail_(PB_EINVAL, "d1 needs w1");
    return launch_spmv_dots(a, x_dev, y_dev, w1, d1, w2, w2 == nullptr, d2, (cudaStream_t)stream);
}

extern "C" int pb_csr_spmv_bench(pb_csr *a, int reps, float *mean_ms) {
    if (!a || reps < 1 || !mean_ms) return pb_fail_(PB_EINVAL, "bad arguments");
    CUDA_TRY(cudaMemsetAsync(a->x, 0, a->ncols * sizeof(double), a->stream));
    for (int i = 0; i < 3; ++i) {
        int rc = launch_spmv(a, a->x, a->y, a->stream);
        if (rc) return rc;
    }
    CUDA_TRY(cudaEventRecord(a->e0, a->stream));
    for (int i = 0; i < reps; ++i) {
        int rc = launch_spmv(a, a->x, a->y, a->stream);
        if (rc) return rc;
    }
    CUDA_TRY(cudaEventRecord(a->e1, a->stream));
    CUDA_TRY(cudaEventSynchronize(a->e1));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, a->e0, a->e1));
    *mean_ms = ms / reps;
    return PB_OK;
}
