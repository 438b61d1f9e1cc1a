// csr_build_harness.cu -- TEST INFRASTRUCTURE ONLY (never loaded by the product).  Runs the shared steps of the device
// CSR builders in porepy_b200/csrc/csr_build.cuh on caller-supplied data: the offset scan (both offset types, on a
// non-blocking stream or the legacy default stream), and the warp bitonic sort with a payload followed by the
// unique-compaction, for the key types the library sorts (int32 row / column keys, 64-bit (cell, face) keys).
//
// The header reports errors and counts launches through functions that live in api.cu; this file defines its own.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../porepy_b200/csrc/csr_build.cuh"

namespace {
std::string g_err;
int64_t g_launches = 0;
}  // namespace

int pb_fail_(int code, const std::string &msg) { g_err = msg; return code; }
void pb_count_launch_() { ++g_launches; }
DevPool &pb_dev_pool_() { static DevPool *pool = new DevPool; return *pool; }
void pb_alloc_stat_(int, double) {}

namespace {

template <class K>
struct Pad;
template <>
struct Pad<int32_t> { static constexpr int32_t v = 0x7fffffff; };
template <>
struct Pad<uint64_t> { static constexpr uint64_t v = ~0ull; };

// one warp: sort keys[0..n) with their payload, then compact the sorted keys into uniq[0..*nuniq)
template <class K>
__global__ void sort_unique_kernel(int n, int P, K *keys, double *pay, K *uniq, int *nuniq) {
    extern __shared__ double sm[];
    double *v = sm;                // the doubles first: 8-byte aligned whatever P is
    K *k = (K *)(sm + P);
    for (int i = threadIdx.x; i < P; i += 32) {
        k[i] = i < n ? keys[i] : Pad<K>::v;
        v[i] = i < n ? pay[i] : 0.0;
    }
    __syncwarp();
    warp_bitonic_sort(P, [&](int i, int l, bool asc) {
        if (warp_cas(k, i, l, asc)) { const double t = v[i]; v[i] = v[l]; v[l] = t; }
    });
    for (int i = threadIdx.x; i < n; i += 32) { keys[i] = k[i]; pay[i] = v[i]; }
    const int cnt = warp_unique(k, n, k);   // in place, as the topology kernel does
    for (int i = threadIdx.x; i < cnt; i += 32) uniq[i] = k[i];
    if (threadIdx.x == 0) *nuniq = cnt;
}

#define CB_TRY(x)                                                                              \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) { g_err = std::string(#x) + ": " + cudaGetErrorString(e_); return PB_ECUDA; } \
    } while (0)

template <class OffT>
int scan(const int32_t *counts, int64_t n, int legacy_stream, OffT *offsets, int64_t *total) {
    cudaStream_t st = nullptr;
    if (!legacy_stream) CB_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    DevBuf c, o;
    int rc = PB_ECUDA;
    if (c.upload(counts, (size_t)n, st) == cudaSuccess && o.ensure((size_t)(n + 1) * sizeof(OffT)) == cudaSuccess) {
        rc = pb_scan_offsets_(c.as<int32_t>(), o.as<OffT>(), n, st, total);
        if (!rc && cudaMemcpy(offsets, o.p, (size_t)(n + 1) * sizeof(OffT), cudaMemcpyDeviceToHost) != cudaSuccess) {
            g_err = "download of the offsets";
            rc = PB_ECUDA;
        }
    } else {
        g_err = "upload of the counts";
    }
    if (st) cudaStreamDestroy(st);
    return rc;
}

template <class K>
int sort_unique(int n, K *keys, double *pay, K *uniq, int *nuniq) {
    int P = 1;
    while (P < n) P <<= 1;
    const size_t smem = (size_t)P * (sizeof(K) + sizeof(double));
    DevBuf dk, dp, du, dn;
    CB_TRY(dk.upload(keys, (size_t)n, 0));
    CB_TRY(dp.upload(pay, (size_t)n, 0));
    CB_TRY(du.ensure((size_t)n * sizeof(K)));
    CB_TRY(dn.ensure(sizeof(int)));
    CB_TRY(cudaFuncSetAttribute(sort_unique_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sort_unique_kernel<K><<<1, 32, smem>>>(n, P, dk.as<K>(), dp.as<double>(), du.as<K>(), dn.as<int>());
    CB_TRY(cudaGetLastError());
    CB_TRY(cudaMemcpy(keys, dk.p, (size_t)n * sizeof(K), cudaMemcpyDeviceToHost));
    CB_TRY(cudaMemcpy(pay, dp.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
    CB_TRY(cudaMemcpy(nuniq, dn.p, sizeof(int), cudaMemcpyDeviceToHost));
    CB_TRY(cudaMemcpy(uniq, du.p, (size_t)*nuniq * sizeof(K), cudaMemcpyDeviceToHost));
    return PB_OK;
}

}  // namespace

extern "C" {

const char *cb_last_error(void) { return g_err.c_str(); }
int64_t cb_launches(void) { return g_launches; }

// offsets (n + 1 entries of int32, or of int64 with off64) = exclusive scan of counts; *total = the exact sum
int cb_scan(int off64, int legacy_stream, const int32_t *counts, int64_t n, void *offsets, int64_t *total) {
    g_err.clear();
    return off64 ? scan(counts, n, legacy_stream, (int64_t *)offsets, total)
                 : scan(counts, n, legacy_stream, (int32_t *)offsets, total);
}

// keys (int32, or uint64 with key64) and pay sorted in place by key; uniq[0..*nuniq) = the unique keys.  n >= 1.
int cb_sort_unique(int key64, int n, void *keys, double *pay, void *uniq, int *nuniq) {
    g_err.clear();
    return key64 ? sort_unique(n, (uint64_t *)keys, pay, (uint64_t *)uniq, nuniq)
                 : sort_unique(n, (int32_t *)keys, pay, (int32_t *)uniq, nuniq);
}

}  // extern "C"
