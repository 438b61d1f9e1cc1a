// csr_build.cuh -- the steps shared by the compressed-row structures built on the device (the plan's patterns and
// sub-cell topology, the AD-chain sparse algebra, the Tpsa system patterns): row counts scanned into row offsets, and
// the per-warp sort and unique-compaction of a row's candidate entries in shared memory.
#pragma once
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>

#include <type_traits>

#include "plan.hpp"

struct PbWiden {
    __host__ __device__ long long operator()(int32_t v) const { return v; }
};

// offsets[0..n] = exclusive scan of counts[0..n) on stream st, so offsets[n] is the sum; *total = the exact sum, also
// when it does not fit OffT.  The sums are accumulated in 64 bits: an int32 accumulation would wrap silently, and the
// caller checks *total against its own index limit before it trusts the offsets.  Synchronises st.
template <class OffT>
int pb_scan_offsets_(const int32_t *counts, OffT *offsets, int64_t n, cudaStream_t st, int64_t *total) {
    static_assert(std::is_same<OffT, int32_t>::value || std::is_same<OffT, int64_t>::value, "int32 or int64 offsets");
    const auto wide = thrust::make_transform_iterator(counts, PbWiden{});
    DevBuf tmp, sum;
    CUDA_TRY(sum.ensure(sizeof(long long)));
    size_t scan_bytes = 0, sum_bytes = 0;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, wide, offsets + 1, n, st));
    CUDA_TRY(cub::DeviceReduce::Sum(nullptr, sum_bytes, wide, sum.as<long long>(), n, st));
    CUDA_TRY(tmp.ensure(std::max(scan_bytes, sum_bytes)));
    CUDA_TRY(cudaMemsetAsync(offsets, 0, sizeof(OffT), st));
    CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp.p, scan_bytes, wide, offsets + 1, n, st));
    CUDA_TRY(cub::DeviceReduce::Sum(tmp.p, sum_bytes, wide, sum.as<long long>(), n, st));
    pb_count_launch_();
    long long t = 0;
    CUDA_TRY(cudaMemcpyAsync(&t, sum.p, sizeof(t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *total = t;
    return PB_OK;
}

// Compare-and-swap of key[i] and key[l] (i < l) into ascending (asc) or descending order; true when they were swapped.
template <class K>
__device__ __forceinline__ bool warp_cas(K *key, int i, int l, bool asc) {
    const K a = key[i], c = key[l];
    if ((a > c) != asc) return false;
    key[i] = c;
    key[l] = a;
    return true;
}

// Bitonic sorting network over the power-of-two span [0, P) in shared memory, run by the 32 lanes of one warp: calls
// cas(i, l, asc) for every compare-and-swap of the network, one stage at a time.  cas sorts the keys with warp_cas and
// moves whatever payload goes with them; the order of equal keys is arbitrary.  Pad [n, P) with a key above all others.
template <class Cas>
__device__ __forceinline__ void warp_bitonic_sort(int P, Cas cas) {
    const int lane = threadIdx.x & 31;
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
                const int l = i ^ j;
                if (l > i) cas(i, l, (i & k) == 0);
            }
            __syncwarp();
        }
}

// Ballot compaction of the sorted span key[0..n) into its unique keys, written to out[0..count) (out may be key
// itself: a write never lands behind its source index; nullptr only counts).  Returns the count on every lane.
template <class K>
__device__ __forceinline__ int warp_unique(const K *key, int n, K *out) {
    const int lane = threadIdx.x & 31;
    int cnt = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const bool flag = i < n && (i == 0 || key[i] != key[i - 1]);
        const K v = i < n ? key[i] : K(0);
        const unsigned m = __ballot_sync(0xffffffffu, flag);
        __syncwarp();
        if (flag && out) out[cnt + __popc(m & ((1u << lane) - 1u))] = v;
        cnt += __popc(m);
        __syncwarp();
    }
    return cnt;
}

// Structural patterns on the device: row r = sorted union over the nodes of row entity r of the
// node's column entities.  One warp per row: gather the (<= CAP) candidates into shared memory,
// bitonic sort, unique.  pass 0 writes the row length, pass 1 the indices.
template <int CAP>
__global__ void pattern_kernel(int64_t nrows, const int32_t *__restrict__ rn_ptr, const int32_t *__restrict__ rn,
                               const int32_t *__restrict__ col_ptr, const int32_t *__restrict__ col_idx,
                               int32_t *__restrict__ counts, const int32_t *__restrict__ indptr,
                               int32_t *__restrict__ indices, int pass, int *overflow) {
    __shared__ int32_t sbuf[8][CAP];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    int32_t *buf = sbuf[wib];
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + wib;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int total = 0;
        bool over = false;
        for (int q = rn_ptr[r]; q < rn_ptr[r + 1]; ++q) {
            const int s = rn[q];
            const int b = col_ptr[s], len = col_ptr[s + 1] - b;
            if (total + len > CAP) { over = true; break; }
            for (int i = lane; i < len; i += 32) buf[total + i] = col_idx[b + i];
            total += len;
        }
        if (over) {
            if (lane == 0) { atomicExch(overflow, 1); if (pass == 0) counts[r] = 0; }
            continue;
        }
        int P = 1;
        while (P < total) P <<= 1;
        for (int i = total + lane; i < P; i += 32) buf[i] = 0x7fffffff;
        __syncwarp();
        warp_bitonic_sort(P, [&](int i, int l, bool asc) { warp_cas(buf, i, l, asc); });
        const int off = warp_unique(buf, total, pass == 1 ? indices + indptr[r] : (int32_t *)nullptr);
        if (pass == 0 && lane == 0) counts[r] = off;
        __syncwarp();
    }
}
