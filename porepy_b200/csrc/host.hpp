// host.hpp -- the host-side idioms every translation unit of libporeb200.so shares: error reporting, pooled device
// buffers, owners of CUDA streams and events, the kernel timer, grid sizing, the dimension dispatch and the internal
// interface of the device CSR matrix (spmv.cu).  Host code only: no kernel or device routine lives here.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/poreb200.h"

int pb_fail_(int code, const std::string &msg);  // api.cu: sets pb_last_error()
void pb_count_launch_();                         // api.cu: pb_launch_count()
void pb_set_error_node_(int64_t node);           // api.cu: pb_last_error_node()
#define CUDA_TRY(x)                                                                        \
    do {                                                                                   \
        cudaError_t e_ = (x);                                                              \
        if (e_ != cudaSuccess)                                                             \
            return pb_fail_(PB_ECUDA, std::string(#x) + ": " + cudaGetErrorString(e_));    \
    } while (0)

// PB_OK when a CUDA device is present; every entry point that creates a handle checks it first, since there is no
// CPU path in this library.
inline int pb_require_device() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1)
        return pb_fail_(PB_ECUDA, "no CUDA device: libporeb200 has no CPU path");
    return PB_OK;
}

// ------------------------------------------------------------------------------------
// device buffers
// ------------------------------------------------------------------------------------
// Freed device arrays are kept in a size-keyed pool (like the page-locked host pool of the Python layer): every
// discretize() of a model allocates and releases the same ~25 GB of value arrays, and cudaMalloc / cudaFree of such
// blocks cost tens of milliseconds each and synchronise the device.  POREB200_DEVICE_POOL_BYTES caps the pool
// (default 64 GiB; 0 disables it).
struct DevPool {
    std::mutex mu;
    std::multimap<size_t, void *> free_blocks;
    size_t held = 0, cap = 64ull << 30;
    DevPool() {
        if (const char *e = getenv("POREB200_DEVICE_POOL_BYTES")) cap = strtoull(e, nullptr, 10);
    }
    void *take(size_t n, size_t &got) {
        std::lock_guard<std::mutex> g(mu);
        // exact size only: a near fit takes a block that the next request of ITS size then misses (measured: two
        // slow re-discretizations, pb_plan_create 0.19-0.27 s instead of 0.045 s, until the pool had spares of every size)
        auto it = free_blocks.find(n);
        if (it == free_blocks.end()) return nullptr;
        void *q = it->second;
        got = it->first;
        free_blocks.erase(it);
        held -= got;
        return q;
    }
    bool give(void *q, size_t n) {
        std::lock_guard<std::mutex> g(mu);
        if (held + n > cap) return false;   // small blocks are pooled as well: their cudaMalloc / cudaFree pairs were
                                            // measured to stall sporadically (26 calls: 0.6 ms, or 230 ms once in four)
        free_blocks.emplace(n, q);
        held += n;
        return true;
    }
    void trim() {
        std::lock_guard<std::mutex> g(mu);
        for (auto &kv : free_blocks) cudaFree(kv.second);
        free_blocks.clear();
        held = 0;
    }
};
DevPool &pb_dev_pool_();  // api.cu
void pb_alloc_stat_(int kind, double seconds);   // api.cu: cudaMalloc (0) / cudaFree (1) calls that missed the pool

struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() {
        if (p && !pb_dev_pool_().give(p, bytes)) {
            const auto t0_ = std::chrono::steady_clock::now();
            cudaFree(p);
            pb_alloc_stat_(1, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0_).count());
        }
        p = nullptr;
        bytes = 0;
    }
    cudaError_t ensure(size_t n) {
        if (n <= bytes && p) return cudaSuccess;
        release();
        if (n == 0) n = 8;
        size_t got = 0;
        if ((p = pb_dev_pool_().take(n, got)) != nullptr) { bytes = got; return cudaSuccess; }
        const auto t0_ = std::chrono::steady_clock::now();
        cudaError_t e = cudaMalloc(&p, n);
        pb_alloc_stat_(0, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0_).count());
        if (e == cudaErrorMemoryAllocation) {   // give the pooled blocks back to the driver and retry once
            (void)cudaGetLastError();
            pb_dev_pool_().trim();
            e = cudaMalloc(&p, n);
        }
        if (e == cudaSuccess) bytes = n; else p = nullptr;
        return e;
    }
    template <class T>
    cudaError_t upload(const T *h, size_t count, cudaStream_t st) {
        cudaError_t e = ensure(count * sizeof(T));
        if (e != cudaSuccess) return e;
        if (count == 0) return cudaSuccess;
        return cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    template <class T>
    cudaError_t upload(const std::vector<T> &v, cudaStream_t st) { return upload(v.data(), v.size(), st); }
    template <class T>
    T *as() const { return (T *)p; }
};

// ------------------------------------------------------------------------------------
// streams, events and kernel timing
// ------------------------------------------------------------------------------------
// Move-only owner of a CUDA stream (non-blocking) or event, created by create() and destroyed with its owner.
// Destroying a stream does not wait for its work: a handle whose buffers may still be in use by that work
// synchronizes the stream in its own destructor first.
template <class H>
class CudaHandle {
  public:
    CudaHandle() = default;
    CudaHandle(CudaHandle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    CudaHandle &operator=(CudaHandle &&o) noexcept { std::swap(h_, o.h_); return *this; }
    ~CudaHandle() { if (h_) destroy(h_); }
    cudaError_t create() { return make(&h_); }
    operator H() const { return h_; }

  private:
    static cudaError_t make(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }
    static cudaError_t make(cudaEvent_t *e) { return cudaEventCreate(e); }
    static void destroy(cudaStream_t s) { cudaStreamDestroy(s); }
    static void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
    H h_ = nullptr;
};
using Stream = CudaHandle<cudaStream_t>;
using Event = CudaHandle<cudaEvent_t>;

// Device time between marks recorded on one stream: marks 0 and 1, and mark 2 for a two-stage timing.
struct KernelTimer {
    Event ev[3];
    cudaError_t create(int marks = 2) {
        for (int i = 0; i < marks; ++i)
            if (cudaError_t e = ev[i].create()) return e;
        return cudaSuccess;
    }
    cudaError_t mark(int i, cudaStream_t st) { return cudaEventRecord(ev[i], st); }
    // ms between marks i and i + 1; the later mark must have completed
    cudaError_t ms(float *out, int i = 0) const { return cudaEventElapsedTime(out, ev[i], ev[i + 1]); }
};

// ------------------------------------------------------------------------------------
// launch configuration
// ------------------------------------------------------------------------------------
// SMs of the current device: the cap of every grid-stride launch (H100 SXM 132, H100 PCIe 114)
inline int pb_sm_count() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (!cache[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 1;
        cache[dev] = n;
    }
    return cache[dev];
}

// Blocks of a grid-stride launch over n items, per_block items per block: enough to cover n, at most waves_per_sm
// blocks per SM, at least one.  Kernels that accumulate with atomics depend on this exact count for bit-identical
// results, so every grid-stride launch sizes its grid here.
inline int grid_stride_blocks(int64_t n, int64_t per_block, int64_t waves_per_sm) {
    return (int)std::max<int64_t>(1, std::min<int64_t>((n + per_block - 1) / per_block,
                                                       (int64_t)pb_sm_count() * waves_per_sm));
}

// Calls f(std::integral_constant<int, ND>{}) for the ND of the list that equals nd, or for the last one when none does,
// and returns what f returns: a launch site names its kernel<ND> once.
template <int ND, int... More, class F>
inline decltype(auto) dispatch_nd(int nd, F &&f) {
    if constexpr (sizeof...(More) == 0) {
        return f(std::integral_constant<int, ND>{});
    } else {
        if (nd == ND) return f(std::integral_constant<int, ND>{});
        return dispatch_nd<More...>(nd, std::forward<F>(f));
    }
}

// ------------------------------------------------------------------------------------
// the device CSR matrix (spmv.cu) inside the library
// ------------------------------------------------------------------------------------
struct pb_csr;
struct CsrView { int64_t nrows, ncols, nnz; int32_t *indptr, *indices; double *data; };
CsrView pb_csr_view_(const pb_csr *a);
// a result matrix under construction: destroyed unless released to the caller
struct CsrDeleter { void operator()(pb_csr *a) const; };
using CsrPtr = std::unique_ptr<pb_csr, CsrDeleter>;
// an empty matrix of the given sizes, for a builder that fills indptr / indices / data
int pb_csr_alloc_(int64_t nrows, int64_t ncols, int64_t nnz, CsrPtr &out);
// a matrix whose pattern is copied from device arrays and whose values (zeroed) the caller fills
int pb_csr_from_device_pattern_(int64_t nrows, int64_t ncols, int64_t nnz, const int32_t *indptr_dev,
                                const int32_t *indices_dev, CsrPtr &out);
