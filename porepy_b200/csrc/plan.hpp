// plan.hpp -- state shared by the translation units of libporeb200.so: device buffers, the solver
// configurations, the plan handle and the per-class kernel launcher.  api.cu owns the C ABI; the
// kernel templates are instantiated in mpfa_launch.cu / mpsa2d.cu / mpsa3d.cu (one TU each so that
// they compile in parallel).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/poreb200.h"
#include "mpsa_node.cuh"
#include "face_kernels.cuh"
#include "node_kernels.cuh"
#include "plan_host.hpp"

int pb_fail_(int code, const std::string &msg);  // api.cu: sets pb_last_error()
void pb_count_launch_();                         // api.cu: pb_launch_count()
void pb_set_error_node_(int64_t node);           // api.cu: pb_last_error_node()
#define CUDA_TRY(x)                                                                        \
    do {                                                                                   \
        cudaError_t e_ = (x);                                                              \
        if (e_ != cudaSuccess)                                                             \
            return pb_fail_(PB_ECUDA, std::string(#x) + ": " + cudaGetErrorString(e_));    \
    } while (0)

using namespace pb;

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

// Solver configurations (node_kernels.cuh).  A node goes to the first one that fits.
using Cfg0 = TileGJ<1, 2, 6, 4>;   // team 32  : MPFA hexahedral nodes (12 x 45), DMMA, one warp per node
using Cfg1 = TileGJ<2, 3, 8, 6>;   // team 64  : MPSA hexahedral nodes (36 x 61), DMMA
using Cfg2 = TileGJ<2, 3, 12, 4>;  // team 64  : Biot hexahedral nodes, DMMA
using Cfg3 = TileGJ<5, 1, 18, 3>;  // team 160 : MPFA tetrahedral nodes (36 x 133), DMMA
using Cfg4 = TileGJ<7, 2, 24, 1>;  // team 224 : MPSA tetrahedral nodes (108 x 181), FP64 tensor cores (DMMA)
                                   // (TileGJ<14,1,24>: 448 threads, half the tile registers -- measured 7 % slower)
using Cfg5 = TileGJ<14, 1, 32, 1>; // team 448 : Biot tetrahedral nodes (108 x 205+), DMMA
using Cfg6 = SmemGJ;               // team 256 : anything else (in-memory Gauss-Jordan)
struct SolverCfg { int team, max_n, max_w; };
static const SolverCfg kCfg[] = {
    {Cfg0::team, Cfg0::max_n, Cfg0::max_w}, {Cfg1::team, Cfg1::max_n, Cfg1::max_w},
    {Cfg2::team, Cfg2::max_n, Cfg2::max_w}, {Cfg3::team, Cfg3::max_n, Cfg3::max_w},
    {Cfg4::team, Cfg4::max_n, Cfg4::max_w}, {Cfg5::team, Cfg5::max_n, Cfg5::max_w},
    {Cfg6::team, 1 << 30, 1 << 30},
};
static const int kNumCfg = 7;      // class key cfg * 2 + a_global: pb_plan_class_counts has 2 * kNumCfg entries
static const int kCatchAll = 6;

struct NodeClass {
    int cfg = 0;
    int team = 32;
    int n = 0;
    bool a_global = false;     // A lives in a global-memory workspace (does not fit shared memory)
    int64_t a_doubles = 0;     // per team
    int64_t rest_doubles = 0;  // per team
    int64_t scr_doubles = 0;   // per team (solver scratch, first in the team's region)
    DevBuf nodes;
};

struct pb_plan {
    HostPlan H;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    // plan arrays
    DevBuf fn_indptr, node_sc_ptr, sc_cell, node_sf_ptr, sf_face, sf_sides, sf_bloc, slot_sf, node_nb,
        sc_ncn, posfc_ptr, posfb_ptr, poscc_ptr, poscb_ptr, pos_fc, pos_fb, pos_cc, pos_cb, nbf_ptr, nbf_idx,
        cn_ptr, cn_idx, face_cells;
    DevBuf pat_ip[4], pat_idx[4];  // CSR of the structural pattern `which` (PB_PAT_*)
    DevBuf cf_ip, cf_ix, cf_sg;    // cell -> faces (CSC of cell_faces): the gather form of div_nd @ stress
    int64_t pat_rows[4] = {0, 0, 0, 0}, pat_cols[4] = {0, 0, 0, 0}, pat_nnz[4] = {0, 0, 0, 0};
    // geometry
    DevBuf nodes, fnorm, fcent, farea, ccent, cvol;
    bool have_geo = false;
    DevBuf cell_map;               // optional: cell e of this plan is cell cell_map[e] of a larger source grid
    int64_t cell_map_src = 0;      //           (cell tensors are then given for the source grid and gathered on the device)
    double node_key_sig = 0.0;
    std::vector<uint32_t> node_key;  // Morton key per node (set with the geometry): launch order of the node classes
    std::vector<uint8_t> active;   // per node: assemble its interaction region (empty = all); pb_plan_set_active_nodes
    PlanView view{};
    GeoView geo{};
    DevBuf err, a_ws, repack_tmp;
    // mpfa
    std::vector<NodeClass> mpfa_cls;
    DevBuf perm, bc, robw;
    bool have_robw = false;
    double eta = 0.0;
    bool mpfa_ready = false;
    DevBuf o_flux, o_bflux, o_bpc, o_bpf, o_vs, o_bpvs;
    // mpsa
    std::vector<NodeClass> mpsa_cls;
    int mpsa_cls_nalpha = -1;
    DevBuf stiff, vbc, vrobw, vbasis, alpha;
    bool have_vrobw = false, have_vbasis = false;
    int n_alpha = 0;
    double veta = 0.0;
    bool mpsa_ready = false;
    DevBuf o_stress, o_bstress, o_bdc, o_bdf;
    DevBuf o_dd[PB_MAX_ALPHA], o_bdd[PB_MAX_ALPHA], o_sg[PB_MAX_ALPHA], o_cons[PB_MAX_ALPHA],
        o_bdp[PB_MAX_ALPHA];
};


static const size_t kMaxSmem = 227 * 1024;
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


// launch one class with kernel template KERNEL<ND, Solver>
#define PB_LAUNCH_CFG(KERNEL, ND, ...)                                              \
    switch (c.cfg) {                                                                \
        case 0: rc = launch_one(KERNEL<ND, Cfg0>, c, p, __VA_ARGS__); break;        \
        case 1: rc = launch_one(KERNEL<ND, Cfg1>, c, p, __VA_ARGS__); break;        \
        case 2: rc = launch_one(KERNEL<ND, Cfg2>, c, p, __VA_ARGS__); break;        \
        case 3: rc = launch_one(KERNEL<ND, Cfg3>, c, p, __VA_ARGS__); break;        \
        case 4: rc = launch_one(KERNEL<ND, Cfg4>, c, p, __VA_ARGS__); break;        \
        case 5: rc = launch_one(KERNEL<ND, Cfg5>, c, p, __VA_ARGS__); break;        \
        default: rc = launch_one(KERNEL<ND, Cfg6>, c, p, __VA_ARGS__); break;       \
    }

template <class K, class Prm, class Out>
static int launch_one(K kernel, const NodeClass &c, pb_plan *p, const Prm &prm, const Out &o) {
    const int blk = c.team == 32 ? 128 : c.team;
    const int tpb = blk / c.team;
    const size_t smem = (size_t)(c.scr_doubles + c.rest_doubles + (c.a_global ? 0 : c.a_doubles)) *
                        sizeof(double) * tpb;
    if (smem > kMaxSmem)
        return pb_fail_(PB_ENOTIMPL, "interaction region needs " + std::to_string(smem) +
                                     " B of shared memory (> 227 KB)");
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // occupancy with the whole carve-out available (the preference set below stays with the kernel)
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutDefault));
    int per_sm = 1;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, blk, smem));
    if (per_sm < 1) per_sm = 1;
    // The part of the SM's 256 KB of unified memory that is not shared memory is L1, which holds the register
    // spills and the gathers of the node routines: ask for the smallest H100 shared-memory carve-out (KB) that keeps
    // per_sm CTAs, each with its 1 KB system reserve.  The percentage is rounded up to a carve-out by the driver.
    {
        static const int kCarveKB[] = {0, 8, 16, 32, 64, 100, 132, 164, 196, 228};
        const size_t need = (smem + 1024) * (size_t)per_sm;
        int pct = 100;
        for (int kb : kCarveKB)
            if ((size_t)kb * 1024 >= need) { pct = kb * 100 / 228; break; }
        CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    }
    int64_t need = ((int64_t)c.n + tpb - 1) / tpb;
    int grid = (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)pb_sm_count() * per_sm));
    double *ws = nullptr;
    if (c.a_global) {
        CUDA_TRY(p->a_ws.ensure((size_t)grid * tpb * c.a_doubles * sizeof(double)));
        ws = p->a_ws.as<double>();
    }
    kernel<<<grid, blk, smem, p->stream>>>(p->view, p->geo, prm, o, c.nodes.as<int32_t>(), c.n,
                                           (int)c.scr_doubles, (int)c.rest_doubles,
                                           (int)c.a_doubles, ws, p->err.as<int>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}


// kernel launches of all node classes of a plan (mpfa_launch.cu, mpsa2d.cu, mpsa3d.cu)
int pb_launch_mpfa_(pb_plan *p, const MpfaParams &prm, const MpfaOut &o);
int pb_launch_mpsa2_(pb_plan *p, const MpsaParams &prm, const MpsaOut &o);
int pb_launch_mpsa3_(pb_plan *p, const MpsaParams &prm, const MpsaOut &o);
// (ncomp, n) row-major host array -> entity-major records on the device (api.cu)
int pb_upload_repacked_(cudaStream_t st, DevBuf &tmp, DevBuf &dst, const double *host, int ncomp, int64_t n);
// sub-cell topology built on the device (plan_device.cu): 0 ok, > 0 error code (pb_fail_), -1 = fall back to the host
int pb_build_device_topology_(pb_plan *p, int nd, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr,
                              const int32_t *cf_indices, const int8_t *cf_data, const int32_t *fn_indptr,
                              const int32_t *fn_indices, DevBuf &fn_idx_dev);
