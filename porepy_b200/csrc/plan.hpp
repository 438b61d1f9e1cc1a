// plan.hpp -- the solver configurations, the plan handle and the per-class kernel launcher.  api.cu owns the C ABI;
// the kernel templates are instantiated in mpfa_launch.cu / mpsa2d.cu / mpsa3d.cu (one TU each so that they compile in
// parallel).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/poreb200.h"
#include "mpsa_node.cuh"
#include "face_kernels.cuh"
#include "node_kernels.cuh"
#include "host.hpp"
#include "plan_host.hpp"

using namespace pb;

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
    Stream stream;
    KernelTimer timer;             // pb_mpfa_assemble / pb_mpsa_assemble
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
    // the stream's copies and kernels may still use the buffers, which go back to the pool right after
    ~pb_plan() { if (stream) cudaStreamSynchronize(stream); }
};

static const size_t kMaxSmem = 227 * 1024;

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
    const int grid = grid_stride_blocks(c.n, tpb, per_sm);
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
