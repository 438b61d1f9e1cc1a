// solver_harness.cu -- TEST INFRASTRUCTURE ONLY (never loaded by the product).  Runs the dense local solvers of
// porepy_b200/csrc/node_kernels.cuh on caller-supplied augmented matrices, one kernel per solver configuration
// Cfg0..Cfg7 of plan.hpp, so that tests/test_zz_local_solvers_gpu.py checks exactly the types the library compiles.
//
// The launch mirrors launch_one (plan.hpp) and the assembly kernels (assembly_kernels.cuh): 32-thread teams run four
// to a 128-thread CTA at per-team offsets of the dynamic shared memory, larger teams one per CTA; the grid is capped
// at (SM count) x (occupancy) and every team walks its systems with a grid-stride loop, reusing its shared memory.
// Per team the shared memory is [solver scratch | row index | A] (A in a global workspace when a_global).
//
// Each system i occupies A_io[a_off[i] .. a_off[i+1]) (row stride W[i]; the doubles past n[i]*W[i] are a guard
// region).  The team copies the whole span in, solves, and copies it back, so that writes outside the system show up
// in the caller's sentinels.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../porepy_b200/csrc/plan.hpp"

namespace {

std::string g_err;

template <class Solver>
__global__ void __launch_bounds__(Solver::team == 32 ? 128 : Solver::team, Solver::min_blocks)
    solve_kernel(int nsys, const int *__restrict__ n_, const int *__restrict__ nrhs_, const int *__restrict__ W_,
                 const int64_t *__restrict__ a_off, const int64_t *__restrict__ r_off, double *A_io, int *rowidx_out,
                 int *ok_out, int scr_doubles, int idx_doubles, int64_t a_doubles, double *a_ws) {
    extern __shared__ double smem[];
    constexpr int TEAM = Solver::team;
    GpuTeam<TEAM> t;
    const int teams_per_block = blockDim.x / TEAM;
    const int team_in_block = threadIdx.x / TEAM;
    double *scratch = smem;
    if (TEAM == 32) scratch += (size_t)team_in_block * (scr_doubles + idx_doubles + (a_ws ? 0 : a_doubles));
    int *rowidx = (int *)(scratch + scr_doubles);
    double *A = a_ws ? a_ws + ((size_t)blockIdx.x * teams_per_block + team_in_block) * a_doubles
                     : scratch + scr_doubles + idx_doubles;
    for (int i = blockIdx.x * teams_per_block + team_in_block; i < nsys; i += gridDim.x * teams_per_block) {
        const int n = n_[i], nrhs = nrhs_[i], W = W_[i];
        const int64_t off = a_off[i], len = a_off[i + 1] - a_off[i];
        for (int64_t k = t.tid(); k < len; k += t.size()) A[k] = A_io[off + k];
        for (int k = t.tid(); k < n; k += t.size()) rowidx[k] = k;
        t.sync();
        const bool ok = Solver::solve(t, A, n, W, nrhs, rowidx, scratch);
        t.sync();
        for (int64_t k = t.tid(); k < len; k += t.size()) A_io[off + k] = A[k];
        for (int k = t.tid(); k < n; k += t.size()) rowidx_out[r_off[i] + k] = rowidx[k];
        if (t.tid() == 0) ok_out[i] = ok ? 1 : 0;
        t.sync();
    }
}

template <class Solver>
int64_t scratch_of(int n) {
    (void)n;
    return Solver::scratch_doubles_c();
}
template <>
int64_t scratch_of<Cfg6>(int n) {
    return Cfg6::scratch_doubles(n);
}

#define HS_TRY(x)                                                                              \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) {                                                               \
            g_err = std::string(#x) + ": " + cudaGetErrorString(e_);                           \
            goto done;                                                                         \
        }                                                                                      \
    } while (0)

template <class Solver>
int run(int a_global, int nsys, const int *n, const int *nrhs, const int *W, const int64_t *a_off, double *A,
        int *rowidx, int *ok) {
    constexpr int team = Solver::team;
    const int blk = team == 32 ? 128 : team;
    const int tpb = blk / team;
    int max_n = 1;
    int64_t max_span = 1;
    std::vector<int64_t> r_off(nsys + 1, 0);
    for (int i = 0; i < nsys; ++i) {
        max_n = std::max(max_n, n[i]);
        max_span = std::max<int64_t>(max_span, a_off[i + 1] - a_off[i]);
        r_off[i + 1] = r_off[i] + n[i];
    }
    const int64_t scr = scratch_of<Solver>(max_n);
    const int idx = (max_n + 1) / 2;  // int rowidx[max_n] in doubles
    const size_t smem = (size_t)(scr + idx + (a_global ? 0 : max_span)) * sizeof(double) * tpb;
    if (smem > kMaxSmem) {
        g_err = "systems need " + std::to_string(smem) + " B of shared memory (> 227 KB)";
        return 1;
    }
    int rc = 1, per_sm = 1, grid = 1;
    int *d_n = nullptr, *d_nrhs = nullptr, *d_W = nullptr, *d_ridx = nullptr, *d_ok = nullptr;
    int64_t *d_aoff = nullptr, *d_roff = nullptr;
    double *d_A = nullptr, *d_ws = nullptr;
    const int64_t total = a_off[nsys];
    HS_TRY(cudaFuncSetAttribute(solve_kernel<Solver>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    HS_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, solve_kernel<Solver>, blk, smem));
    if (per_sm < 1) per_sm = 1;
    grid = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)nsys + tpb - 1) / tpb, (int64_t)pb_sm_count() * per_sm));
    HS_TRY(cudaMalloc(&d_n, sizeof(int) * nsys));
    HS_TRY(cudaMalloc(&d_nrhs, sizeof(int) * nsys));
    HS_TRY(cudaMalloc(&d_W, sizeof(int) * nsys));
    HS_TRY(cudaMalloc(&d_ok, sizeof(int) * nsys));
    HS_TRY(cudaMalloc(&d_ridx, sizeof(int) * std::max<int64_t>(1, r_off[nsys])));
    HS_TRY(cudaMalloc(&d_aoff, sizeof(int64_t) * (nsys + 1)));
    HS_TRY(cudaMalloc(&d_roff, sizeof(int64_t) * (nsys + 1)));
    HS_TRY(cudaMalloc(&d_A, sizeof(double) * std::max<int64_t>(1, total)));
    if (a_global) HS_TRY(cudaMalloc(&d_ws, sizeof(double) * (size_t)grid * tpb * max_span));
    HS_TRY(cudaMemcpy(d_n, n, sizeof(int) * nsys, cudaMemcpyHostToDevice));
    HS_TRY(cudaMemcpy(d_nrhs, nrhs, sizeof(int) * nsys, cudaMemcpyHostToDevice));
    HS_TRY(cudaMemcpy(d_W, W, sizeof(int) * nsys, cudaMemcpyHostToDevice));
    HS_TRY(cudaMemcpy(d_aoff, a_off, sizeof(int64_t) * (nsys + 1), cudaMemcpyHostToDevice));
    HS_TRY(cudaMemcpy(d_roff, r_off.data(), sizeof(int64_t) * (nsys + 1), cudaMemcpyHostToDevice));
    HS_TRY(cudaMemcpy(d_A, A, sizeof(double) * total, cudaMemcpyHostToDevice));
    HS_TRY(cudaMemset(d_ok, 0xff, sizeof(int) * nsys));   // -1: the system was never visited
    solve_kernel<Solver><<<grid, blk, smem>>>(nsys, d_n, d_nrhs, d_W, d_aoff, d_roff, d_A, d_ridx, d_ok, (int)scr,
                                              idx, max_span, d_ws);
    HS_TRY(cudaGetLastError());
    HS_TRY(cudaDeviceSynchronize());
    HS_TRY(cudaMemcpy(A, d_A, sizeof(double) * total, cudaMemcpyDeviceToHost));
    HS_TRY(cudaMemcpy(rowidx, d_ridx, sizeof(int) * r_off[nsys], cudaMemcpyDeviceToHost));
    HS_TRY(cudaMemcpy(ok, d_ok, sizeof(int) * nsys, cudaMemcpyDeviceToHost));
    rc = 0;
done:
    cudaFree(d_n); cudaFree(d_nrhs); cudaFree(d_W); cudaFree(d_ok); cudaFree(d_ridx);
    cudaFree(d_aoff); cudaFree(d_roff); cudaFree(d_A); cudaFree(d_ws);
    return rc;
}

}  // namespace

extern "C" {

const char *sh_last_error(void) { return g_err.c_str(); }

// team size, largest n and largest row stride W the dispatcher sends to configuration cfg (kCfg of plan.hpp)
int sh_limits(int cfg, int *team, int *max_n, int *max_w) {
    if (cfg < 0 || cfg >= kNumCfg) { g_err = "no such configuration"; return 1; }
    *team = kCfg[cfg].team;
    *max_n = kCfg[cfg].max_n;
    *max_w = kCfg[cfg].max_w;
    return 0;
}

// 1 when a batch of systems of order <= max_n and spans <= span doubles fits the shared memory of configuration cfg
int sh_fits_shared(int cfg, int max_n, int64_t span) {
    int64_t scr = 0;
    switch (cfg) {
        case 0: scr = Cfg0::scratch_doubles_c(); break;
        case 1: scr = Cfg1::scratch_doubles_c(); break;
        case 2: scr = Cfg2::scratch_doubles_c(); break;
        case 3: scr = Cfg3::scratch_doubles_c(); break;
        case 4: scr = Cfg4::scratch_doubles_c(); break;
        case 5: scr = Cfg5::scratch_doubles_c(); break;
        case 6: scr = Cfg6::scratch_doubles(max_n); break;
        case 7: scr = Cfg7::scratch_doubles_c(); break;
        default: return 0;
    }
    const int tpb = kCfg[cfg].team == 32 ? 4 : 1;
    return (size_t)(scr + (max_n + 1) / 2 + span) * sizeof(double) * tpb <= kMaxSmem ? 1 : 0;
}

// Solves nsys systems in one launch.  System i: n[i] x n[i] matrix and nrhs[i] right-hand sides, row stride W[i],
// stored at A[a_off[i] ..) (a_off has nsys + 1 entries; the span may extend past n*W as a guard).  On return A holds
// what the solver left there, rowidx[sum(n[:i]) + p] the physical row of pivot p and ok[i] the solver's verdict.
// Returns 0, or 1 with the reason in sh_last_error().
int sh_solve(int cfg, int a_global, int nsys, const int *n, const int *nrhs, const int *W, const int64_t *a_off,
             double *A, int *rowidx, int *ok) {
    g_err.clear();
    if (nsys < 1) { g_err = "no systems"; return 1; }
    switch (cfg) {
        case 0: return run<Cfg0>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 1: return run<Cfg1>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 2: return run<Cfg2>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 3: return run<Cfg3>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 4: return run<Cfg4>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 5: return run<Cfg5>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 6: return run<Cfg6>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        case 7: return run<Cfg7>(a_global, nsys, n, nrhs, W, a_off, A, rowidx, ok);
        default: g_err = "no such configuration"; return 1;
    }
}

}  // extern "C"
