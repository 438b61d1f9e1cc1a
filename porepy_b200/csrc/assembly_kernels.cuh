// assembly_kernels.cuh -- the two __global__ entry points of the interaction-region assembly (one team
// of threads per grid node; node_kernels.cuh / mpsa_node.cuh hold the per-node routines).
#pragma once
#include "plan.hpp"

// ------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------
// shared memory of one team: [solver scratch | index lists, sub-cell products ... | A]
template <int ND, class Solver>
__global__ void __launch_bounds__(Solver::team == 32 ? 128 : Solver::team, Solver::min_blocks)
    mpfa_kernel(PlanView P, GeoView G, MpfaParams prm, MpfaOut o, const int32_t *__restrict__ nodes,
                int n_nodes, int scr_doubles, int rest_doubles, int a_doubles, double *a_ws, int *err) {
    extern __shared__ double smem[];
    constexpr int TEAM = Solver::team;
    GpuTeam<TEAM> t;
    const int teams_per_block = blockDim.x / TEAM;
    const int team_in_block = threadIdx.x / TEAM;
    double *scratch = smem;
    if (TEAM == 32) scratch += (size_t)team_in_block * (scr_doubles + rest_doubles + (a_ws ? 0 : a_doubles));
    double *rest = scratch + scr_doubles;
    double *A = a_ws ? a_ws + ((size_t)blockIdx.x * teams_per_block + team_in_block) * a_doubles
                     : rest + rest_doubles;
    for (int i = blockIdx.x * teams_per_block + team_in_block; i < n_nodes;
         i += gridDim.x * teams_per_block)
        mpfa_node<ND, Solver>(t, P, G, prm, o, (int64_t)nodes[i], A, rest, scratch, err);
}

template <int ND, class Solver>
__global__ void __launch_bounds__(Solver::team == 32 ? 128 : Solver::team, Solver::min_blocks)
    mpsa_kernel(PlanView P, GeoView G, MpsaParams prm, MpsaOut o, const int32_t *__restrict__ nodes,
                int n_nodes, int scr_doubles, int rest_doubles, int a_doubles, double *a_ws, int *err) {
    extern __shared__ double smem[];
    constexpr int TEAM = Solver::team;
    GpuTeam<TEAM> t;
    const int teams_per_block = blockDim.x / TEAM;
    const int team_in_block = threadIdx.x / TEAM;
    double *scratch = smem;
    if (TEAM == 32) scratch += (size_t)team_in_block * (scr_doubles + rest_doubles + (a_ws ? 0 : a_doubles));
    double *rest = scratch + scr_doubles;
    double *A = a_ws ? a_ws + ((size_t)blockIdx.x * teams_per_block + team_in_block) * a_doubles
                     : rest + rest_doubles;
    for (int i = blockIdx.x * teams_per_block + team_in_block; i < n_nodes;
         i += gridDim.x * teams_per_block) {
        const int inext = i + gridDim.x * teams_per_block;  // prefetched into L2 during this region's output phase
        const int64_t s_next = inext < n_nodes ? (int64_t)nodes[inext] : -1;
        mpsa_node<ND, Solver>(t, P, G, prm, o, (int64_t)nodes[i], A, rest, scratch, err, s_next);
    }
}

