// peaks.cu -- FP64 peak microbenchmarks for the roofline denominators of the assembly kernels (SURVEY.md 8d: "measure
// achieved peaks").  Dependency-free register loops: the FP64 tensor pipe (mma.sync .f64 in each shape sm_90 has:
// m8n8k4, m16n8k4, m16n8k8, m16n8k16) and scalar DFMA.  One persistent wave: the device's SMs x 8 CTAs.
#include "plan.hpp"

__global__ void __launch_bounds__(256) dmma_peak_kernel(int iters, double *sink) {
    double c[8][2];
#pragma unroll
    for (int t = 0; t < 8; ++t) { c[t][0] = threadIdx.x * 1e-9; c[t][1] = t * 1e-9; }
    const double a = 1.0 + threadIdx.x * 1e-12, b = 1.0 - threadIdx.x * 1e-12;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int t = 0; t < 8; ++t) pb_dmma(c[t], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int t = 0; t < 8; ++t) s += c[t][0] + c[t][1];
    if (s == 123.456) sink[0] = s;  // never true: keeps the loop alive
}

// mma.sync.m16n8k{K}.f64: A K/4 doubles, B K/8 (k4: 1) doubles, C 4 doubles per lane; 8 independent accumulators
template <int K>
__global__ void __launch_bounds__(256) dmma16_peak_kernel(int iters, double *sink) {
    double c[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
        for (int q = 0; q < 4; ++q) c[t][q] = threadIdx.x * 1e-9 + q * 1e-10 + t * 1e-9;
    const double a = 1.0 + threadIdx.x * 1e-12, b = 1.0 - threadIdx.x * 1e-12;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            if constexpr (K == 4) {
                asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                             : "+d"(c[t][0]), "+d"(c[t][1]), "+d"(c[t][2]), "+d"(c[t][3]) : "d"(a), "d"(b), "d"(a));
            } else if constexpr (K == 8) {
                asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                             "{%0,%1,%2,%3};"
                             : "+d"(c[t][0]), "+d"(c[t][1]), "+d"(c[t][2]), "+d"(c[t][3])
                             : "d"(a), "d"(b), "d"(a), "d"(b), "d"(a), "d"(b));
            } else {
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                             "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                             : "+d"(c[t][0]), "+d"(c[t][1]), "+d"(c[t][2]), "+d"(c[t][3])
                             : "d"(a), "d"(b), "d"(a), "d"(b), "d"(a), "d"(b), "d"(a), "d"(b),
                               "d"(a), "d"(b), "d"(a), "d"(b));
            }
        }
    }
    double s = 0.0;
#pragma unroll
    for (int t = 0; t < 8; ++t) s += c[t][0] + c[t][1] + c[t][2] + c[t][3];
    if (s == 123.456) sink[0] = s;
}

__global__ void __launch_bounds__(256) dfma_peak_kernel(int iters, double *sink) {
    double x[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) x[t] = threadIdx.x * 1e-9 + t;
    const double a = 1.0 - 1e-12, b = 1e-13;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int t = 0; t < 8; ++t) x[t] = fma(x[t], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int t = 0; t < 8; ++t) s += x[t];
    if (s == 123.456) sink[0] = s;
}

// kind 0: DMMA m8n8k4 (512 flops per warp instruction), 1: DFMA (2 flops per thread instruction), 2 / 3 / 4: DMMA
// m16n8k4 / m16n8k8 / m16n8k16 (1024 / 2048 / 4096 flops per warp instruction).  Best of 5 launches.
extern "C" int pb_fp64_peak(int kind, double *tflops) {
    if (!tflops || kind < 0 || kind > 4) return pb_fail_(PB_EINVAL, "bad arguments");
    DevBuf sink;
    CUDA_TRY(sink.ensure(8));
    KernelTimer timer;
    CUDA_TRY(timer.create());
    const int iters = 1 << 15, block = 256, grid = pb_sm_count() * 8;
    double best = 0.0;
    for (int rep = 0; rep < 6; ++rep) {
        CUDA_TRY(timer.mark(0, 0));
        if (kind == 0) dmma_peak_kernel<<<grid, block>>>(iters, sink.as<double>());
        else if (kind == 1) dfma_peak_kernel<<<grid, block>>>(iters, sink.as<double>());
        else if (kind == 2) dmma16_peak_kernel<4><<<grid, block>>>(iters, sink.as<double>());
        else if (kind == 3) dmma16_peak_kernel<8><<<grid, block>>>(iters, sink.as<double>());
        else dmma16_peak_kernel<16><<<grid, block>>>(iters, sink.as<double>());
        CUDA_TRY(timer.mark(1, 0));
        CUDA_TRY(cudaEventSynchronize(timer.ev[1]));
        pb_count_launch_();
        float ms = 0.f;
        CUDA_TRY(timer.ms(&ms));
        const double per_thread_instr = (double)iters * 8;
        const double per_warp_instr[5] = {512.0, 0.0, 1024.0, 2048.0, 4096.0};
        const double flops = kind == 1 ? per_thread_instr * (grid * (double)block) * 2.0
                                       : per_thread_instr * (grid * (double)block / 32) * per_warp_instr[kind];
        if (rep > 0) best = std::max(best, flops / (ms * 1e-3) / 1e12);
    }
    *tflops = best;
    return PB_OK;
}
