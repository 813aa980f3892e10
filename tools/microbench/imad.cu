// Integer-pipe microbenchmark for sm_90a: what does a 32x32 multiply cost in each SASS form?
// Prints warp-instructions per clock per SM for independent chains of each op.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "ffu.cuh"  // the measured-and-rejected carry-free prototype lives next to its microbenchmark
using namespace bzk;

#define ITERS 4096
#define CHAINS 8

template <int OP>
__global__ void __launch_bounds__(256) k(uint32_t *out, uint32_t seed, long long *cycles) {
    uint32_t a[CHAINS], b[CHAINS], c[CHAINS];
    uint64_t w[CHAINS];
    double d[CHAINS];
    for (int i = 0; i < CHAINS; i++) { a[i] = seed + threadIdx.x * 7 + i; b[i] = seed * 3 + i * 5 + 1; c[i] = i; w[i] = i; d[i] = 1.0 + i; }
    long long t0 = clock64();
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < CHAINS; i++) {
            if (OP == 0) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(c[i]) : "r"(a[i]), "r"(b[i]));
            if (OP == 1) asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(c[i]) : "r"(a[i]), "r"(b[i]));
            if (OP == 2) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(b[i]));
            if (OP == 3) asm volatile("add.u32 %0, %0, %1;" : "+r"(c[i]) : "r"(a[i]));
            if (OP == 4) asm volatile("fma.rn.f64 %0, %0, %1, %0;" : "+d"(d[i]) : "d"(1.0000001));
            if (OP == 5) {  // lo+hi pair with carry chain (what ff.cuh emits)
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(c[i]), "+r"(a[i]) : "r"(b[i]), "r"(seed));
            }
            if (OP == 6) {  // imad + iadd3 mixed 1:1 (do they dual-issue on different pipes?)
                asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(c[i]) : "r"(a[i]), "r"(b[i]));
                asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b[i]));
            }
            if (OP == 7) asm volatile("mul.lo.u32 %0, %1, %0;" : "+r"(c[i]) : "r"(a[i]));
            if (OP == 8) {  // 16x16->32 via mul24? (IMAD on 16-bit operands: same pipe)
                asm volatile("mul24.lo.u32 %0, %1, %0;" : "+r"(c[i]) : "r"(a[i]));
            }
            if (OP == 9) asm volatile("fma.rn.f32 %0, %0, %1, %0;" : "+f"(*(float *)&c[i]) : "f"(1.0001f));
        }
    }
    long long t1 = clock64();
    uint32_t s = 0;
    for (int i = 0; i < CHAINS; i++) s += c[i] + a[i] + (uint32_t)w[i] + (uint32_t)(w[i] >> 32) + (uint32_t)d[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

// compute-bound field multiplication: each thread squares-and-multiplies in registers
template <class F, int MODE>
__global__ void __launch_bounds__(256) kmul(F *out, const F *in, int iters, long long *cycles) {
    F x = in[threadIdx.x + blockIdx.x * blockDim.x], y = in[(threadIdx.x + 1) % 256];
    long long t0 = clock64();
    for (int i = 0; i < iters; i++) {
        if (MODE == 0) { x = x * y; y = y * x; }
        if (MODE == 1) { x = x + y; y = y - x; }
    }
    long long t1 = clock64();
    out[threadIdx.x + blockIdx.x * blockDim.x] = x + y;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int OP>
void run(const char *name, int ops_per_iter, int warps_per_sm_list[], int nl) {
    uint32_t *out; long long *cyc, h;
    cudaMalloc(&out, 148 * 64 * 256 * 4); cudaMalloc(&cyc, 8);
    for (int li = 0; li < nl; li++) {
        int wps = warps_per_sm_list[li];
        int threads = 256, blocks = 148 * wps * 32 / threads;
        k<OP><<<blocks, threads>>>(out, 12345, cyc);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        k<OP><<<blocks, threads>>>(out, 12345, cyc);
        cudaEventRecord(e1); cudaDeviceSynchronize();
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        double winst = (double)ITERS * CHAINS * ops_per_iter * (wps);  // warp-instr per SM
        printf("%-28s warps/SM %2d: %.3f warp-instr/clk/SM  (%.2f lanes/clk/SM)  block0 cycles %lld, %.3f ms\n", name, wps,
               winst / h, 32.0 * winst / h, h, ms);
    }
    cudaFree(out); cudaFree(cyc);
}

template <class F, int MODE>
void runmul(const char *name, int blocks_per_sm) {
    F *in, *out; long long *cyc, h;
    int blocks = 148 * blocks_per_sm, threads = 256, iters = 512;
    cudaMalloc(&in, sizeof(F) * 256); cudaMalloc(&out, sizeof(F) * blocks * threads); cudaMalloc(&cyc, 8);
    cudaMemset(in, 0x11, sizeof(F) * 256);
    kmul<F, MODE><<<blocks, threads>>>(out, in, iters, cyc);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    kmul<F, MODE><<<blocks, threads>>>(out, in, iters, cyc);
    cudaEventRecord(e1); cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    double ops = 2.0 * iters * blocks * threads;
    printf("%-28s blocks/SM %d: %.2f G op/s  (%.1f cycles per op per warp-slot: block0 %lld cyc / %d ops, x%d warps)\n", name, blocks_per_sm,
           ops / ms / 1e6, (double)h / (2.0 * iters), h, 2 * iters, blocks_per_sm * 8);
}

int main() {
    int l[] = {4, 8, 16, 32};
    run<0>("IMAD (mad.lo.u32)", 1, l, 4);
    run<1>("IMAD.HI (mad.hi.u32)", 1, l, 4);
    run<2>("IMAD.WIDE (mad.wide.u32)", 1, l, 4);
    run<7>("IMAD (mul.lo.u32)", 1, l, 4);
    run<8>("mul24.lo", 1, l, 4);
    run<3>("IADD3 (add.u32)", 1, l, 4);
    run<9>("FFMA", 1, l, 4);
    run<4>("DFMA", 1, l, 4);
    run<5>("mad.lo.cc+madc.hi pair", 2, l, 4);
    run<6>("IMAD + IADD3 1:1", 2, l, 4);
    for (int b = 1; b <= 4; b *= 2) { runmul<Fp, 0>("Fp mul (even/odd)", b); }
    for (int b = 1; b <= 8; b *= 2) { runmul<Fr, 0>("Fr mul (even/odd)", b); }
    runmul<Fp, 1>("Fp add/sub", 4);
    for (int b = 1; b <= 4; b *= 2) { runmul<FpU, 0>("FpU mul (13x30 carry-free)", b); }
    runmul<FpU, 1>("FpU add/sub", 4);
    return 0;
}
