// Issue-rate micro-benchmark for the pipes the modular butterflies use: IMAD.WIDE, IMAD (lo), IADD3, DFMA, DADD, LOP3.
// Reports warp-instructions per clock per SM.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipe_bench pipe_bench.cu
#include <cstdio>
#include <cuda_runtime.h>
typedef unsigned long long u64;
#define ITERS 4096
#define UNROLL 8
template <int KIND> __global__ void k(u64 *out, u64 seed) {
    u64 a[UNROLL];
    double d[UNROLL];
    for (int i = 0; i < UNROLL; i++) { a[i] = seed + threadIdx.x * 977 + i * 13; d[i] = (double)(a[i] & 0xfffff) + 1.5; }
    unsigned b = (unsigned)seed | 1;
    double e = 1.0000001, f = 0.25;
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < UNROLL; i++) {
            if (KIND == 0) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(a[i]) : "r"((unsigned)a[i]), "r"(b));
            if (KIND == 1) { unsigned x = (unsigned)a[i]; asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(b), "r"(b)); a[i] = x; }
            if (KIND == 2) { unsigned x = (unsigned)a[i]; asm volatile("add.u32 %0, %0, %1;" : "+r"(x) : "r"(b)); a[i] = x; }
            if (KIND == 3) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(f));
            if (KIND == 4) asm volatile("add.rn.f64 %0, %0, %1;" : "+d"(d[i]) : "d"(f));
            if (KIND == 5) { unsigned x = (unsigned)a[i]; asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(b), "r"(b + 7)); a[i] = x; }
            if (KIND == 6) asm volatile("mul.hi.u64 %0, %0, %1;" : "+l"(a[i]) : "l"(seed | 0x8000000000000001ULL));
            if (KIND == 7) { // mixed: one DFMA + one IMAD.WIDE (independent chains) -- do the pipes overlap?
                asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(f));
                asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(a[i]) : "r"((unsigned)a[i]), "r"(b));
            }
            if (KIND == 9) asm volatile("cvt.rni.f64.f64 %0, %0;" : "+d"(d[i]));                       // FRND.F64: which pipe, what rate?
            if (KIND == 10) { // DFMA + FRND.F64 on independent chains: do they overlap?
                asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(f));
                double g = (double)a[i]; asm volatile("cvt.rni.f64.f64 %0, %0;" : "+d"(g)); a[i] = (u64)__double_as_longlong(g);
            }
            if (KIND == 11) { // the butterfly's ratio: 7 DFMA-pipe ops per rounding
                double g = d[i];
                asm volatile("cvt.rni.f64.f64 %0, %0;" : "+d"(g));
#pragma unroll
                for (int r = 0; r < 7; r++) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(g));
            }
            if (KIND == 12) { long long x; asm volatile("cvt.rni.s64.f64 %0, %1;" : "=l"(x) : "d"(d[i])); asm volatile("cvt.rn.f64.s64 %0, %1;" : "=d"(d[i]) : "l"(x + 1)); }
            if (KIND == 13) { // same 7:1 ratio with the magic-constant rounding (2 DP ops): the current butterfly
                double g;
                asm volatile("fma.rn.f64 %0, %1, %2, %3;" : "=d"(g) : "d"(d[i]), "d"(f), "d"(6755399441055744.0));
                asm volatile("add.rn.f64 %0, %0, %1;" : "+d"(g) : "d"(-6755399441055744.0));
#pragma unroll
                for (int r = 0; r < 6; r++) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(g));
            }
            if (KIND == 8) { // DFMA + IADD3
                asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(d[i]) : "d"(e), "d"(f));
                unsigned x = (unsigned)a[i]; asm volatile("add.u32 %0, %0, %1;" : "+r"(x) : "r"(b)); a[i] = x;
            }
        }
    }
    u64 s = 0;
    for (int i = 0; i < UNROLL; i++) s += a[i] + (u64)d[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int KIND> void run(const char *name, int per_iter) {
    int dev = 0; cudaDeviceProp p; cudaGetDeviceProperties(&p, dev);
    int blocks = p.multiProcessorCount * 2, threads = 512;
    u64 *out; cudaMalloc(&out, (size_t)blocks * threads * 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<KIND><<<blocks, threads>>>(out, 12345);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    for (int r = 0; r < 5; r++) k<KIND><<<blocks, threads>>>(out, 12345 + r);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    int clk_khz; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, dev);
    double warp_instr = 5.0 * blocks * (threads / 32) * (double)ITERS * UNROLL * per_iter;
    double per_s = warp_instr / (ms * 1e-3);
    printf("%-28s %8.3f ms  %7.2f G warp-instr/s  = %5.2f warp-instr/clk/SM at max clock %d MHz (thread-ops/s %.2f T)\n", name, ms, per_s / 1e9,
           per_s / p.multiProcessorCount / (clk_khz * 1e3), clk_khz / 1000, per_s * 32 / 1e12);
    cudaFree(out);
}
int main() {
    run<0>("IMAD.WIDE.U32", 1); run<1>("IMAD (lo32)", 1); run<2>("IADD3", 1); run<3>("DFMA", 1); run<4>("DADD", 1); run<5>("LOP3", 1);
    run<6>("mul.hi.u64", 1); run<7>("DFMA + IMAD.WIDE (2 instr)", 2); run<8>("DFMA + IADD3 (2 instr)", 2);
    run<9>("FRND.F64 (cvt.rni.f64.f64)", 1); run<10>("DFMA + FRND.F64 (2 instr)", 2); run<11>("7 DFMA + 1 FRND (8 instr)", 8);
    run<12>("F2I.S64.F64 + I2F.F64.S64", 2); run<13>("8 DP ops (magic rounding)", 8);
    return 0;
}
