// L2 read-bandwidth probe: every SM streams an L2-resident buffer with 16-byte ld.global.nc loads, the access form the fused key switch
// uses for its source and key words (ntt.cu).  Reports TB/s per buffer size (the largest one, 2 GiB, is an HBM reference) with the card's
// name, SM clock and power limit.  Read-only and bounded: a fixed number of passes per size.
//     make -C tools l2_bench && tools/l2_bench
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>
#include <nvml.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ uint4 ldg_nc(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
// each pass reads the whole buffer once; CTA b starts its share at a rotated offset so the SMs do not walk the same lines in lock step
__global__ void __launch_bounds__(512) k_l2_read(const uint4 *buf, size_t n16, int passes, unsigned *out) {
    const size_t nthr = (size_t)gridDim.x * blockDim.x, gt = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned acc = 0;
    for (int r = 0; r < passes; r++) {
        const size_t rot = ((size_t)(blockIdx.x + r) * 4096) % n16;
        size_t i = gt;
        for (; i + 3 * nthr < n16; i += 4 * nthr) {
            size_t j0 = i + rot, j1 = j0 + nthr, j2 = j1 + nthr, j3 = j2 + nthr;
            const uint4 a = ldg_nc(buf + (j0 >= n16 ? j0 - n16 : j0)), b = ldg_nc(buf + (j1 >= n16 ? j1 - n16 : j1));
            const uint4 c = ldg_nc(buf + (j2 >= n16 ? j2 - n16 : j2)), d = ldg_nc(buf + (j3 >= n16 ? j3 - n16 : j3));
            acc ^= a.x ^ a.w ^ b.x ^ b.w ^ c.x ^ c.w ^ d.x ^ d.w;
        }
        for (; i < n16; i += nthr) {
            size_t j = i + rot;
            const uint4 a = ldg_nc(buf + (j >= n16 ? j - n16 : j));
            acc ^= a.x ^ a.w;
        }
    }
    out[gt] = acc;
}

int main() {
    int dev = 0;
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, dev));
    int clk_khz = 0;
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, dev));
    unsigned plimit_mw = 0;
    if (nvmlInit() == NVML_SUCCESS) {
        nvmlDevice_t h;
        char bus[32];
        CK(cudaDeviceGetPCIBusId(bus, sizeof bus, dev));
        if (nvmlDeviceGetHandleByPciBusId(bus, &h) == NVML_SUCCESS) nvmlDeviceGetEnforcedPowerLimit(h, &plimit_mw);
        nvmlShutdown();
    }
    printf("{\"gpu\": \"%s\", \"sms\": %d, \"l2_mib\": %.1f, \"max_sm_clock_mhz\": %d, \"power_limit_w\": %.0f}\n", p.name, p.multiProcessorCount,
           p.l2CacheSize / 1048576.0, clk_khz / 1000, plimit_mw / 1000.0);
    const size_t sizes_mib[] = {8, 16, 24, 32, 2048};
    const int blocks = p.multiProcessorCount * 4, threads = 512;
    uint4 *buf;
    unsigned *out;
    CK(cudaMalloc(&buf, sizes_mib[4] << 20));
    CK(cudaMemset(buf, 0x5a, sizes_mib[4] << 20));
    CK(cudaMalloc(&out, (size_t)blocks * threads * 4));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (size_t mib : sizes_mib) {
        const size_t bytes = mib << 20, n16 = bytes / 16;
        const int passes = mib >= 1024 ? 4 : (int)(16384 / mib); // ~16 GiB read per timed launch from L2, 8 GiB from HBM
        k_l2_read<<<blocks, threads>>>(buf, n16, 2, out);          // warm: the buffer is now L2-resident (when it fits)
        CK(cudaGetLastError());
        std::vector<float> ms;
        for (int rep = 0; rep < 7; rep++) {
            CK(cudaEventRecord(e0));
            k_l2_read<<<blocks, threads>>>(buf, n16, passes, out);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float t;
            CK(cudaEventElapsedTime(&t, e0, e1));
            ms.push_back(t);
        }
        std::sort(ms.begin(), ms.end());
        const double tb = (double)bytes * passes;
        printf("{\"buffer_mib\": %zu, \"passes\": %d, \"median_tb_s\": %.3f, \"best_tb_s\": %.3f}\n", mib, passes, tb / (ms[3] * 1e-3) / 1e12,
               tb / (ms[0] * 1e-3) / 1e12);
    }
    CK(cudaFree(buf));
    CK(cudaFree(out));
    return 0;
}
