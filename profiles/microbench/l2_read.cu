// l2_read.cu — read bandwidth of the L2 cache on sm_90a (H100) at the fused ct x ct kernel's shape.
// Each thread streams 16-byte loads (ld.global.cg: cached in L2 only, so that every load is an L2 access) over a buffer that fits
// the L2, `IN` loads in flight per thread (issued together, consumed before the next group), 2 CTAs x 256 threads per SM as
// ks_fused_kernel<13,256,2,...> runs.  The buffer sizes are multiples of the relinearisation key of the bench shape
// (N = 8192, L = 4: 2 MiB of key words, 2 MiB of companions).  Bytes/s from CUDA events, best and median of REPS launches; the
// card's name, SM count and power limit are printed in the same run.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 l2_read.cu -o l2_read
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));  \
            exit(1);                                                                            \
        }                                                                                       \
    } while (0)

constexpr int NT = 256, CTAS_PER_SM = 2, REPS = 7;

__device__ __forceinline__ uint4 ld_cg16(const uint4 *p) {
    uint4 v;
    asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// n16: 16-byte words of the buffer; passes: how often it is read
template <int IN>
__global__ void __launch_bounds__(NT, CTAS_PER_SM) l2_read(const uint4 *buf, size_t n16, int passes, unsigned *sink) {
    const size_t T = (size_t)gridDim.x * NT, g = (size_t)blockIdx.x * NT + threadIdx.x;
    unsigned acc = 0;
    for (int ps = 0; ps < passes; ++ps) {
        // every pass starts one CTA further, so that a CTA reads other words in consecutive passes
        const size_t rot = ((size_t)ps * NT) % n16;
#pragma unroll 1
        for (size_t i = g; i < n16; i += IN * T) {
            uint4 v[IN];
#pragma unroll
            for (int k = 0; k < IN; ++k) {
                size_t j = i + k * T + rot;
                j = j >= n16 ? j - n16 : j;
                v[k] = ld_cg16(buf + j);
            }
#pragma unroll
            for (int k = 0; k < IN; ++k) acc ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
        }
    }
    if (acc == 0x9e3779b9u) sink[0] = acc;   // keeps the loads; practically never taken
}

template <int IN>
void run(const uint4 *buf, size_t bytes, int grid, unsigned *sink) {
    const size_t n16 = bytes / 16;
    const int passes = (int)std::max<size_t>(1, ((size_t)4 << 30) / bytes);   // ~4 GiB read per launch
    l2_read<IN><<<grid, NT>>>(buf, n16, 2, sink);                               // the buffer into the L2, clocks up
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    std::vector<double> tbs;
    for (int r = 0; r < REPS; ++r) {
        CK(cudaEventRecord(e0));
        l2_read<IN><<<grid, NT>>>(buf, n16, passes, sink);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        tbs.push_back((double)bytes * passes / (ms * 1e-3) / 1e12);
    }
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    std::sort(tbs.begin(), tbs.end());
    printf("{\"buffer_mib\": %zu, \"loads_in_flight\": %d, \"ctas\": %d, \"tb_per_s_best\": %.3f, \"tb_per_s_median\": %.3f}\n",
           bytes >> 20, IN, grid, tbs.back(), tbs[REPS / 2]);
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    char power[128] = "unknown";
    if (FILE *f = popen("nvidia-smi -i 0 --query-gpu=power.limit,clocks.max.sm --format=csv,noheader", "r")) {
        if (fgets(power, sizeof power, f)) power[strcspn(power, "\n")] = 0;
        pclose(f);
    }
    printf("{\"device\": \"%s\", \"sms\": %d, \"l2_mib\": %d, \"power_limit_and_max_sm_clock\": \"%s\"}\n", prop.name, prop.multiProcessorCount,
           prop.l2CacheSize >> 20, power);
    const int grid = prop.multiProcessorCount * CTAS_PER_SM;
    const size_t max_bytes = (size_t)16 << 20;
    uint4 *buf;
    unsigned *sink;
    CK(cudaMalloc(&buf, max_bytes));
    CK(cudaMalloc(&sink, sizeof(unsigned)));
    CK(cudaMemset(buf, 0x5a, max_bytes));
    for (size_t mib : {4, 16}) {
        const size_t bytes = mib << 20;
        run<1>(buf, bytes, grid, sink);
        run<2>(buf, bytes, grid, sink);
        run<4>(buf, bytes, grid, sink);
    }
    CK(cudaFree(buf));
    CK(cudaFree(sink));
    return 0;
}
