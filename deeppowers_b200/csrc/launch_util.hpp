// launch_util.hpp — helpers shared by the kernel launchers of kernels.cu, keys.cu and eval.cu.  Every name has internal linkage:
// these units are compiled once per arithmetic variant (and kernels.cu in parts) and all link into one library.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <type_traits>

#include "launch.hpp"

namespace dpfhe {
namespace {

// f(std::integral_constant<int, LOGN>{}) for the context's ring degree N = 2^LOGN, 4096 .. 16384; `other` for any other N
template <class F>
cudaError_t with_log_n(u32 log_n, cudaError_t other, F &&f) {
    switch (log_n) {
        case 12: return f(std::integral_constant<int, 12>{});
        case 13: return f(std::integral_constant<int, 13>{});
        case 14: return f(std::integral_constant<int, 14>{});
    }
    return other;
}

// "already configured on this device" bits of one kernel (a function-local static of its launcher).  Several host threads may drive
// different devices at once (dpfhe_multi_*): the attribute call is idempotent, the bit set atomic.
struct ConfiguredMask {
    std::atomic<unsigned long long> bits{0};
    bool has(int device) const { return (bits.load(std::memory_order_acquire) >> (device & 63)) & 1ull; }
    void set(int device) { bits.fetch_or(1ull << (device & 63), std::memory_order_release); }
};

// dynamic shared-memory limit of one kernel, or of two kernels that share a mask, set once per device
template <class K1, class K2 = std::nullptr_t>
cudaError_t set_smem_once(ConfiguredMask &configured, int device, size_t smem, K1 k1, K2 k2 = nullptr) {
    if (configured.has(device)) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if constexpr (!std::is_same_v<K2, std::nullptr_t>) {
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    if (e == cudaSuccess) configured.set(device);
    return e;
}

// grid of the element-wise kernels: one thread per work item, at most 8 resident CTAs of 256 threads per SM, 4 waves
inline unsigned ew_grid(const LaunchCtx &lc, size_t work_items) {
    size_t blocks = (work_items + 255) / 256;
    const size_t cap = (size_t)lc.num_sms * 32;
    if (blocks > cap) blocks = cap;
    return (unsigned)(blocks ? blocks : 1);
}

}  // namespace
}  // namespace dpfhe
