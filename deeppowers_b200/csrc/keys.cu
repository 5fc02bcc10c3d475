// keys.cu — sm_90a kernels and launchers of key generation, encryption and decryption (DESIGN.md §2.14, §4.10).
//
// Compiled once per arithmetic variant (-DDPFHE_FAST=0 / 1, namespace dpfhe::gen / dpfhe::fast), like kernels.cu.  A separate
// compilation unit: no kernel of kernels.cu shares a body with these.
#include <cuda_runtime.h>

#include <type_traits>

#include "keys.cuh"
#include "launch_util.hpp"

namespace dpfhe {
namespace DPFHE_VNS {

template <int NT>
struct KeyCta {
    template <class F>
    __device__ __forceinline__ void par(F f) {
        f((int)threadIdx.x);
        __syncthreads();
    }
    template <class F>
    __device__ __forceinline__ void par_dom(F f) {
        f((int)threadIdx.x);
        if (NT <= 256) __syncthreads();
        else asm volatile("bar.sync %0, 256;" ::"r"(1 + ((int)threadIdx.x >> 8)) : "memory");
    }
    template <class F>
    __device__ __forceinline__ void par_warp(F f) {
        f((int)threadIdx.x);
        __syncwarp();
    }
};

// one CTA per (item, limb): the limb's transform in shared memory, followed by the item's small row (N int8)
template <int LOGN, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) keys_ntt_kernel(const __grid_constant__ KeyArgs A, const Twiddle *__restrict__ tw,
                                                            const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    signed char *small = reinterpret_cast<signed char *>(smem_raw + N * 8);
    KeyCta<NT> cta;
    const size_t w = blockIdx.x;
    const u32 l = (u32)(w % L);
    if constexpr (MODE == KM_ENC_PUBLIC) pub_enc_body<LOGN, NT>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L, 0);
    else keys_limb_body<LOGN, NT, MODE>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L);
}

// N = 16384: two CTAs per (item, limb), each keeping half of the outer radix-4 step
template <int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) keys_ntt_pair_kernel(const __grid_constant__ KeyArgs A, const Twiddle *__restrict__ tw,
                                                                 const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << NTT_PAIR_LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    signed char *small = reinterpret_cast<signed char *>(smem_raw + N * 4);   // after half a limb
    KeyCta<NT> cta;
    const size_t w = blockIdx.x / 2;
    const int h = (int)(blockIdx.x & 1);
    const u32 l = (u32)(w % L);
    if constexpr (MODE == KM_ENC_PUBLIC) pub_enc_body<NTT_PAIR_LOGN, NT>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L, h);
    else keys_half_body<NT, MODE>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L, h);
}

// the seeded modes (DESIGN.md §2.23) of keys_ntt_kernel and keys_ntt_pair_kernel: kernels of their own, whose parameter block carries
// the public seed after the KeyArgs, so that the unseeded instances keep theirs
template <int LOGN, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) keys_seeded_ntt_kernel(const __grid_constant__ SeededKeyArgs A, const Twiddle *__restrict__ tw,
                                                                   const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    signed char *small = reinterpret_cast<signed char *>(smem_raw + N * 8);
    KeyCta<NT> cta;
    const size_t w = blockIdx.x;
    const u32 l = (u32)(w % L);
    keys_limb_body<LOGN, NT, MODE>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L);
}

template <int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) keys_seeded_ntt_pair_kernel(const __grid_constant__ SeededKeyArgs A, const Twiddle *__restrict__ tw,
                                                                        const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << NTT_PAIR_LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    signed char *small = reinterpret_cast<signed char *>(smem_raw + N * 4);
    KeyCta<NT> cta;
    const size_t w = blockIdx.x / 2;
    const int h = (int)(blockIdx.x & 1);
    const u32 l = (u32)(w % L);
    keys_half_body<NT, MODE>(cta, buf, small, A, tw + (size_t)l * N, lt.lp[l], l, L, w / L, h);
}

// pt [n][L][N] = c0 + c1 s (+ c2 s^2), ct [n][n_comp][L][N], s [L][N]
template <int LOGN>
__global__ void __launch_bounds__(256) decrypt_kernel(const U64x2 *__restrict__ ct, const U64x2 *__restrict__ s, U64x2 *__restrict__ pt,
                                                      const LimbParams *__restrict__ lps, u32 L, u32 n_comp, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    const size_t pc = NC * L;
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const size_t k = c / pc, in_poly = c % pc;
        st_stream(pt + c, decrypt_chunk(ct + k * n_comp * pc + in_poly, s + in_poly, pc, n_comp, lps[in_poly / NC]));
    }
}

// seeded rows [n][L][N] (src; nullptr: already in place in dst) -> [n][2][L][N] (dst): one ChaCha20 block per thread
template <int LOGN, bool KEYS>
__global__ void __launch_bounds__(256) expand_seeded_kernel(const __grid_constant__ SeededKeyArgs A, const U64x2 *__restrict__ src, U64x2 *__restrict__ dst,
                                                            const __grid_constant__ LimbTable lt, u32 L, size_t n_blocks) {
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_blocks; w += (size_t)gridDim.x * blockDim.x)
        expand_block<LOGN, KEYS>(src, dst, A, lt.lp[(w >> (LOGN - 2)) % L], L, w);
}

namespace {

template <int LOGN, int MODE>
cudaError_t launch_keys_mode(const LaunchCtx &lc, const KeyArgs &A_, size_t n_items, cudaStream_t st) {
    constexpr size_t N = (size_t)1 << LOGN;
    constexpr bool SEEDED = key_mode_seeded(MODE);
    using Args = std::conditional_t<SEEDED, SeededKeyArgs, KeyArgs>;
    const Args &A = static_cast<const Args &>(A_);   // a seeded mode is launched with SeededKeyArgs
    const size_t n_limbs = n_items * lc.L;
    static ConfiguredMask conf;
    auto launch = [&](auto k, size_t grid, size_t smem) {
        cudaError_t e = set_smem_once(conf, lc.device, smem, k);
        if (e != cudaSuccess) return e;
        k<<<(unsigned)grid, 256, smem, st>>>(A, lc.tw, lc.lt, lc.L);
        return cudaGetLastError();
    };
    // half a limb + the small row per CTA of a pair at N = 16384, else the limb + the small row.  At 3 CTAs per SM (80 registers)
    // the generic variant's store stage spills: 2 per SM
    if constexpr (LOGN == NTT_PAIR_LOGN) {
        if constexpr (SEEDED) return launch(keys_seeded_ntt_pair_kernel<256, 2, MODE>, 2 * n_limbs, N * 4 + N);
        else return launch(keys_ntt_pair_kernel<256, 2, MODE>, 2 * n_limbs, N * 4 + N);
    } else {
        if constexpr (SEEDED) return launch(keys_seeded_ntt_kernel<LOGN, 256, 2, MODE>, n_limbs, N * 8 + N);
        else return launch(keys_ntt_kernel<LOGN, 256, 2, MODE>, n_limbs, N * 8 + N);
    }
}

template <int LOGN>
cudaError_t launch_keys_n(const LaunchCtx &lc, int mode, const KeyArgs &A, size_t n_items, cudaStream_t st) {
    switch (mode) {
        case KM_SECRET: return launch_keys_mode<LOGN, KM_SECRET>(lc, A, n_items, st);
        case KM_ENC: return launch_keys_mode<LOGN, KM_ENC>(lc, A, n_items, st);
        case KM_RELIN: return launch_keys_mode<LOGN, KM_RELIN>(lc, A, n_items, st);
        case KM_GALOIS: return launch_keys_mode<LOGN, KM_GALOIS>(lc, A, n_items, st);
        case KM_PUBLIC_KEY: return launch_keys_mode<LOGN, KM_PUBLIC_KEY>(lc, A, n_items, st);
        case KM_ENC_PUBLIC: return launch_keys_mode<LOGN, KM_ENC_PUBLIC>(lc, A, n_items, st);
        case KM_ENC_SEEDED: return launch_keys_mode<LOGN, KM_ENC_SEEDED>(lc, A, n_items, st);
        case KM_RELIN_SEEDED: return launch_keys_mode<LOGN, KM_RELIN_SEEDED>(lc, A, n_items, st);
        case KM_GALOIS_SEEDED: return launch_keys_mode<LOGN, KM_GALOIS_SEEDED>(lc, A, n_items, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace

// n_items: 1 (secret, public key), ciphertexts (encryption, public-key encryption), n_elts * ndig (switch keys); one launch.  A seeded
// mode's A is a SeededKeyArgs.
cudaError_t launch_keys(const LaunchCtx &lc, int mode, const KeyArgs &A, size_t n_items, cudaStream_t st) {
    if (n_items == 0) return cudaSuccess;
    if (n_items * lc.L * 2 > 0x7fffffffull) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) { return launch_keys_n<decltype(lg)::value>(lc, mode, A, n_items, st); });
}

// n_rows seeded rows of lc.L limbs (ciphertexts, or n_keys * ndig key digits when keys) expanded into [n_rows][2][L][N]; one launch
cudaError_t launch_expand_seeded(const LaunchCtx &lc, bool keys, const SeededKeyArgs &A, const u64 *src, u64 *dst, size_t n_rows, cudaStream_t st) {
    const size_t n_blocks = n_rows * lc.L << (lc.log_n - 2);
    if (!n_blocks) return cudaSuccess;
    auto S = reinterpret_cast<const U64x2 *>(src);
    auto D = reinterpret_cast<U64x2 *>(dst);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        auto k = keys ? expand_seeded_kernel<LOGN, true> : expand_seeded_kernel<LOGN, false>;
        k<<<ew_grid(lc, n_blocks), 256, 0, st>>>(A, S, D, lc.lt, lc.L, n_blocks);
        return cudaGetLastError();
    });
}

cudaError_t launch_decrypt(const LaunchCtx &lc, const u64 *ct, const u64 *s, u64 *pt, u32 n_comp, size_t n, cudaStream_t st) {
    const size_t n_chunks = n * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!n_chunks) return cudaSuccess;
    auto C = reinterpret_cast<const U64x2 *>(ct), S = reinterpret_cast<const U64x2 *>(s);
    auto O = reinterpret_cast<U64x2 *>(pt);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        decrypt_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(C, S, O, lc.lp, lc.L, n_comp, n_chunks);
        return cudaGetLastError();
    });
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
