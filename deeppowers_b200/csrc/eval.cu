// eval.cu — sm_90a kernel and launcher of the scalar linear combination of ciphertexts (DESIGN.md §2.15, §4.11).
//
// Compiled once per arithmetic variant (-DDPFHE_FAST=0 / 1, namespace dpfhe::gen / dpfhe::fast), like kernels.cu and keys.cu.  A
// separate compilation unit: no kernel of kernels.cu or keys.cu shares a body with it.
#include <cuda_runtime.h>

#include "eval.cuh"
#include "launch_util.hpp"

namespace dpfhe {
namespace DPFHE_VNS {

// grid-stride over 128-bit chunks: every input row is read once and every output row written once.  No __restrict__: `out` may
// be any of the inputs (each chunk is read in full before it is written, by the same thread).
template <int MAXT>
__global__ void __launch_bounds__(256) ct_lincomb_kernel(const __grid_constant__ LincombArgs<MAXT> A, const LimbParams *__restrict__ lps) {
    const size_t half = (size_t)1 << A.log_half;
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < A.n_chunks; c += (size_t)gridDim.x * blockDim.x)
        A.out[c] = lincomb_chunk(A, c, lps[(c / half) % A.L]);
}

namespace {

template <int MAXT>
cudaError_t launch_lincomb_t(const LaunchCtx &lc, const u64 *const *in, const int64_t *coeffs, u32 n_terms, int64_t constant, const u64 *pt,
                             u64 *out, size_t batch, cudaStream_t st) {
    LincombArgs<MAXT> A;
    build_lincomb_coeffs(lc.lt.lp, lc.L, coeffs, n_terms, constant, A);
    for (u32 i = 0; i < n_terms; ++i) A.in[i] = reinterpret_cast<const U64x2 *>(in[i]);
    A.out = reinterpret_cast<U64x2 *>(out);
    A.pt = reinterpret_cast<const U64x2 *>(pt);
    A.log_half = lc.log_n - 1;
    A.n_chunks = batch * 2 * lc.L * ((size_t)1 << (lc.log_n - 1));
    ct_lincomb_kernel<MAXT><<<ew_grid(lc, A.n_chunks), 256, 0, st>>>(A, lc.lp);
    return cudaGetLastError();
}

}  // namespace

// out [batch][2][L][N] = sum_i coeffs[i] in[i] + constant (+ pt) on the c0 rows; 1 <= n_terms <= 64; one launch.  Up to 8 terms
// the launch carries the smaller parameter block.
cudaError_t launch_lincomb(const LaunchCtx &lc, const u64 *const *in, const int64_t *coeffs, u32 n_terms, int64_t constant, const u64 *pt,
                           u64 *out, size_t batch, cudaStream_t st) {
    if (batch == 0) return cudaSuccess;
    if (n_terms < 1 || n_terms > (u32)LINCOMB_MAX_TERMS || lc.L > 16) return cudaErrorInvalidValue;
    if (n_terms <= 8) return launch_lincomb_t<8>(lc, in, coeffs, n_terms, constant, pt, out, batch, st);
    return launch_lincomb_t<LINCOMB_MAX_TERMS>(lc, in, coeffs, n_terms, constant, pt, out, batch, st);
}

// ---- CKKS combination fused into the final rescale (DESIGN.md §2.16, §4.12)

// kernel parameters stay below the 32 KiB limit (32764 bytes) at 64 terms
static_assert(sizeof(CkksCombArgs<CKKS_COMB_MAX_TERMS>) + sizeof(LimbTable) + 2 * sizeof(void *) + sizeof(size_t) <= 32764,
              "ckks_comb kernel parameters exceed 32 KiB");

// the CTA policy of the transform passes (ntt_core.cuh), as kernels.cu's
template <int NT>
struct CombCta {
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

// one CTA per polynomial: tau' of row Lc-1 of the combination
template <int LOGN, int NT, int MINB, int MAXT>
__global__ void __launch_bounds__(NT, MINB) ckks_comb_tau_kernel(const __grid_constant__ CkksCombArgs<MAXT> A, const __grid_constant__ LimbTable lt,
                                                                  const Twiddle *__restrict__ itw, u64 *tau, size_t n_polys) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    CombCta<NT> cta;
    const u32 l = A.Lc - 1;
    for (size_t w = blockIdx.x; w < n_polys; w += gridDim.x) ckks_comb_tau_body<LOGN, NT>(cta, buf, A, w, itw + (size_t)l * N, lt.lp[l], tau + w * N);
}

// one CTA per (polynomial, kept limb): out [n_polys][Lc-1][N]
template <int LOGN, int NT, int MINB, int MAXT>
__global__ void __launch_bounds__(NT, MINB) ckks_comb_limb_kernel(const __grid_constant__ CkksCombArgs<MAXT> A, const __grid_constant__ LimbTable lt,
                                                                   const Twiddle *__restrict__ tw, const u64 *tau, u64 *out, size_t n_items) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    CombCta<NT> cta;
    const u32 Lo = A.Lc - 1;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const size_t poly = w / Lo;
        const u32 i = (u32)(w % Lo);
        ckks_comb_limb_body<LOGN, NT>(cta, buf, A, poly, i, tau + poly * N, out + (poly * Lo + i) * N, tw + (size_t)i * N, lt.lp[i]);
    }
}

namespace {

template <int LOGN, int NT, int MINB, int MAXT>
cudaError_t launch_ckks_comb_t(const LaunchCtx &lc, const u64 *const *in, const u32 *levels, const double *coeffs, u32 n_terms, double constant,
                               const MsConsts &K, u64 *tau, u64 *out, size_t batch, cudaStream_t st) {
    auto k1 = ckks_comb_tau_kernel<LOGN, NT, MINB, MAXT>;
    auto k2 = ckks_comb_limb_kernel<LOGN, NT, MINB, MAXT>;
    const size_t smem = (size_t)8 << LOGN;
    static ConfiguredMask configured;
    cudaError_t e = set_smem_once(configured, lc.device, smem, k1, k2);
    if (e != cudaSuccess) return e;
    CkksCombArgs<MAXT> A;
    build_ckks_comb_coeffs(lc.lt.lp, lc.L, coeffs, n_terms, constant, A);
    for (u32 i = 0; i < n_terms; ++i) {
        A.in[i] = reinterpret_cast<const U64x2 *>(in[i]);
        A.Lk[i] = levels[i];
    }
    A.log_half = LOGN - 1;
    A.K = K;
    const size_t n_polys = 2 * batch, n_items = n_polys * (lc.L - 1);
    k1<<<(unsigned)(n_polys < 0x7fffffffull ? n_polys : 0x7fffffffull), NT, smem, st>>>(A, lc.lt, lc.itw, tau, n_polys);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k2<<<(unsigned)(n_items < 0x7fffffffull ? n_items : 0x7fffffffull), NT, smem, st>>>(A, lc.lt, lc.tw, tau, out, n_items);
    return cudaGetLastError();
}

template <int LOGN, int NT, int MINB>
cudaError_t launch_ckks_comb_n(const LaunchCtx &lc, const u64 *const *in, const u32 *levels, const double *coeffs, u32 n_terms, double constant,
                               const MsConsts &K, u64 *tau, u64 *out, size_t batch, cudaStream_t st) {
    if (n_terms <= 8) return launch_ckks_comb_t<LOGN, NT, MINB, 8>(lc, in, levels, coeffs, n_terms, constant, K, tau, out, batch, st);
    return launch_ckks_comb_t<LOGN, NT, MINB, CKKS_COMB_MAX_TERMS>(lc, in, levels, coeffs, n_terms, constant, K, tau, out, batch, st);
}

}  // namespace

// out [batch][2][Lc-1][N] = mod_switch_down_{t=0}(sum_i coeffs[i] in[i]|_Lc + constant on c0), Lc = lc.L >= 2; in[i] is
// [batch][2][levels[i]][N] with levels[i] >= Lc; coeffs and constant are integer-valued doubles; tau: 2 batch N words of scratch.
// Two launches, as mod_switch_down; 1 <= n_terms <= 64.  The geometry (threads, CTAs per SM) is that of launch_mod_switch.
cudaError_t launch_ckks_comb(const LaunchCtx &lc, const u64 *const *in, const u32 *levels, const double *coeffs, u32 n_terms, double constant,
                             const MsConsts &K, u64 *tau, u64 *out, size_t batch, cudaStream_t st) {
    if (batch == 0) return cudaSuccess;
    if (n_terms < 1 || n_terms > (u32)CKKS_COMB_MAX_TERMS || lc.L < 2 || lc.L > 16) return cudaErrorInvalidValue;
    for (u32 i = 0; i < n_terms; ++i)
        if (levels[i] < lc.L) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value, NT = LOGN == 14 ? 512 : 256, MINB = LOGN == 12 ? 2 : LOGN == 13 ? 3 : 1;
        return launch_ckks_comb_n<LOGN, NT, MINB>(lc, in, levels, coeffs, n_terms, constant, K, tau, out, batch, st);
    });
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
