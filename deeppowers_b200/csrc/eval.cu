// eval.cu — sm_90a kernel and launcher of the scalar linear combination of ciphertexts (DESIGN.md §2.15, §4.11).
//
// Compiled once per arithmetic variant (-DDPFHE_FAST=0 / 1, namespace dpfhe::gen / dpfhe::fast), like kernels.cu and keys.cu.  A
// separate compilation unit: no kernel of kernels.cu or keys.cu shares a body with it.
#include <cuda_runtime.h>

#include "eval.cuh"
#include "launch.hpp"

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
    size_t blocks = (A.n_chunks + 255) / 256;
    const size_t cap = (size_t)lc.num_sms * 32;   // as the element-wise kernels of kernels.cu
    if (blocks > cap) blocks = cap;
    ct_lincomb_kernel<MAXT><<<(unsigned)blocks, 256, 0, st>>>(A, lc.lp);
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

}  // namespace DPFHE_VNS
}  // namespace dpfhe
