// eval.cuh — the scalar linear combination of ciphertexts (DESIGN.md §2.15, §4.11).
//
// __host__ __device__ like every kernel body, so that the host emulator (tests/emu/emu_lincomb.cpp) runs the product's code.
#pragma once
#include "modarith.cuh"

namespace dpfhe {

constexpr int LINCOMB_MAX_TERMS = 64;

// One launch of ct_lincomb_kernel, passed by value in the kernel parameter block (up to 64 pointers and [64][16] coefficient
// pairs: 17 KiB at MAXT = 64, 2.3 KiB at MAXT = 8).  The parameter block rather than a __constant__ buffer: two contexts on one
// device, or one context on two streams, may launch concurrently, and a symbol shared by all of them would need its own ordering.
// Every index into it is uniform across a CTA (a CTA's chunks lie within one limb row, since N/2 >= 2048 is a multiple of 256).
template <int MAXT>
struct LincombArgs {
    const U64x2 *in[MAXT];   // [batch][2][L][N] ciphertexts; any of them may be `out`
    U64x2 *out;              // [batch][2][L][N]
    const U64x2 *pt;         // nullptr, or [L][N] added to every c0 row (shared by the batch)
    u64 w[MAXT][16];         // c_i mod q_l
    u64 ws[MAXT][16];        // its Shoup companion floor(w 2^64 / q_l)
    u64 cst[16];             // a0 mod q_l, added to every position of every c0 row
    u32 n_terms, L, log_half;   // log_half = log2(N / 2): a row holds 2^log_half chunks of two coefficients
    u32 pad_;
    size_t n_chunks;         // batch * 2 * L * N / 2
};

// c mod q with floor semantics (the result is in [0, q) for negative c too, INT64_MIN included)
inline u64 floor_mod(int64_t c, u64 q) { return c >= 0 ? (u64)c % q : q - 1 - (u64)(-(c + 1)) % q; }

// the coefficient pairs and the constant of one launch over the limbs `lps` (host side; the pointers stay unset)
template <int MAXT>
void build_lincomb_coeffs(const LimbParams *lps, u32 L, const int64_t *coeffs, u32 n_terms, int64_t constant, LincombArgs<MAXT> &A) {
    for (u32 l = 0; l < L; ++l) {
        const u64 q = lps[l].q;
        for (u32 i = 0; i < n_terms; ++i) {
            const u64 w = floor_mod(coeffs[i], q);
            A.w[i][l] = w;
            A.ws[i][l] = (u64)(((unsigned __int128)w << 64) / q);
        }
        A.cst[l] = floor_mod(constant, q);
    }
    A.n_terms = n_terms;
    A.L = L;
}

namespace DPFHE_VNS {

// chunk c (two coefficients) of out = sum_i w_i in_i (+ cst + pt on the c0 rows), canonical.  Each term adds < SB q = 4q
// (shoup_lazy, any 64-bit input); the accumulator starts below 2q and is word-reduced (< 3q) after every third term, so it
// stays below 3q + 3 * 4q = 15q < 16q <= 2^64 and canon() applies at the end.
template <int MAXT>
DPFHE_HD U64x2 lincomb_chunk(const LincombArgs<MAXT> &A, size_t c, const LimbParams &p) {
    const size_t row = c >> A.log_half;
    const u32 l = (u32)(row % A.L);
    u64 x = 0, y = 0;
    if ((row / A.L) % 2 == 0) {   // c0
        x = y = A.cst[l];
        if (A.pt) {
            const U64x2 v = A.pt[((size_t)l << A.log_half) + (c & (((size_t)1 << A.log_half) - 1))];
            x += v.x;
            y += v.y;
        }
    }
    u32 i = 0;
    for (; i + 3 <= A.n_terms; i += 3) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const U64x2 v = A.in[i + j][c];
            x += shoup_lazy(v.x, A.w[i + j][l], A.ws[i + j][l], p);
            y += shoup_lazy(v.y, A.w[i + j][l], A.ws[i + j][l], p);
        }
        x = word_reduce(x, p);
        y = word_reduce(y, p);
    }
    for (; i < A.n_terms; ++i) {
        const U64x2 v = A.in[i][c];
        x += shoup_lazy(v.x, A.w[i][l], A.ws[i][l], p);
        y += shoup_lazy(v.y, A.w[i][l], A.ws[i][l], p);
    }
    return U64x2{canon(x, p), canon(y, p)};
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
