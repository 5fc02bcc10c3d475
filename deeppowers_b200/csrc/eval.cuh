// eval.cuh — the scalar linear combination of ciphertexts (DESIGN.md §2.15, §4.11) and the CKKS combination fused into the final
// rescale (§2.16, §4.12).
//
// __host__ __device__ like every kernel body, so that the host emulators (tests/emu/emu_lincomb.cpp, emu_ckks_comb.cpp) run the
// product's code.
#pragma once
#include <cmath>

#include "kernel_bodies.cuh"
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

// ---- CKKS polynomial evaluation: the combination fused into the final rescale (DESIGN.md §2.16, §4.12) ----------------------

constexpr int CKKS_COMB_MAX_TERMS = 64;

// One launch pair of ckks_comb_tau_kernel / ckks_comb_limb_kernel, passed by value in the kernel parameter block (17.7 KiB at
// MAXT = 64, 3.0 KiB at MAXT = 8; eval.cu asserts the 32 KiB limit with the other parameters).  Term k is a ciphertext at its
// own level Lk[k] >= Lc, of which only the rows below Lc are read: the prefix is the ciphertext at level Lc (§2.16), so no cut
// copy is made.  The combination is sum_k w_k in_k + cst on the c0 rows, over q_0 .. q_{Lc-1}, and the result is divided by
// q_{Lc-1} (K: the constants of mod_switch_down with t = 0 at level Lc).
template <int MAXT>
struct CkksCombArgs {
    const U64x2 *in[MAXT];   // term k: [batch][2][Lk[k]][N]
    u32 Lk[MAXT];
    u64 w[MAXT][16];         // c_k mod q_l, l < Lc
    u64 ws[MAXT][16];        // its Shoup companion floor(w 2^64 / q_l)
    u64 cst[16];             // c_0 mod q_l
    u32 n_terms, Lc, log_half;   // log_half = log2(N / 2)
    u32 pad_;
    MsConsts K;
};

// 2^e mod q (host)
inline u64 host_pow2_mod(int e, u64 q) {
    u64 r = 1 % q, b = 2 % q;
    for (; e > 0; e >>= 1) {
        if (e & 1) r = (u64)((unsigned __int128)r * b % q);
        b = (u64)((unsigned __int128)b * b % q);
    }
    return r;
}

// an integer-valued double reduced exactly mod q: x = +-M 2^e with M < 2^53 an integer, x mod q = +-(M mod q)(2^e mod q)
// (as the encoder of §2.12; any finite magnitude, 2^90 and beyond included).  -0.0 gives 0.
inline u64 double_mod(double x, u64 q) {
    int e = 0;
    const double f = std::frexp(std::fabs(x), &e);   // |x| = f 2^e, f in [1/2, 1)
    if (f == 0.0) return 0;
    u64 m = (u64)std::ldexp(f, 53);
    e -= 53;
    if (e < 0) {   // an integer below 2^53: the shifted-out bits are zero
        m >>= -e;
        e = 0;
    }
    const u64 r = (u64)((unsigned __int128)(m % q) * host_pow2_mod(e, q) % q);
    return x < 0 && r ? q - r : r;
}

// c = rint((a * m) / s), round half to even (the default rounding mode), each operation rounded on its own (DESIGN.md §2.16)
inline double ckks_comb_coeff(double a, double m, double s) { return std::nearbyint((a * m) / s); }

// the coefficient pairs and the constant of one launch over q_0 .. q_{Lc-1} (host side; the pointers, Lk and K stay unset)
template <int MAXT>
void build_ckks_comb_coeffs(const LimbParams *lps, u32 Lc, const double *coeffs, u32 n_terms, double constant, CkksCombArgs<MAXT> &A) {
    for (u32 l = 0; l < Lc; ++l) {
        const u64 q = lps[l].q;
        for (u32 i = 0; i < n_terms; ++i) {
            const u64 w = double_mod(coeffs[i], q);
            A.w[i][l] = w;
            A.ws[i][l] = (u64)(((unsigned __int128)w << 64) / q);
        }
        A.cst[l] = double_mod(constant, q);
    }
    A.n_terms = n_terms;
    A.Lc = Lc;
}

namespace DPFHE_VNS {

// chunk j (two coefficients) of row l of polynomial `poly` (= 2 * ciphertext + component) of the combination, canonical: the
// arithmetic of lincomb_chunk (every term < 4q, word-reduced after every third, canon() at the end)
template <int MAXT>
DPFHE_HD U64x2 ckks_comb_chunk(const CkksCombArgs<MAXT> &A, size_t poly, u32 l, u32 j, const LimbParams &p) {
    const size_t off = ((size_t)l << A.log_half) + j;
    u64 x = 0, y = 0;
    if (poly % 2 == 0) x = y = A.cst[l];
    u32 i = 0;
    for (; i + 3 <= A.n_terms; i += 3) {
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const U64x2 v = ld_stream(A.in[i + t] + ((poly * A.Lk[i + t]) << A.log_half) + off);
            x += shoup_lazy(v.x, A.w[i + t][l], A.ws[i + t][l], p);
            y += shoup_lazy(v.y, A.w[i + t][l], A.ws[i + t][l], p);
        }
        x = word_reduce(x, p);
        y = word_reduce(y, p);
    }
    for (; i < A.n_terms; ++i) {
        const U64x2 v = ld_stream(A.in[i] + ((poly * A.Lk[i]) << A.log_half) + off);
        x += shoup_lazy(v.x, A.w[i][l], A.ws[i][l], p);
        y += shoup_lazy(v.y, A.w[i][l], A.ws[i][l], p);
    }
    return U64x2{canon(x, p), canon(y, p)};
}

// step 1, one polynomial: tau' = INTT_{Lc-1}(row Lc-1 of the combination), canonical, to `tau` (ms_tau_body with t = 0, its row
// computed in the load stage instead of read).  The whole limb in shared memory: LOGN <= 13, or N = 16384 with 512 threads.
template <int LOGN, int NT, int MAXT, class CTA>
DPFHE_HD void ckks_comb_tau_body(CTA &cta, u64 *buf, const CkksCombArgs<MAXT> &A, size_t poly, const Twiddle *itw, const LimbParams &p, u64 *tau) {
    static_assert(LOGN <= 13 || NT >= 512, "the limb is transformed in one piece");
    constexpr int NC = 1 << (LOGN - 1);
    const u32 l = A.Lc - 1;
    cta.par([&](int tid) {
        for (int c = tid; c < NC; c += NT) reinterpret_cast<U64x2 *>(buf)[swz_chunk(c)] = ckks_comb_chunk(A, poly, l, (u32)c, p);
    });
    inv_passes<LOGN, NT>(cta, buf, itw, p);
    U64x2 *dst = reinterpret_cast<U64x2 *>(tau);
    cta.par([&](int tid) { inv_store_stage<LOGN, NT>(buf, itw, p, tid, [&](int c, const U64x2 &v) { st_cg(dst + c, v); }); });
}

// step 2, one (polynomial, kept limb i < Lc - 1): out = (comb_i - NTT_i(centred(tau') mod q_i)) * q_{Lc-1}^-1 mod q_i, the lift and
// forward passes of ms_limb_body with the combination's chunk of limb i in place of the loaded c[i]
template <int LOGN, int NT, int MAXT, class CTA>
DPFHE_HD void ckks_comb_limb_body(CTA &cta, u64 *buf, const CkksCombArgs<MAXT> &A, size_t poly, u32 i, const u64 *tau, u64 *out_limb,
                                  const Twiddle *tw, const LimbParams &p) {
    static_assert(LOGN <= 13 || NT >= 512, "the limb is transformed in one piece");
    constexpr int NC = 1 << (LOGN - 1);
    const MsConsts &K = A.K;
    const U64x2 *src = reinterpret_cast<const U64x2 *>(tau);
    const u64 half = K.half, neg_ql = p.q - K.qlm[i];   // adding (q_i - q_last mod q_i) subtracts q_last
    auto lift = [&](int c) {
        const U64x2 v = ld_cg(src + c);
        U64x2 r;                                 // centred lift, lazy: < 3q (+ < q when tau' is "negative")
        r.x = word_reduce(v.x, p) + (v.x > half ? neg_ql : 0);
        r.y = word_reduce(v.y, p) + (v.y > half ? neg_ql : 0);
        return r;
    };
    cta.par([&](int tid) { fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, lift); });
    fwd_passes<LOGN, NT, 4>(cta, buf, tw, p);
    const u64 inv = K.inv[i], inv_s = K.inv_s[i], sinv = K.sinv[i], sinv_s = K.sinv_s[i];
    U64x2 *dst = reinterpret_cast<U64x2 *>(out_limb);
    cta.par([&](int tid) {
        for (int c = tid; c < NC; c += NT) {
            const U64x2 u = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c)], cv = ckks_comb_chunk(A, poly, i, (u32)c, p);
            U64x2 r;   // c*inv - u*(s*inv), as ms_limb_core
            r.x = canon4(shoup_exact(cv.x, inv, inv_s, p) + p.q2 - shoup_exact(u.x, sinv, sinv_s, p), p);
            r.y = canon4(shoup_exact(cv.y, inv, inv_s, p) + p.q2 - shoup_exact(u.y, sinv, sinv_s, p), p);
            st_stream(dst + c, r);
        }
    });
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
