// kernel_bodies.cuh — CTA-level bodies of every kernel (DESIGN.md §4).
//
// Each body is written against a tiny CTA policy:
//     cta.par(f)   run f(tid) for all NT threads, then barrier
// On the GPU (kernels.cu) par() is "f(threadIdx.x); __syncthreads();".  tests/emu provides
// a sequential policy so the identical bodies run on the CPU for index-algebra checks
// (test infrastructure only — the product has no CPU path).
#pragma once
#include "ntt_core.cuh"

namespace dpfhe {
namespace DPFHE_VNS {

DPFHE_HD u32 bitrev_n(u32 x, int bits) {
#if defined(__CUDA_ARCH__)
    return __brev(x) >> (32 - bits);
#else
    u32 r = 0;
    for (int i = 0; i < bits; ++i) {
        r = (r << 1) | (x & 1);
        x >>= 1;
    }
    return r;
#endif
}

// Evaluation-form index map of the automorphism X -> X^g (DESIGN.md §2.8):
// out[i] = in[pi(i)],  2*br(pi(i)) + 1 = g * (2*br(i) + 1)  mod 2N.
template <int LOGN>
DPFHE_HD int galois_index(int i, u32 g) {
    const u32 mask2n = (2u << LOGN) - 1;
    u32 e = (g * (2u * bitrev_n((u32)i, LOGN) + 1u)) & mask2n;
    return (int)bitrev_n((e - 1u) >> 1, LOGN);
}

// ---- memory access policy -------------------------------------------------------------
// ld_stream / st_stream: data touched once (ciphertext in/out)   -> read-only path, no L1 allocation
// ld_cg / st_cg        : cross-CTA scratch written in this launch -> L2-coherent (.cg)
// ld_keep              : tables / keys shared by the whole batch  -> default caching
DPFHE_HD U64x2 ld_stream(const U64x2 *p) {
#if defined(__CUDA_ARCH__)
    U64x2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
    return v;
#else
    return *p;
#endif
}
DPFHE_HD void st_stream(U64x2 *p, const U64x2 &v) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
#else
    *p = v;
#endif
}
#if defined(__CUDA_ARCH__) && defined(DPFHE_L2_KEEP)
// tuning variant: cross-CTA scratch marked evict-last in L2
__device__ __forceinline__ u64 l2_keep_policy() {
    u64 pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
#endif
DPFHE_HD U64x2 ld_cg(const U64x2 *p) {
#if defined(__CUDA_ARCH__) && defined(DPFHE_L2_KEEP)
    U64x2 v;
    asm volatile("ld.global.cg.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(l2_keep_policy()) : "memory");
    return v;
#elif defined(__CUDA_ARCH__)
    U64x2 v;
    asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
    return v;
#else
    return *p;
#endif
}
DPFHE_HD void st_cg(U64x2 *p, const U64x2 &v) {
#if defined(__CUDA_ARCH__) && defined(DPFHE_L2_KEEP)
    asm volatile("st.global.cg.L2::cache_hint.v2.u64 [%0], {%1,%2}, %3;" ::"l"(p), "l"(v.x), "l"(v.y), "l"(l2_keep_policy()) : "memory");
#elif defined(__CUDA_ARCH__)
    asm volatile("st.global.cg.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
#else
    *p = v;
#endif
}
DPFHE_HD U64x2 ld_keep(const U64x2 *p) {
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const U64x2 *>(__builtin_assume_aligned(p, 16));
#else
    return *p;
#endif
}

// ---- standalone transforms (one limb per call) ----------------------------------------
// data: [N] coefficients of limb `p`, in place.  buf: N words of shared memory.
// SRC(chunk) -> U64x2: the canonical input chunk (a limb in memory, or values reduced into the limb as they are loaded)
template <int LOGN, int NT, class CTA, class SRC>
DPFHE_HD void ntt_fwd_src_body(CTA &cta, u64 *buf, SRC src, u64 *data, const Twiddle *tw, const LimbParams &p) {
    cta.par([&](int tid) { fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, src); });
    fwd_passes<LOGN, NT, 1>(cta, buf, tw, p);
    U64x2 *dst = reinterpret_cast<U64x2 *>(data);
    cta.par([&](int tid) {
        for (int c = tid; c < (1 << (LOGN - 1)); c += NT) {
            U64x2 v = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c)];
            v.x = canon_store(v.x, p);
            v.y = canon_store(v.y, p);
            st_stream(dst + c, v);
        }
    });
}
template <int LOGN, int NT, class CTA>
DPFHE_HD void ntt_fwd_body(CTA &cta, u64 *buf, u64 *data, const Twiddle *tw, const LimbParams &p) {
    const U64x2 *src = reinterpret_cast<const U64x2 *>(data);
    ntt_fwd_src_body<LOGN, NT>(cta, buf, [&](int c) { return ld_stream(src + c); }, data, tw, p);
}

// the limb already sits in shared memory in the swizzled layout (copied by the threads below, or by the TMA unit:
// ntt_inv_tma_kernel): register passes, then the outermost stage straight to global memory
template <int LOGN, int NT, class CTA>
DPFHE_HD void ntt_inv_resident(CTA &cta, u64 *buf, u64 *data, const Twiddle *itw, const LimbParams &p) {
    inv_passes<LOGN, NT>(cta, buf, itw, p);
    U64x2 *dst = reinterpret_cast<U64x2 *>(data);
    cta.par([&](int tid) {
        inv_store_stage<LOGN, NT>(buf, itw, p, tid, [&](int c, const U64x2 &v) { st_stream(dst + c, v); });
    });
}

template <int LOGN, int NT, class CTA>
DPFHE_HD void ntt_inv_body(CTA &cta, u64 *buf, u64 *data, const Twiddle *itw, const LimbParams &p) {
    const U64x2 *src = reinterpret_cast<const U64x2 *>(data);
    cta.par([&](int tid) {
        for (int c = tid; c < (1 << (LOGN - 1)); c += NT)
            reinterpret_cast<U64x2 *>(buf)[swz_chunk(c)] = ld_stream(src + c);
    });
    ntt_inv_resident<LOGN, NT>(cta, buf, data, itw, p);
}

// ---- N = 16384 standalone transforms by a PAIR of CTAs (a thread-block cluster of two) ------------------------------
// A 128 KiB limb in one CTA's shared memory allows one CTA per SM; the transform kernels need about three to hide each
// other's memory phases (DESIGN.md §6).  So the limb is split as in the fused kernel: CTA h of the pair owns the two
// 4096-point blocks {2h, 2h+1} in 64 KiB of shared memory.
//   forward: both CTAs read the whole limb (the outer radix-4 step needs all four blocks) and keep their half of its
//            result; a cluster barrier separates the reads from the in-place stores.
//   inverse: each CTA runs the block-local passes on its half; the outer radix-4 step then reads two blocks from its own
//            shared memory and two from the partner's (distributed shared memory), each CTA finishing half of the columns.
constexpr int NTT_PAIR_LOGN = 14;

template <int NT, class CTA, class SRC>
DPFHE_HD void ntt_fwd_half_load_src(CTA &cta, u64 *buf, SRC src, const Twiddle *tw, const LimbParams &p, int h) {
    cta.par([&](int tid) { fwd_load_stage_half<NTT_PAIR_LOGN, NT, false>(buf, tw, p, tid, src, h); });
}
template <int NT, class CTA>
DPFHE_HD void ntt_fwd_half_load(CTA &cta, u64 *buf, const u64 *data, const Twiddle *tw, const LimbParams &p, int h) {
    const U64x2 *src = reinterpret_cast<const U64x2 *>(data);
    ntt_fwd_half_load_src<NT>(cta, buf, [&](int c) { return ld_stream(src + c); }, tw, p, h);
}
template <int NT, class CTA>
DPFHE_HD void ntt_fwd_half_finish(CTA &cta, u64 *buf, u64 *data, const Twiddle *tw, const LimbParams &p, int h) {
    constexpr int HC = 1 << (NTT_PAIR_LOGN - 2);   // chunks of half a limb
    fwd_passes_blk<NTT_PAIR_LOGN, NT, 1, 2>(cta, buf, tw, p, 2 * h);
    U64x2 *dst = reinterpret_cast<U64x2 *>(data) + h * HC;
    cta.par([&](int tid) {
        for (int lc = tid; lc < HC; lc += NT) {
            U64x2 v = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)];
            v.x = canon_store(v.x, p);
            v.y = canon_store(v.y, p);
            st_stream(dst + lc, v);
        }
    });
}
template <int NT, class CTA>
DPFHE_HD void ntt_inv_half_passes(CTA &cta, u64 *buf, const u64 *data, const Twiddle *itw, const LimbParams &p, int h) {
    constexpr int HC = 1 << (NTT_PAIR_LOGN - 2);
    const U64x2 *src = reinterpret_cast<const U64x2 *>(data) + h * HC;
    cta.par([&](int tid) {
        for (int lc = tid; lc < HC; lc += NT) reinterpret_cast<U64x2 *>(buf)[swz_chunk(lc)] = ld_stream(src + lc);
    });
    inv_passes_blk<NTT_PAIR_LOGN, NT, 2>(cta, buf, itw, p, 2 * h);
}
// peer: the partner CTA's buffer (its shared memory through the cluster mapping; a plain second buffer in the emulator)
template <int NT, class CTA>
DPFHE_HD void ntt_inv_half_outer(CTA &cta, const u64 *buf, const u64 *peer, u64 *data, const Twiddle *itw, const LimbParams &p, int h) {
    constexpr int CPB = 1 << (NTT_PAIR_LOGN - 3);   // chunks per 4096-point block
    U64x2 *dst = reinterpret_cast<U64x2 *>(data);
    cta.par([&](int tid) {
        inv_outer_stage<NTT_PAIR_LOGN, NT>(
            itw, p, tid,
            [&](int c) {   // chunk c of the limb lives in block c / CPB: blocks {2h, 2h+1} here, the other two at the partner
                const int b = c / CPB, lc = (b & 1) * CPB + (c - b * CPB);
                return reinterpret_cast<const U64x2 *>((b >> 1) == h ? buf : peer)[swz_chunk(lc)];
            },
            [&](int c, const U64x2 &v) { st_stream(dst + c, v); }, h * (CPB / 2), (h + 1) * (CPB / 2));
    });
}

// ---- element-wise kernels -------------------------------------------------------------
// chunk-granular (two coefficients); `l` is the limb of the chunk.
DPFHE_HD U64x2 mul_chunk(const U64x2 &a, const U64x2 &b, const LimbParams &p) {
    U64x2 r;
    r.x = mulmod(a.x, b.x, p);
    r.y = mulmod(a.y, b.y, p);
    return r;
}

// 128-bit accumulate of a product
DPFHE_HD void mac128(u64 &hi, u64 &lo, u64 a, u64 b) {
    u64 h, l;
    mul128(a, b, h, l);
#if defined(__CUDA_ARCH__)
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, %3;" : "+l"(lo), "+l"(hi) : "l"(l), "l"(h));
#else
    lo += l;
    hi += h + (lo < l ? 1ull : 0ull);
#endif
}

// Lazy accumulators gain one Shoup product (< SB*q) per step from a start bound b0 (b0 + SB <= 16).  Whenever the next
// addition could pass 16q the value takes one csub(8q) right after the current one ([0,16q) -> [0,8q)).
// Returns whether the addition with 0-based index `step` is followed by that trim; uniform scalar code.
DPFHE_HD bool acc_trim_after(int b0, int step) {
    int b = b0;
    bool t = false;
    for (int s = 0; s <= step; ++s) {
        b += SB;
        t = b + SB > 16;
        if (t) b = 8;
    }
    return t;
}

// tensor of one coefficient: canonical inputs; d0,d2 in [0,SB*q), d1 in [0,(SB+1)q)
DPFHE_HD void tensor_coeff(u64 a0, u64 a1, u64 b0, u64 b1, const LimbParams &p, u64 &d0, u64 &d1, u64 &d2) {
#if DPFHE_TENSOR_KARATSUBA
    // three 128-bit products instead of four (the multiplier is the scarce unit, DESIGN.md §6): a0 b1 + a1 b0 =
    // (a0 + a1)(b0 + b1) - a0 b0 - a1 b1 over the integers; the sums are below 2^61, every term fits 128 bits
    u64 h0, l0, h2, l2, hk, lk;
    mul128(a0, b0, h0, l0);
    mul128(a1, b1, h2, l2);
    mul128(a0 + a1, b0 + b1, hk, lk);
    sub128(hk, lk, h0, l0);
    sub128(hk, lk, h2, l2);
    d0 = barrett_lazy(h0, l0, p);
    d2 = barrett_lazy(h2, l2, p);
    d1 = barrett_lazy(hk, lk, p);
#else
    d0 = mulmod_lazy(a0, b0, p);
    d2 = mulmod_lazy(a1, b1, p);
    u64 hi, lo;
    mul128(a0, b1, hi, lo);
    mac128(hi, lo, a1, b0);
    d1 = barrett_lazy(hi, lo, p);
#endif
}

// ---- fused key-switch family (DESIGN.md §4.4) ------------------------------------------
// One work item = (ciphertext ct, output limb i).  Shared memory holds only the swizzled transform
// buffer buf[N]; the two lazy accumulators live in two scratch rows owned by the CTA's slot (acc_rows:
// L2-resident read-modify-write by the owning thread, values kept below 16q), which keeps the CTA at
// one limb of shared memory so that three CTAs share an SM and hide each other's memory phases.  The
// output rows out[ct][0|1][i] are written exactly once, with the final canonical values — so `out` may
// be memory of another GPU (peer-mapped: the result gather of a multi-GPU job rides on these stores).
//   phase 1: build the digit d = d2[i] (tensor / input / permuted c1), write
//            acc = (own terms) + d o key[i][.][i], INTT(d) -> t_i, publish t_i to the slot.
//   phase 2: for every other digit j: u = NTT_i(t_j mod q_i); acc += u o key[j][.][i];
//            the last digit writes canon(acc) to the output rows.
struct KsArgs {
    const u64 *a;        // MUL_RELIN: a [batch][2][L][N]; PLAIN: d [batch][L][N]; ROTATE: ct [batch][2][L][N]
    const u64 *b;        // MUL_RELIN: b
    const u64 *key;      // [L][2][L][N]
    const u64 *key_s;    // Shoup companions floor(key * 2^64 / q_limb), same layout (built per launch)
    u64 *out;            // [batch][2][L][N]: written once, final values (may be peer memory)
    u64 *acc;            // [slots][acc_par][2][N] lazy accumulators of the resident work items
    u64 *scratch;        // [slots][2 parities][N]
    const Twiddle *tw;   // [L][N] forward tables
    const Twiddle *itw;  // [L][N] inverse tables
    u32 L;               // limbs of a ciphertext polynomial = number of digits
    u32 galois;          // ROTATE only
    u32 Lk;              // limbs of a key polynomial: L, or L + 1 with a special prime (hybrid, DESIGN.md §2.10)
    u64 *hyb;            // hybrid only: [groups][KS_HYB_ROWS][N]: special-limb accumulators (rows 0,1) and tau'
    const u32 *only;     // optional [batch]: process only the ciphertexts whose entry is non-zero (hoisted-rotation fallback)
    u32 acc_par;         // accumulator row pairs per slot: 1, or 2 in hybrid key switching (the division step runs one round late)
    u32 lift_reduce;     // 0: every modulus is below twice every other one, a digit needs no reduction when it changes limb; 1: reduce
};
// tau' rows of a hybrid group are double-buffered by round parity (KS_HYB_ROWS, types.hpp)
DPFHE_HD u32 ks_hyb_tau_row(u32 parity, u32 c) { return 2u + 2u * parity + c; }

// The key row that limb i of a level view over lq ciphertext limbs reads (LV instances, DESIGN.md §4.17): the key is the top-level
// one, restricted by the choice of rows alone.  Limbs below lq read their own row, the special limbs the row `shift` further down
// (shift = Lq - l; the key's stride, A.Lk, is the top-level L).  The Shoup companions have the key's layout and use the same map.
// Without LV the bodies keep their own expressions for the row, so that the instances that existed before compile as they did.
DPFHE_HD size_t ks_key_row(u32 i, u32 lq, u32 shift) { return i >= lq ? (size_t)i + shift : (size_t)i; }

// operands of one 16-byte chunk position of phase 1, fetched one iteration ahead of their use
struct KsP1Operands {
    U64x2 a0, a1, b0, b1;   // MUL_RELIN: the four input chunks; PLAIN: a0 = digit; ROTATE: a0 = c0 gather, a1 = c1 gather
    U64x2 kb, ka, kbs, kas; // key[i][b|a][i] chunk and Shoup companions
};

// base pointers of one work item's phase-1 streams (computed once, outside the chunk loop)
struct KsP1Pointers {
    const U64x2 *a0, *a1, *b0, *b1, *kb, *ka, *kbs, *kas;
    const u64 *c0, *c1;   // ROTATE: scalar gathers
};

template <int LOGN, int MODE>
DPFHE_HD KsP1Operands ks_p1_fetch(const KsP1Pointers &ptr, u32 galois, int c) {
    KsP1Operands o;
    o.kb = ld_keep(ptr.kb + c);
    o.ka = ld_keep(ptr.ka + c);
    o.kbs = ld_keep(ptr.kbs + c);
    o.kas = ld_keep(ptr.kas + c);
    if (MODE == KS_MUL_RELIN) {
        o.a0 = ld_stream(ptr.a0 + c);
        o.a1 = ld_stream(ptr.a1 + c);
        o.b0 = ld_stream(ptr.b0 + c);
        o.b1 = ld_stream(ptr.b1 + c);
    } else if (MODE == KS_PLAIN) {
        o.a0 = ld_stream(ptr.a0 + c);
        o.a1 = o.b0 = o.b1 = o.a0;
    } else {
        const int n0 = galois_index<LOGN>(2 * c, galois), n1 = galois_index<LOGN>(2 * c + 1, galois);
        o.a0.x = ptr.c0[n0];
        o.a0.y = ptr.c0[n1];
        o.a1.x = ptr.c1[n0];
        o.a1.y = ptr.c1[n1];
        o.b0 = o.b1 = o.a0;
    }
    return o;
}

// digit + accumulator start values of one chunk position
// HYB: the own terms are scaled by the special prime (pm = p_special mod q_i), so that the final division by it
// leaves them unchanged: out = ((p*d + sum) - s*u) / p.
template <int MODE, bool HYB = false>
DPFHE_HD void ks_p1_chunk(const KsP1Operands &o, const LimbParams &p, bool only, u64 *buf, U64x2 *acc0, U64x2 *acc1, U64x2 *out0, U64x2 *out1,
                          int c, int c_buf, u64 pm = 0, u64 pm_s = 0) {
    U64x2 d, s0, s1;   // digit (< SB*q), own contributions to acc0 (< SB*q) / acc1 (< (SB+1) q)
    if (MODE == KS_MUL_RELIN) {
        tensor_coeff(o.a0.x, o.a1.x, o.b0.x, o.b1.x, p, s0.x, s1.x, d.x);
        tensor_coeff(o.a0.y, o.a1.y, o.b0.y, o.b1.y, p, s0.y, s1.y, d.y);
    } else if (MODE == KS_PLAIN) {
        d = o.a0;
        s0.x = s0.y = s1.x = s1.y = 0;
    } else {
        d = o.a1;
        s0 = o.a0;
        s1.x = s1.y = 0;
    }
    if (HYB && MODE != KS_PLAIN) {
        s0.x = shoup_lazy(s0.x, pm, pm_s, p);
        s0.y = shoup_lazy(s0.y, pm, pm_s, p);
        if (MODE == KS_MUL_RELIN) {
            s1.x = shoup_lazy(s1.x, pm, pm_s, p);
            s1.y = shoup_lazy(s1.y, pm, pm_s, p);
        }
    }
    // digit enters the inverse transform below SB*q (tensor) or canonical
    reinterpret_cast<U64x2 *>(buf)[swz_chunk(c_buf)] = d;
    U64x2 r0, r1;   // s < (SB+1) q (< SB*q after the hybrid scaling), Shoup term < SB*q  ->  accumulator starts below (2 SB + 1) q
    r0.x = s0.x + shoup_lazy(d.x, o.kb.x, o.kbs.x, p);
    r0.y = s0.y + shoup_lazy(d.y, o.kb.y, o.kbs.y, p);
    r1.x = s1.x + shoup_lazy(d.x, o.ka.x, o.kas.x, p);
    r1.y = s1.y + shoup_lazy(d.y, o.ka.y, o.kas.y, p);
    if (only) {   // a single digit: this is already the result
        r0.x = canon(r0.x, p); r0.y = canon(r0.y, p);
        r1.x = canon(r1.x, p); r1.y = canon(r1.y, p);
        st_stream(out0 + c, r0);
        st_stream(out1 + c, r1);
    } else {
        st_cg(acc0 + c, r0);
        st_cg(acc1 + c, r1);
    }
}

// ---- encrypted inner product (KS_DOT, DESIGN.md §2.18 / §4.15) ------------------------------------------------------------
// The operand tables of one call: pair t is (a[t], b[t]), each [batch][2][Lq][N] canonical.  Passed by value in the kernel
// parameter block, so a pair's pointers are constant-bank operands with a CTA-uniform index.
struct DotArgs {
    const u64 *a[DOT_MAX_TERMS];
    const u64 *b[DOT_MAX_TERMS];
    u32 n_terms;   // 1 .. DOT_MAX_TERMS
};

// Test hook (host builds with DPFHE_DOT_TRACK only): the largest 128-bit running sum in units of 2^(2b) (b = bit length of q; the
// precondition of barrett_lazy_long is "below 16") and the largest reduced value in units of q (its result is below 15).
#if defined(DPFHE_DOT_TRACK) && !defined(__CUDA_ARCH__)
struct DotTrack {
    double sum_over_q2 = 0, red_over_q = 0;
};
inline DotTrack &dot_track() {
    static DotTrack t;
    return t;
}
inline void dot_track_note(u64 hi, u64 lo, u64 r, const LimbParams &p) {
    const double z = (double)hi * 18446744073709551616.0 + (double)lo, pb = (double)(1ull << (p.bar_shift + 2));
    DotTrack &t = dot_track();
    const double s = z / (pb * pb), d = (double)r / (double)p.q;
    if (s > t.sum_over_q2) t.sum_over_q2 = s;
    if (d > t.red_over_q) t.red_over_q = d;
}
#define DPFHE_DOT_NOTE(hi, lo, r, p) dot_track_note(hi, lo, r, p)
#else
#define DPFHE_DOT_NOTE(hi, lo, r, p)
#endif

// A running sum of 128-bit products folded to one word: (hi:lo) < 2^(2b+4)  ->  (0 : r), r < 15q
DPFHE_HD void dot_fold(u64 &hi, u64 &lo, const LimbParams &p) {
    const u64 r = barrett_lazy_long(hi, lo, p);
    DPFHE_DOT_NOTE(hi, lo, r, p);
    lo = r;
    hi = 0;
}

// D_c = sum_t tensor(a_t, b_t)_c of one coefficient position `pos` (word offset into a ciphertext's c0 row; c1 is P words on),
// congruent mod q and below 15q.  The four products of a pair are summed in 128 bits and reduced once per 16 products: a folded
// sum r < 15q plus 16 products of canonical factors is 15q + 16 (q - 1)^2 < 16 q^2 < 2^(2b+4), the precondition of
// barrett_lazy_long, so D_1 (two products per pair) folds every 8 pairs and D_0, D_2 every 16.
DPFHE_HD void dot_coeff_pair(const DotArgs &D, size_t pos, size_t P, const LimbParams &p, U64x2 &d0, U64x2 &d1, U64x2 &d2) {
    u64 h0x = 0, l0x = 0, h1x = 0, l1x = 0, h2x = 0, l2x = 0, h0y = 0, l0y = 0, h1y = 0, l1y = 0, h2y = 0, l2y = 0;
    const u32 n = D.n_terms;
#pragma unroll 1
    for (u32 t = 0; t < n; ++t) {
        if (t != 0 && (t & 7u) == 0) {
            dot_fold(h1x, l1x, p);
            dot_fold(h1y, l1y, p);
            if ((t & 15u) == 0) {
                dot_fold(h0x, l0x, p);
                dot_fold(h0y, l0y, p);
                dot_fold(h2x, l2x, p);
                dot_fold(h2y, l2y, p);
            }
        }
        const U64x2 *pa = reinterpret_cast<const U64x2 *>(D.a[t] + pos), *pb = reinterpret_cast<const U64x2 *>(D.b[t] + pos);
        const U64x2 a0 = ld_stream(pa), a1 = ld_stream(pa + P / 2), b0 = ld_stream(pb), b1 = ld_stream(pb + P / 2);
        mac128(h0x, l0x, a0.x, b0.x);
        mac128(h0y, l0y, a0.y, b0.y);
        mac128(h1x, l1x, a0.x, b1.x);
        mac128(h1y, l1y, a0.y, b1.y);
        mac128(h1x, l1x, a1.x, b0.x);
        mac128(h1y, l1y, a1.y, b0.y);
        mac128(h2x, l2x, a1.x, b1.x);
        mac128(h2y, l2y, a1.y, b1.y);
    }
    dot_fold(h0x, l0x, p);
    dot_fold(h0y, l0y, p);
    dot_fold(h1x, l1x, p);
    dot_fold(h1y, l1y, p);
    dot_fold(h2x, l2x, p);
    dot_fold(h2y, l2y, p);
    d0.x = l0x; d0.y = l0y;
    d1.x = l1x; d1.y = l1y;
    d2.x = l2x; d2.y = l2y;
}

// One chunk position of a limb CTA's phase 1: what ks_p1_chunk<KS_MUL_RELIN, true> does with one pair's tensor, done with the sums.
// D_2 enters the inverse transform below SB*q; P*D_0, P*D_1 (Shoup products accept any word) start the accumulators below SB*q each,
// and the own-digit key terms add another SB*q: below (2 SB + 1) q as phase 2 expects.
DPFHE_HD void ks_p1_dot_chunk(const DotArgs &D, size_t pos, size_t P, const KsP1Pointers &ptr, const LimbParams &p, u64 *buf, U64x2 *acc0,
                              U64x2 *acc1, int c, int c_buf, u64 pm, u64 pm_s) {
    U64x2 s0, s1, d;
    dot_coeff_pair(D, pos, P, p, s0, s1, d);
    d.x = word_reduce(d.x, p);   // < 3q
    d.y = word_reduce(d.y, p);
    if (SB < 3) {
        d.x = csub(d.x, p.q);
        d.y = csub(d.y, p.q);
    }
    reinterpret_cast<U64x2 *>(buf)[swz_chunk(c_buf)] = d;
    const U64x2 kb = ld_keep(ptr.kb + c), ka = ld_keep(ptr.ka + c), kbs = ld_keep(ptr.kbs + c), kas = ld_keep(ptr.kas + c);
    U64x2 r0, r1;
    r0.x = shoup_lazy(s0.x, pm, pm_s, p) + shoup_lazy(d.x, kb.x, kbs.x, p);
    r0.y = shoup_lazy(s0.y, pm, pm_s, p) + shoup_lazy(d.y, kb.y, kbs.y, p);
    r1.x = shoup_lazy(s1.x, pm, pm_s, p) + shoup_lazy(d.x, ka.x, kas.x, p);
    r1.y = shoup_lazy(s1.y, pm, pm_s, p) + shoup_lazy(d.y, ka.y, kas.y, p);
    st_cg(acc0 + c, r0);
    st_cg(acc1 + c, r1);
}

// slot_free / slot_free_target: when non-null, the digit slot is single-buffered and may only be overwritten once the counter has
// reached the target (every reader of the previous digit has signalled); cta.wait_ge spins on it (a no-op in the host emulator,
// whose sequential order already guarantees it).
template <int LOGN, int NT, int MODE, bool HYB = false, bool LV = false, class CTA>
DPFHE_HD void ks_phase1(CTA &cta, u64 *buf, const KsArgs &A, const LimbParams &p, size_t ct, u32 i, u64 *t_slot, u64 *acc_rows, u64 pm = 0,
                        u64 pm_s = 0, const u32 *slot_free = nullptr, u32 slot_free_target = 0, u32 key_digit = ~0u, const DotArgs *dot = nullptr,
                        u32 key_shift = 0) {
    constexpr int N = 1 << LOGN, NC = N / 2;
    static_assert((NC / NT) % 2 == 0, "chunk loops may be unrolled by two (ping-pong operand buffers)");
    static_assert(MODE != KS_DOT || HYB, "the inner product exists with special-prime keys only");
    const size_t P = (size_t)A.L * N, PK = HYB ? (size_t)A.Lk * N : P;
    U64x2 *acc0 = reinterpret_cast<U64x2 *>(acc_rows), *acc1 = reinterpret_cast<U64x2 *>(acc_rows + N);
    U64x2 *out0 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + (size_t)i * N);
    U64x2 *out1 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + P + (size_t)i * N);
    const bool only = !HYB && A.L == 1;   // a single digit: no phase 2, write the canonical result here
    KsP1Pointers ptr;
    {
        const u32 kd = key_digit == ~0u ? i : key_digit;   // the key digit that limb i belongs to (grouped digits: i / K)
        size_t koff_b, koff_a;
        if constexpr (LV) {
            const size_t kr = ks_key_row(i, A.L, key_shift);
            koff_b = ((size_t)kd * 2 + 0) * PK + kr * N;
            koff_a = ((size_t)kd * 2 + 1) * PK + kr * N;
        } else {
            koff_b = ((size_t)kd * 2 + 0) * PK + (size_t)i * N;
            koff_a = ((size_t)kd * 2 + 1) * PK + (size_t)i * N;
        }
        ptr.kb = reinterpret_cast<const U64x2 *>(A.key + koff_b);
        ptr.ka = reinterpret_cast<const U64x2 *>(A.key + koff_a);
        ptr.kbs = reinterpret_cast<const U64x2 *>(A.key_s + koff_b);
        ptr.kas = reinterpret_cast<const U64x2 *>(A.key_s + koff_a);
        const size_t in_off = (MODE == KS_PLAIN ? ct * P : ct * 2 * P) + (size_t)i * N;
        ptr.a0 = reinterpret_cast<const U64x2 *>(A.a + in_off);
        ptr.a1 = reinterpret_cast<const U64x2 *>(A.a + in_off + P);
        ptr.b0 = reinterpret_cast<const U64x2 *>((MODE == KS_MUL_RELIN ? A.b : A.a) + in_off);
        ptr.b1 = reinterpret_cast<const U64x2 *>((MODE == KS_MUL_RELIN ? A.b : A.a) + in_off + P);
        ptr.c0 = A.a + in_off;
        ptr.c1 = A.a + in_off + P;
    }
    const u32 galois = A.galois;
    // chunk range [c_lo, c_lo + n_c) of the limb goes to shared-memory chunks [0, n_c)
    auto build = [&](int c_lo, int n_c) {
        cta.par([&](int tid) {
            if constexpr (MODE == KS_DOT) {
                // the pair loop runs inside a chunk position: three 128-bit sums per coefficient stay in registers (§4.15)
                const size_t pos0 = ct * 2 * P + (size_t)i * N;
#pragma unroll 1
                for (int lc = tid; lc < n_c; lc += NT)
                    ks_p1_dot_chunk(*dot, pos0 + 2 * (size_t)(c_lo + lc), P, ptr, p, buf, acc0, acc1, c_lo + lc, lc, pm, pm_s);
            } else if (MODE == KS_MUL_RELIN) {
                // No software prefetch for the tensor product: three co-resident CTAs hide the load latency, and a
                // second operand set (32 registers) would push the 80-register kernel into spills (+5% instructions).
#pragma unroll 1
                for (int lc = tid; lc < n_c; lc += NT) {
                    const KsP1Operands o = ks_p1_fetch<LOGN, MODE>(ptr, galois, c_lo + lc);
                    ks_p1_chunk<MODE, HYB>(o, p, only, buf, acc0, acc1, out0, out1, c_lo + lc, lc, pm, pm_s);
                }
            } else {
                // rotate / key switch: the gathered operands have long latency and are few: fetch one chunk ahead
                KsP1Operands nxt = ks_p1_fetch<LOGN, MODE>(ptr, galois, c_lo + tid);
#pragma unroll 1
                for (int lc = tid; lc < n_c; lc += NT) {
                    const KsP1Operands o = nxt;
                    if (lc + NT < n_c) nxt = ks_p1_fetch<LOGN, MODE>(ptr, galois, c_lo + lc + NT);
                    ks_p1_chunk<MODE, HYB>(o, p, only, buf, acc0, acc1, out0, out1, c_lo + lc, lc, pm, pm_s);
                }
            }
        });
    };
    const Twiddle *itw = A.itw + (size_t)i * N;
    U64x2 *dst = reinterpret_cast<U64x2 *>(t_slot);
    if constexpr (LOGN <= 13) {
        build(0, NC);
        cta.mark(0);   // tensor / digit build + own key terms
        if (only) return;   // no other digit needs t
        inv_passes<LOGN, NT>(cta, buf, itw, p);
        cta.mark(1);   // inverse register passes
        if (slot_free) cta.wait_ge(slot_free, slot_free_target);
        cta.par([&](int tid) {
            inv_store_stage<LOGN, NT>(buf, itw, p, tid, [&](int c, const U64x2 &v) { st_cg(dst + c, v); });
        });
        cta.mark(2);   // outer inverse stage + digit publish
    } else {
        // N = 16384: the limb is processed as two halves of two 4096-blocks each (64 KiB of shared memory, so three
        // CTAs share an SM); the block-local register passes leave their result in the digit slot, and the two
        // outermost stages then run in place over the slot (each thread reads and rewrites its own four chunks).
        constexpr int HC = NC / 2;
        for (int h = 0; h < 2; ++h) {
            build(h * HC, HC);
            cta.mark(0);
            if (only) continue;
            inv_passes_blk<LOGN, NT, 2>(cta, buf, itw, p, 2 * h);
            cta.mark(1);
            if (slot_free && h == 0) cta.wait_ge(slot_free, slot_free_target);
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) st_cg(dst + h * HC + lc, reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)]);
            });
        }
        if (only) return;
        cta.par([&](int tid) {
            inv_outer_stage<LOGN, NT>(itw, p, tid, [&](int c) { return ld_cg(dst + c); }, [&](int c, const U64x2 &v) { st_cg(dst + c, v); });
        });
        cta.mark(2);
    }
}

// t_src: the published t of digit j (N words, natural order, canonical mod q_j)
// HYB: key polynomials carry A.Lk limbs and nothing is final here (the division by the special prime follows).
// acc_rows: the two accumulator rows of this work item, acc_rows[0..N) and acc_rows[N..2N).
// SPECIAL (hybrid only): limb i = A.L is the special prime; jj = 0 .. L-1 counts its digits and its accumulators start from zero.
// LOAD(h): fills the transform buffer with the first forward stage(s) of the lifted digit (h = half for N = 16384, else 0), from
// values below BIN*q.  n_digits: how many digits the accumulation runs over (the last one finishes a non-hybrid result).
template <int LOGN, int NT, bool HYB, bool SPECIAL, int BIN, bool LV = false, class CTA, class LOAD>
DPFHE_HD void ks_phase2_core(CTA &cta, u64 *buf, const KsArgs &A, const LimbParams &p, size_t ct, u32 i, u32 j, u32 jj, u32 n_digits, LOAD load,
                             u64 *acc_rows, u32 key_shift = 0) {
    constexpr int N = 1 << LOGN, NC = N / 2;
    static_assert(HYB || !SPECIAL, "the special limb exists only in hybrid key switching");
    const size_t P = (size_t)A.L * N, PK = HYB ? (size_t)A.Lk * N : P;
    const Twiddle *tw = A.tw + (size_t)i * N;
    size_t koff_b, koff_a;
    if constexpr (LV) {
        const size_t kr = ks_key_row(i, A.L, key_shift);
        koff_b = ((size_t)j * 2 + 0) * PK + kr * N;
        koff_a = ((size_t)j * 2 + 1) * PK + kr * N;
    } else {
        koff_b = ((size_t)j * 2 + 0) * PK + (size_t)i * N;
        koff_a = ((size_t)j * 2 + 1) * PK + (size_t)i * N;
    }
    const U64x2 *kb = reinterpret_cast<const U64x2 *>(A.key + koff_b), *ka = reinterpret_cast<const U64x2 *>(A.key + koff_a);
    const U64x2 *kbs = reinterpret_cast<const U64x2 *>(A.key_s + koff_b), *kas = reinterpret_cast<const U64x2 *>(A.key_s + koff_a);
    U64x2 *acc0 = reinterpret_cast<U64x2 *>(acc_rows), *acc1 = reinterpret_cast<U64x2 *>(acc_rows + N);
    // the output rows, written once by the last digit (unused in hybrid key switching: the division step writes them)
    U64x2 *out0 = reinterpret_cast<U64x2 *>(HYB ? acc_rows : A.out + ct * 2 * P + (size_t)i * N);
    U64x2 *out1 = reinterpret_cast<U64x2 *>(HYB ? acc_rows + N : A.out + ct * 2 * P + P + (size_t)i * N);
    // lazy accumulator bound: below (2 SB + 1) q after phase 1 (0 for the special limb), + SB*q per digit; trimmed
    // with one csub(8q) whenever the next digit could pass 16q
    constexpr int B0 = 2 * SB + 1;
    // no trim after the final digit: nothing is added any more, and whoever reads the accumulator next (canon below, the division
    // step of the special-prime variants) accepts any value below 16q
    const bool final_digit = jj + 1 == n_digits, last = !HYB && final_digit;
    const bool trim = !final_digit && (SPECIAL ? acc_trim_after(0, (int)jj) : acc_trim_after(B0, (int)jj - 1));
    const bool first = SPECIAL && jj == 0;
    struct MacOperands {
        U64x2 vb, va, vbs, vas, r0, r1;
    };
    auto fetch = [&](int c) {
        MacOperands m;
        m.vb = ld_keep(kb + c);
        m.va = ld_keep(ka + c);
        m.vbs = ld_keep(kbs + c);
        m.vas = ld_keep(kas + c);
        if (first) {
            m.r0.x = m.r0.y = m.r1.x = m.r1.y = 0;
        } else {
            m.r0 = ld_cg(acc0 + c);
            m.r1 = ld_cg(acc1 + c);
        }
        return m;
    };
    // c: chunk of the limb (key / accumulator position); c_buf: where its transform output sits in shared memory
    auto mac = [&](MacOperands &m, int c, int c_buf) {
        // u < 16q straight from the transform: Shoup multiplication accepts any 64-bit operand
        const U64x2 u = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c_buf)];
        m.r0.x += shoup_lazy(u.x, m.vb.x, m.vbs.x, p);
        m.r0.y += shoup_lazy(u.y, m.vb.y, m.vbs.y, p);
        m.r1.x += shoup_lazy(u.x, m.va.x, m.vas.x, p);
        m.r1.y += shoup_lazy(u.y, m.va.y, m.vas.y, p);
        if (trim) {
            m.r0.x = csub(m.r0.x, p.q8); m.r0.y = csub(m.r0.y, p.q8);
            m.r1.x = csub(m.r1.x, p.q8); m.r1.y = csub(m.r1.y, p.q8);
        }
        if (last) {
            m.r0.x = canon(m.r0.x, p); m.r0.y = canon(m.r0.y, p);
            m.r1.x = canon(m.r1.x, p); m.r1.y = canon(m.r1.y, p);
            st_stream(out0 + c, m.r0);
            st_stream(out1 + c, m.r1);
        } else {
            st_cg(acc0 + c, m.r0);
            st_cg(acc1 + c, m.r1);
        }
    };
    // multiply-accumulate of the chunk range [c_lo, c_lo + n_c), whose transform output sits in chunks [0, n_c)
    auto mac_range = [&](int c_lo, int n_c) {
        cta.par([&](int tid) {
            MacOperands nxt = fetch(c_lo + tid);
#pragma unroll 1
            for (int lc = tid; lc < n_c; lc += NT) {
                MacOperands m = nxt;
                if (lc + NT < n_c) nxt = fetch(c_lo + lc + NT);   // next chunk's key / accumulator loads fly during this chunk's math
                mac(m, c_lo + lc, lc);
            }
        });
    };
    if constexpr (LOGN <= 13) {
        load(0);
        cta.mark(4);   // digit fetch + lift + outer forward stage
        fwd_passes<LOGN, NT, BIN>(cta, buf, tw, p);
        cta.mark(5);   // forward register passes
        mac_range(0, NC);
        cta.mark(6);   // multiply-accumulate with the key column (the last digit also canonicalises and stores)
    } else {
        // N = 16384: two halves of two 4096-blocks; each half re-reads the digit and keeps its two output blocks
        constexpr int HC = NC / 2;
        for (int h = 0; h < 2; ++h) {
            load(h);
            cta.mark(4);
            fwd_passes_blk<LOGN, NT, BIN, 2>(cta, buf, tw, p, 2 * h);
            cta.mark(5);
            mac_range(h * HC, HC);
            cta.mark(6);
        }
    }
}

// one digit = one limb (BV-RNS, and hybrid key switching with one special prime): the lift is t_j itself
template <int LOGN, int NT, bool HYB = false, bool SPECIAL = false, bool LV = false, class CTA>
DPFHE_HD void ks_phase2_digit(CTA &cta, u64 *buf, const KsArgs &A, const LimbParams &p, size_t ct, u32 i, u32 j, u32 jj, const u64 *t_src,
                              u64 *acc_rows, u32 key_shift = 0) {
    const Twiddle *tw = A.tw + (size_t)i * ((size_t)1 << LOGN);
    const U64x2 *src = reinterpret_cast<const U64x2 *>(t_src);
    // lift of the digit into Z_{q_i}: t_j < q_j.  When every modulus of the basis is below twice every other one (the default
    // basis: all within 2^-22 of 2^60), t_j < 2 q_i already and the word reduction (three multiplies per coefficient) is skipped.
    const bool lift = A.lift_reduce != 0u;
    auto get = [&](int c) { return ld_cg(src + c); };
    auto load = [&](int h) {
        cta.par([&](int tid) {
            if constexpr (LOGN <= 13) {
                if (lift) fwd_load_stage<LOGN, NT, true>(buf, tw, p, tid, get);
                else fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, get);
            } else {
                if (lift) fwd_load_stage_half<LOGN, NT, true>(buf, tw, p, tid, get, h);
                else fwd_load_stage_half<LOGN, NT, false>(buf, tw, p, tid, get, h);
            }
        });
    };
    ks_phase2_core<LOGN, NT, HYB, SPECIAL, 3, LV>(cta, buf, A, p, ct, i, j, jj, A.L, load, acc_rows, key_shift);
}

// ---- fused key switch at N <= 8192: one 4096-point block per CTA (DESIGN.md §4.4) -----------------------------------------
// Work item = (ciphertext ct, limb i, half h).  At N = 8192 the two halves of a limb are a CTA pair (a thread-block cluster of
// two); at N = 4096 the limb is one block and h = 0.  Shared memory holds the CTA's 4096-point transform buffer buf (32 KiB) and
// its two lazy accumulator half-rows acc[0, HC) and acc[HC, 2 HC) (64 KiB), so the accumulators never leave the SM.  The output
// rows are written once, with the final canonical values, by the last digit, so `out` may still be peer memory.
//   phase 1: ks_blk_phase1_local: digit + own key terms, inverse register passes on the block;
//            (pair barrier) ks_blk_phase1_outer: the outermost inverse stage over the pair -> t_i, half of the columns per CTA.
//   phase 2: ks_blk_phase2 for every other digit j: lift of all of t_j and the first forward stage for the CTA's own block,
//            the three forward passes, multiply-accumulate with the key half-row.
// Every lazy value is the one ks_phase1 / ks_phase2_digit compute for the same coefficient, so the results are bit-identical.
constexpr int KS_BLK_LOGN = 12;                  // the block a CTA owns
constexpr int KS_BLK_HC = 1 << (KS_BLK_LOGN - 1);   // its 16-byte chunks
template <int LOGN>
DPFHE_HD constexpr int ks_blk_pair() {   // CTAs per limb
    return 1 << (LOGN - KS_BLK_LOGN);
}

// Phase-1 operands and start values of one chunk, as ks_phase1 / ks_p1_chunk compute them (non-hybrid).  They are restated here
// rather than factored out of those two: ks_phase1 also serves the hybrid, grouped and N = 16384 kernels, which compile to the
// same SASS as before this body existed only while its code is left as it is.
template <int MODE>
DPFHE_HD KsP1Pointers ks_blk_p1_pointers(const KsArgs &A, size_t ct, u32 i, size_t N) {
    const size_t P = (size_t)A.L * N;
    const size_t koff_b = ((size_t)i * 2 + 0) * P + (size_t)i * N, koff_a = ((size_t)i * 2 + 1) * P + (size_t)i * N;
    const size_t in_off = (MODE == KS_PLAIN ? ct * P : ct * 2 * P) + (size_t)i * N;
    KsP1Pointers ptr;
    ptr.kb = reinterpret_cast<const U64x2 *>(A.key + koff_b);
    ptr.ka = reinterpret_cast<const U64x2 *>(A.key + koff_a);
    ptr.kbs = reinterpret_cast<const U64x2 *>(A.key_s + koff_b);
    ptr.kas = reinterpret_cast<const U64x2 *>(A.key_s + koff_a);
    ptr.a0 = reinterpret_cast<const U64x2 *>(A.a + in_off);
    ptr.a1 = reinterpret_cast<const U64x2 *>(A.a + in_off + P);
    ptr.b0 = reinterpret_cast<const U64x2 *>((MODE == KS_MUL_RELIN ? A.b : A.a) + in_off);
    ptr.b1 = reinterpret_cast<const U64x2 *>((MODE == KS_MUL_RELIN ? A.b : A.a) + in_off + P);
    ptr.c0 = A.a + in_off;
    ptr.c1 = A.a + in_off + P;
    return ptr;
}
// d: the digit (< SB*q); r0, r1: accumulator start values (< (2 SB + 1) q)
template <int MODE>
DPFHE_HD void ks_blk_p1_terms(const KsP1Operands &o, const LimbParams &p, U64x2 &d, U64x2 &r0, U64x2 &r1) {
    U64x2 s0, s1;   // own contributions to acc0 (< SB*q) / acc1 (< (SB+1) q)
    if (MODE == KS_MUL_RELIN) {
        tensor_coeff(o.a0.x, o.a1.x, o.b0.x, o.b1.x, p, s0.x, s1.x, d.x);
        tensor_coeff(o.a0.y, o.a1.y, o.b0.y, o.b1.y, p, s0.y, s1.y, d.y);
    } else if (MODE == KS_PLAIN) {
        d = o.a0;
        s0.x = s0.y = s1.x = s1.y = 0;
    } else {
        d = o.a1;
        s0 = o.a0;
        s1.x = s1.y = 0;
    }
    r0.x = s0.x + shoup_lazy_cc(d.x, o.kb.x, o.kbs.x, p);
    r0.y = s0.y + shoup_lazy_cc(d.y, o.kb.y, o.kbs.y, p);
    r1.x = s1.x + shoup_lazy_cc(d.x, o.ka.x, o.kas.x, p);
    r1.y = s1.y + shoup_lazy_cc(d.y, o.ka.y, o.kas.y, p);
}

template <int LOGN, int NT, int MODE, class CTA>
DPFHE_HD void ks_blk_phase1_local(CTA &cta, u64 *buf, U64x2 *acc, const KsArgs &A, const LimbParams &p, size_t ct, u32 i, int h) {
    static_assert(LOGN == 12 || LOGN == 13, "one or two 4096-point blocks per limb");
    constexpr int N = 1 << LOGN, HC = KS_BLK_HC;
    const size_t P = (size_t)A.L * N;
    const int c0 = h * HC;   // first chunk of the block in the limb
    U64x2 *out0 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + (size_t)i * N) + c0;
    U64x2 *out1 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + P + (size_t)i * N) + c0;
    const bool only = A.L == 1;   // a single digit: no phase 2, write the canonical result here
    const KsP1Pointers ptr = ks_blk_p1_pointers<MODE>(A, ct, i, N);
    const u32 galois = A.galois;
    cta.par([&](int tid) {
        // operands one chunk ahead: the 128-register budget of two CTAs per SM has room for a second operand set
        KsP1Operands nxt = ks_p1_fetch<LOGN, MODE>(ptr, galois, c0 + tid);
#pragma unroll 1
        for (int lc = tid; lc < HC; lc += NT) {
            const KsP1Operands o = nxt;
            if (lc + NT < HC) nxt = ks_p1_fetch<LOGN, MODE>(ptr, galois, c0 + lc + NT);
            U64x2 d, r0, r1;
            ks_blk_p1_terms<MODE>(o, p, d, r0, r1);
            reinterpret_cast<U64x2 *>(buf)[swz_chunk(lc)] = d;
            if (only) {
                r0.x = canon(r0.x, p); r0.y = canon(r0.y, p);
                r1.x = canon(r1.x, p); r1.y = canon(r1.y, p);
                st_stream(out0 + lc, r0);
                st_stream(out1 + lc, r1);
            } else {
                acc[lc] = r0;
                acc[HC + lc] = r1;
            }
        }
    });
    cta.mark(0);   // tensor / digit build + own key terms
    if (only) return;
    inv_passes_blk<LOGN, NT, 1>(cta, buf, A.itw + (size_t)i * N, p, h);
    cta.mark(1);   // inverse register passes
}

// peer: the partner's transform buffer (distributed shared memory at N = 8192; unused at N = 4096; a plain second buffer in the
// emulator).  CTA h finishes chunk columns [h, h + 1) * HC / pair of both blocks and stores them to t_slot (the limb's digit slot).
template <int LOGN, int NT, class CTA>
DPFHE_HD void ks_blk_phase1_outer(CTA &cta, const u64 *buf, const u64 *peer, const KsArgs &A, const LimbParams &p, u32 i, int h, u64 *t_slot) {
    constexpr int HC = KS_BLK_HC, CW = HC / ks_blk_pair<LOGN>();
    U64x2 *dst = reinterpret_cast<U64x2 *>(t_slot);
    cta.par([&](int tid) {
        inv_outer_stage<LOGN, NT>(
            A.itw + ((size_t)i << LOGN), p, tid,
            [&](int c) {
                const int b = c / HC;
                return reinterpret_cast<const U64x2 *>(b == h ? buf : peer)[swz_chunk(c - b * HC)];
            },
            [&](int c, const U64x2 &v) { st_cg(dst + c, v); }, h * CW, (h + 1) * CW);
    });
    cta.mark(2);   // outer inverse stage + digit publish
}

// t_src: the published t of digit j (N words, natural order, canonical mod q_j)
template <int LOGN, int NT, class CTA>
DPFHE_HD void ks_blk_phase2(CTA &cta, u64 *buf, U64x2 *acc, const KsArgs &A, const LimbParams &p, size_t ct, u32 i, u32 j, u32 jj, int h,
                            const u64 *t_src) {
    constexpr int N = 1 << LOGN, HC = KS_BLK_HC, BIN = 3;
    const size_t P = (size_t)A.L * N;
    const int c0 = h * HC;
    const Twiddle *tw = A.tw + (size_t)i * N;
    const U64x2 *src = reinterpret_cast<const U64x2 *>(t_src);
    // lift of the digit into Z_{q_i}, as ks_phase2_digit
    const bool lift = A.lift_reduce != 0u;
    auto get = [&](int c) { return ld_cg(src + c); };
    cta.par([&](int tid) {
        if (lift) fwd_load_stage_blk<LOGN, NT, true>(buf, tw, p, tid, get, h);
        else fwd_load_stage_blk<LOGN, NT, false>(buf, tw, p, tid, get, h);
    });
    cta.mark(4);   // digit fetch + lift + outer forward stage
    fwd_passes_blk<LOGN, NT, BIN, 1>(cta, buf, tw, p, h);
    cta.mark(5);   // forward register passes
    const size_t koff_b = ((size_t)j * 2 + 0) * P + (size_t)i * N, koff_a = ((size_t)j * 2 + 1) * P + (size_t)i * N;
    const U64x2 *kb = reinterpret_cast<const U64x2 *>(A.key + koff_b) + c0, *ka = reinterpret_cast<const U64x2 *>(A.key + koff_a) + c0;
    const U64x2 *kbs = reinterpret_cast<const U64x2 *>(A.key_s + koff_b) + c0, *kas = reinterpret_cast<const U64x2 *>(A.key_s + koff_a) + c0;
    U64x2 *out0 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + (size_t)i * N) + c0;
    U64x2 *out1 = reinterpret_cast<U64x2 *>(A.out + ct * 2 * P + P + (size_t)i * N) + c0;
    // lazy accumulator bound and trims as ks_phase2_core: below (2 SB + 1) q after phase 1, + SB*q per digit
    constexpr int B0 = 2 * SB + 1;
    const bool last = jj + 1 == A.L;
    const bool trim = !last && acc_trim_after(B0, (int)jj - 1);
    // chunk lc with the key words b, a and their Shoup companions bs, as
    auto mac = [&](int lc, const U64x2 &b, const U64x2 &a, const U64x2 &bs, const U64x2 &as) {
        // u < 16q straight from the transform: Shoup multiplication accepts any 64-bit operand
        const U64x2 u = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)];
        U64x2 r0 = acc[lc], r1 = acc[HC + lc];
        r0.x += shoup_lazy(u.x, b.x, bs.x, p);
        r0.y += shoup_lazy(u.y, b.y, bs.y, p);
        r1.x += shoup_lazy(u.x, a.x, as.x, p);
        r1.y += shoup_lazy(u.y, a.y, as.y, p);
        if (trim) {
            r0.x = csub(r0.x, p.q8); r0.y = csub(r0.y, p.q8);
            r1.x = csub(r1.x, p.q8); r1.y = csub(r1.y, p.q8);
        }
        if (last) {
            r0.x = canon(r0.x, p); r0.y = canon(r0.y, p);
            r1.x = canon(r1.x, p); r1.y = canon(r1.y, p);
            st_stream(out0 + lc, r0);
            st_stream(out1 + lc, r1);
        } else {
            acc[lc] = r0;
            acc[HC + lc] = r1;
        }
    };
    cta.par([&](int tid) {
        if constexpr (DPFHE_FAST) {
            // Only the companions are read and each key word is rebuilt from its own (shoup_w_from_companion, two IMAD.WIDE):
            // half the key bytes.  Two chunks are in flight, in the registers one chunk of words and companions took: the loop
            // takes the chunks two at a time, and each set is refilled as soon as its chunk's products have read it.
            static_assert(HC % (2 * NT) == 0, "the key-column loop takes two chunks per iteration");
            auto mac_s = [&](int lc, const U64x2 &bs, const U64x2 &as) {
                U64x2 b, a;
                b.x = shoup_w_from_companion(bs.x, p); b.y = shoup_w_from_companion(bs.y, p);
                a.x = shoup_w_from_companion(as.x, p); a.y = shoup_w_from_companion(as.y, p);
                mac(lc, b, a, bs, as);
            };
            U64x2 s0b = ld_keep(kbs + tid), s0a = ld_keep(kas + tid), s1b = ld_keep(kbs + tid + NT), s1a = ld_keep(kas + tid + NT);
#pragma unroll 1
            for (int lc = tid; lc < HC; lc += 2 * NT) {
                mac_s(lc, s0b, s0a);
                if (lc + 2 * NT < HC) {
                    s0b = ld_keep(kbs + lc + 2 * NT);
                    s0a = ld_keep(kas + lc + 2 * NT);
                }
                mac_s(lc + NT, s1b, s1a);
                if (lc + 3 * NT < HC) {
                    s1b = ld_keep(kbs + lc + 3 * NT);
                    s1a = ld_keep(kas + lc + 3 * NT);
                }
            }
        } else {
            // gen: rebuilding a word would take a full 64 x 64 product, so both rows are read
            U64x2 vb = ld_keep(kb + tid), va = ld_keep(ka + tid), vbs = ld_keep(kbs + tid), vas = ld_keep(kas + tid);
#pragma unroll 1
            for (int lc = tid; lc < HC; lc += NT) {
                const U64x2 b = vb, a = va, bs = vbs, as = vas;
                if (lc + NT < HC) {   // the next chunk's key loads fly during this chunk's math
                    vb = ld_keep(kb + lc + NT);
                    va = ld_keep(ka + lc + NT);
                    vbs = ld_keep(kbs + lc + NT);
                    vas = ld_keep(kas + lc + NT);
                }
                mac(lc, b, a, bs, as);
            }
        }
    });
    cta.mark(6);   // multiply-accumulate with the key half-row (the last digit also canonicalises and stores)
}

// a digit of several limbs (grouped hybrid key switching, DESIGN.md §2.11): the lift of group g into limb i is the fast basis
// conversion sum_{j in g} y_j * (Qhat_j mod q_i), y_j = the scaled inverse transforms the members published.
// t_rows + j * t_stride: the published row of limb j.
template <int LOGN, int NT, bool SPECIAL, bool LV = false, class CTA>
DPFHE_HD void ks_phase2_group(CTA &cta, u64 *buf, const KsArgs &A, const GroupConsts &G, const LimbParams &p, size_t ct, u32 i, u32 g, u32 jj,
                              const u64 *t_rows, size_t t_stride, u64 *acc_rows, u32 key_shift = 0) {
    const Twiddle *tw = A.tw + (size_t)i * ((size_t)1 << LOGN);
    const u32 lo = g * G.K, hi = lo + G.K < G.Lq ? lo + G.K : G.Lq;
    auto get = [&](int c) {
        U64x2 r;
        r.x = r.y = 0;
        for (u32 j = lo; j < hi; ++j) {   // each term below SB*q = 4q; at most KS_MAX_SPECIAL = 4 of them: the sum stays below 16q
            const U64x2 v = ld_cg(reinterpret_cast<const U64x2 *>(t_rows + (size_t)j * t_stride) + c);
            r.x += shoup_lazy(v.x, G.up[j][i], G.up_s[j][i], p);
            r.y += shoup_lazy(v.y, G.up[j][i], G.up_s[j][i], p);
        }
        if (hi - lo > 2) {   // < 16q -> < 8q
            r.x = csub(r.x, p.q8);
            r.y = csub(r.y, p.q8);
        }
        r.x = csub(r.x, p.q4);   // < 8q  ->  < 4q
        r.y = csub(r.y, p.q4);
        return r;
    };
    auto load = [&](int h) {
        cta.par([&](int tid) {
            if constexpr (LOGN <= 13) fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, get);
            else fwd_load_stage_half<LOGN, NT, false>(buf, tw, p, tid, get, h);
        });
    };
    ks_phase2_core<LOGN, NT, true, SPECIAL, 4, LV>(cta, buf, A, p, ct, i, g, jj, G.dnum, load, acc_rows, key_shift);
}

// ---- modulus switching: drop the last limb (DESIGN.md §2.9) -------------------------------------

// step 1, one polynomial: tau' = INTT_last(c[L-1]) (times t^-1 mod q_last for BGV), canonical, to `tau`.
// LAZY: the source row is L2-resident scratch written in this launch, with values below 16q (hybrid key switching);
// otherwise canonical streamed input.  With 256 threads and N = 16384 the limb is transformed as two halves through
// the `work` row (N words of scratch, may be the source row itself when that is scratch).
template <int LOGN, int NT, bool LAZY = false, class CTA>
DPFHE_HD void ms_tau_body(CTA &cta, u64 *buf, const u64 *row, u64 *work, const Twiddle *itw, const LimbParams &p, u64 *tau, const MsConsts &K) {
    constexpr int NC = 1 << (LOGN - 1);
    const U64x2 *src = reinterpret_cast<const U64x2 *>(row);
    auto fetch = [&](int c) {
        if (!LAZY) return ld_stream(src + c);
        U64x2 v = ld_cg(src + c);   // < 16q  ->  [0, 2q), what the inverse passes expect
        v.x = csub(word_reduce(v.x, p), p.q2);
        v.y = csub(word_reduce(v.y, p), p.q2);
        return v;
    };
    U64x2 *dst = reinterpret_cast<U64x2 *>(tau);
    const bool has_t = K.has_t != 0;
    auto emit = [&](int c, const U64x2 &v) {
        U64x2 r = v;
        if (has_t) {
            r.x = csub(shoup_exact(v.x, K.tinv, K.tinv_s, p), p.q);
            r.y = csub(shoup_exact(v.y, K.tinv, K.tinv_s, p), p.q);
        }
        st_cg(dst + c, r);
    };
    if constexpr (LOGN <= 13 || NT >= 512) {
        cta.par([&](int tid) {
            for (int c = tid; c < NC; c += NT) reinterpret_cast<U64x2 *>(buf)[swz_chunk(c)] = fetch(c);
        });
        inv_passes<LOGN, NT>(cta, buf, itw, p);
        cta.par([&](int tid) { inv_store_stage<LOGN, NT>(buf, itw, p, tid, emit); });
    } else {
        constexpr int HC = NC / 2;
        U64x2 *wrk = reinterpret_cast<U64x2 *>(work);
        for (int h = 0; h < 2; ++h) {
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) reinterpret_cast<U64x2 *>(buf)[swz_chunk(lc)] = fetch(h * HC + lc);
            });
            inv_passes_blk<LOGN, NT, 2>(cta, buf, itw, p, 2 * h);
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) st_cg(wrk + h * HC + lc, reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)]);
            });
        }
        cta.par([&](int tid) { inv_outer_stage<LOGN, NT>(itw, p, tid, [&](int c) { return ld_cg(wrk + c); }, emit); });
    }
}

// step 2, one (polynomial, kept limb i): out = (c[i] - s * NTT_i(centred(tau') mod q_i)) * q_last^-1 mod q_i.
// COHERENT: c[i] is an L2-resident lazy accumulator written in this launch (any 64-bit value; may be `out_limb`).
// LIFT(chunk): the residue mod q_i of the (centred) value to subtract, lazy below 4q.
// ADD: add_limb (canonical, N words) is added to the result before the store, one csub(q) keeping it canonical: a Horner step
// rot(acc) + inner_g of a linear layer in the store that writes the rotation anyway (bit-identical to a separate poly_add).
template <int LOGN, int NT, bool COHERENT, bool ADD = false, class CTA, class LIFT>
DPFHE_HD void ms_limb_core(CTA &cta, u64 *buf, LIFT lift, const u64 *c_limb, u64 *out_limb, const Twiddle *tw, const LimbParams &p,
                           const MsConsts &K, u32 i, const u64 *add_limb = nullptr) {
    constexpr int NC = 1 << (LOGN - 1);
    const U64x2 *cin = reinterpret_cast<const U64x2 *>(c_limb);
    const U64x2 *addend = reinterpret_cast<const U64x2 *>(add_limb);
    U64x2 *dst = reinterpret_cast<U64x2 *>(out_limb);
    const u64 inv = K.inv[i], inv_s = K.inv_s[i], sinv = K.sinv[i], sinv_s = K.sinv_s[i];
    // c: chunk of the limb; c_buf: where its transform output sits in shared memory
    auto finish = [&](int c, int c_buf) {
        const U64x2 u = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c_buf)], cv = COHERENT ? ld_cg(cin + c) : ld_stream(cin + c);
        U64x2 r;   // c*inv - u*(s*inv): both Shoup products below 2q, difference kept positive with + 2q
        r.x = canon4(shoup_exact(cv.x, inv, inv_s, p) + p.q2 - shoup_exact(u.x, sinv, sinv_s, p), p);
        r.y = canon4(shoup_exact(cv.y, inv, inv_s, p) + p.q2 - shoup_exact(u.y, sinv, sinv_s, p), p);
        if constexpr (ADD) {   // both canonical: the sum is below 2q
            const U64x2 a = ld_stream(addend + c);
            r.x = csub(r.x + a.x, p.q);
            r.y = csub(r.y + a.y, p.q);
        }
        st_stream(dst + c, r);
    };
    if constexpr (LOGN <= 13 || NT >= 512) {
        cta.par([&](int tid) { fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, lift); });
        fwd_passes<LOGN, NT, 4>(cta, buf, tw, p);
        cta.par([&](int tid) {
            for (int c = tid; c < NC; c += NT) finish(c, c);
        });
    } else {
        constexpr int HC = NC / 2;
        for (int h = 0; h < 2; ++h) {
            cta.par([&](int tid) { fwd_load_stage_half<LOGN, NT, false>(buf, tw, p, tid, lift, h); });
            fwd_passes_blk<LOGN, NT, 4, 2>(cta, buf, tw, p, 2 * h);
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) finish(h * HC + lc, lc);
            });
        }
    }
}

template <int LOGN, int NT, bool COHERENT = false, class CTA>
DPFHE_HD void ms_limb_body(CTA &cta, u64 *buf, const u64 *tau, const u64 *c_limb, u64 *out_limb, const Twiddle *tw, const LimbParams &p,
                           const MsConsts &K, u32 i) {
    const U64x2 *src = reinterpret_cast<const U64x2 *>(tau);
    const u64 half = K.half, neg_ql = p.q - K.qlm[i];   // adding (q_i - q_last mod q_i) subtracts q_last
    auto lift = [&](int c) {
        const U64x2 v = ld_cg(src + c);
        U64x2 r;                                 // centred lift, lazy: < 3q (+ < q when tau' is "negative")
        r.x = word_reduce(v.x, p) + (v.x > half ? neg_ql : 0);
        r.y = word_reduce(v.y, p) + (v.y > half ? neg_ql : 0);
        return r;
    };
    ms_limb_core<LOGN, NT, COHERENT>(cta, buf, lift, c_limb, out_limb, tw, p, K, i);
}

// division by the product P of K special primes (DESIGN.md §2.11): tau_rows + k * tau_stride is y_k = tau'_k * Phat_k^-1 of
// special prime k; the value to subtract is sum_k centred(y_k) * Phat_k, converted term by term.  ADD / add_limb: as ms_limb_core.
// DROP (multiply-and-rescale, DESIGN.md §2.19 / §4.16): the divided set has a fifth row, y_qbar of the dropped limb in drop_row, with
// its own constants in R (P mod q_i, floor(qbar / 2)); G and K then describe P' = P * qbar.  K + 1 terms: the per-term reduction
// holds up to five (15q < 16q), and the slim form up to three.
template <int LOGN, int NT, bool COHERENT = true, bool ADD = false, bool DROP = false, class CTA>
DPFHE_HD void ms_limb_group(CTA &cta, u64 *buf, const u64 *tau_rows, size_t tau_stride, const u64 *c_limb, u64 *out_limb, const Twiddle *tw,
                            const LimbParams &p, const MsConsts &K, const GroupConsts &G, u32 i, const u64 *add_limb = nullptr,
                            const u64 *drop_row = nullptr, const RescaleConsts *R = nullptr) {
    const u64 neg_p = G.neg_p[i];
    auto lift = [&](int c) {
        U64x2 r;
        r.x = r.y = 0;
        const bool slim = G.K + (DROP ? 1u : 0u) <= 3;   // terms below SB*q + q = 5q: three of them stay below 16q, four or five need the per-term reduction (3q each)
        for (u32 k = 0; k < G.K; ++k) {
            const U64x2 v = ld_cg(reinterpret_cast<const U64x2 *>(tau_rows + (size_t)k * tau_stride) + c);
            u64 tx = shoup_lazy(v.x, G.dn[k][i], G.dn_s[k][i], p), ty = shoup_lazy(v.y, G.dn[k][i], G.dn_s[k][i], p);
            if (!slim) {
                tx = csub(tx, p.q2);
                ty = csub(ty, p.q2);
            }
            r.x += tx + (v.x > G.half[k] ? neg_p : 0);
            r.y += ty + (v.y > G.half[k] ? neg_p : 0);
        }
        if constexpr (DROP) {   // the fifth row: the same term with the dropped limb's constants
            const U64x2 v = ld_cg(reinterpret_cast<const U64x2 *>(drop_row) + c);
            u64 tx = shoup_lazy(v.x, R->dn[i], R->dn_s[i], p), ty = shoup_lazy(v.y, R->dn[i], R->dn_s[i], p);
            if (!slim) {
                tx = csub(tx, p.q2);
                ty = csub(ty, p.q2);
            }
            r.x += tx + (v.x > R->half ? neg_p : 0);
            r.y += ty + (v.y > R->half ? neg_p : 0);
        }
        r.x = csub(csub(r.x, p.q8), p.q4);   // < 16q  ->  < 4q
        r.y = csub(csub(r.y, p.q8), p.q4);
        return r;
    };
    ms_limb_core<LOGN, NT, COHERENT, ADD>(cta, buf, lift, c_limb, out_limb, tw, p, K, i, add_limb);
}

// ---- hoisted rotations (DESIGN.md §2.8b, §4.4d) ---------------------------------------------------
// Many rotations of the SAME ciphertexts share everything that does not depend on the Galois element: the inverse
// transform of the digits and their forward transforms into every other limb.  With t_j = INTT_j(c1[j]) and
// U_ji = NTT_i(t_j mod q_i), the digit of rotation g satisfies, in Z_{q_i},
//     NTT_i( canonical(sigma_g t_j) mod q_i ) = perm_g(U_ji) + (q_j mod q_i) * NTT_i(negmask_g)
// whenever no coefficient of t_j is zero: a negated coefficient is stored as q_j - t, and (q_j - t) mod q_i differs from
// -(t mod q_i) by q_j mod q_i.  The data-independent second term is folded into a per-rotation constant (kprime).
// Ciphertexts with a zero coefficient in some t_j are flagged and recomputed by the ordinary rotate kernel.
struct HoistArgs {
    const u64 *ct;       // [batch][2][L][N]
    u64 *U;              // [batch][L j][L i][N]: NTT_i(t_j mod q_i), lazy (< 16 q_i); the diagonal j == i holds c1[i] itself
    u64 *scratch;        // digit exchange slots, as KsArgs::scratch
    u32 *zero;           // [batch] set to 1 when some t_j has a zero coefficient
    const Twiddle *tw, *itw;
    u32 L;
};

// digit = the limb `row` as it is: copy it to `own` (its entry of U) and publish its inverse transform; zero (optional) is set when
// a coefficient of the inverse transform is zero
template <int LOGN, int NT, class CTA>
DPFHE_HD void hoist_phase1_core(CTA &cta, u64 *buf, const u64 *row, u64 *own, u32 *zero, const Twiddle *itw, const LimbParams &p, u64 *t_slot) {
    constexpr int N = 1 << LOGN, NC = N / 2;
    const U64x2 *src = reinterpret_cast<const U64x2 *>(row);
    U64x2 *dst = reinterpret_cast<U64x2 *>(t_slot);
    U64x2 *diag = reinterpret_cast<U64x2 *>(own);
    auto build = [&](int c_lo, int n_c) {
        cta.par([&](int tid) {
            for (int lc = tid; lc < n_c; lc += NT) {
                const U64x2 v = ld_stream(src + c_lo + lc);
                reinterpret_cast<U64x2 *>(buf)[swz_chunk(lc)] = v;
                st_stream(diag + c_lo + lc, v);
            }
        });
    };
    auto emit = [&](int c, const U64x2 &v) {
        if (zero && (v.x == 0 || v.y == 0)) *zero = 1u;
        st_cg(dst + c, v);
    };
    if constexpr (LOGN <= 13) {
        build(0, NC);
        inv_passes<LOGN, NT>(cta, buf, itw, p);
        cta.par([&](int tid) { inv_store_stage<LOGN, NT>(buf, itw, p, tid, emit); });
    } else {
        constexpr int HC = NC / 2;
        for (int h = 0; h < 2; ++h) {
            build(h * HC, HC);
            inv_passes_blk<LOGN, NT, 2>(cta, buf, itw, p, 2 * h);
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) st_cg(dst + h * HC + lc, reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)]);
            });
        }
        cta.par([&](int tid) { inv_outer_stage<LOGN, NT>(itw, p, tid, [&](int c) { return ld_cg(dst + c); }, emit); });
    }
}

// digit = c1[i] as it is
template <int LOGN, int NT, class CTA>
DPFHE_HD void hoist_phase1(CTA &cta, u64 *buf, const HoistArgs &A, const LimbParams &p, size_t ct, u32 i, u64 *t_slot) {
    constexpr size_t N = (size_t)1 << LOGN;
    const size_t P = (size_t)A.L * N;
    // the digit itself is the i == j entry of U (a plain copy), so that the apply step reads every digit the same way
    hoist_phase1_core<LOGN, NT>(cta, buf, A.ct + ct * 2 * P + P + (size_t)i * N, A.U + ((ct * A.L + i) * A.L + i) * N, A.zero + ct,
                                A.itw + (size_t)i * N, p, t_slot);
}

// forward transform of a lifted digit into `out_row` (lazy, below 16q).  LOAD(h) as in ks_phase2_core, values below BIN*q.
template <int LOGN, int NT, int BIN, class CTA, class LOAD>
DPFHE_HD void hoist_phase2_core(CTA &cta, u64 *buf, const Twiddle *tw, const LimbParams &p, LOAD load, u64 *out_row) {
    constexpr int N = 1 << LOGN, NC = N / 2;
    U64x2 *dst = reinterpret_cast<U64x2 *>(out_row);
    if constexpr (LOGN <= 13) {
        load(0);
        fwd_passes<LOGN, NT, BIN>(cta, buf, tw, p);
        cta.par([&](int tid) {
            for (int c = tid; c < NC; c += NT) st_stream(dst + c, reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c)]);
        });
    } else {
        constexpr int HC = NC / 2;
        for (int h = 0; h < 2; ++h) {
            load(h);
            fwd_passes_blk<LOGN, NT, BIN, 2>(cta, buf, tw, p, 2 * h);
            cta.par([&](int tid) {
                for (int lc = tid; lc < HC; lc += NT) st_stream(dst + h * HC + lc, reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lc)]);
            });
        }
    }
}

// U[ct][j][i] = NTT_i(t_j mod q_i)
template <int LOGN, int NT, class CTA>
DPFHE_HD void hoist_phase2(CTA &cta, u64 *buf, const HoistArgs &A, const LimbParams &p, size_t ct, u32 i, u32 j, const u64 *t_src) {
    constexpr size_t N = (size_t)1 << LOGN;
    const Twiddle *tw = A.tw + (size_t)i * N;
    const U64x2 *src = reinterpret_cast<const U64x2 *>(t_src);
    auto get = [&](int c) { return ld_cg(src + c); };
    auto load = [&](int h) {
        cta.par([&](int tid) {
            if constexpr (LOGN <= 13) fwd_load_stage<LOGN, NT, true>(buf, tw, p, tid, get);
            else fwd_load_stage_half<LOGN, NT, true>(buf, tw, p, tid, get, h);
        });
    };
    hoist_phase2_core<LOGN, NT, 3>(cta, buf, tw, p, load, A.U + ((ct * A.L + j) * A.L + i) * N);
}

// ---- hoisted rotations with grouped hybrid keys (DESIGN.md §2.11b) ------------------------------------
// The rotations of one batch share the whole mod-up: U[ct][g][i] = the lift of digit g of the UNPERMUTED c1 in limb i (evaluation
// form; the member limbs hold c1[i] itself).  A rotation permutes the rows of U instead of lifting the permuted digits: the same
// plaintext and noise bound, not the bits of the non-hoisted rotate.
struct HoistGArgs {
    const u64 *ct;       // [batch][2][Lq][N]
    u64 *U;              // [batch][dnum][L][N]
    u64 *scratch;        // digit exchange slots, as KsArgs::scratch
    const Twiddle *tw, *itw;
};

template <int LOGN, int NT, class CTA>
DPFHE_HD void hoistg_phase1(CTA &cta, u64 *buf, const HoistGArgs &A, const GroupConsts &G, size_t ct, u32 i, u64 *t_slot) {
    constexpr size_t N = (size_t)1 << LOGN;
    const size_t Pq = (size_t)G.Lq * N, L = G.Lq + G.K;
    hoist_phase1_core<LOGN, NT>(cta, buf, A.ct + ct * 2 * Pq + Pq + (size_t)i * N, A.U + ((ct * G.dnum + i / G.K) * L + i) * N, nullptr,
                                A.itw + (size_t)i * N, G.lp_up[i], t_slot);
}

// U[ct][g][i] for a limb i outside digit g (ciphertext or special limb): the basis conversion of ks_phase2_group, then the transform
template <int LOGN, int NT, class CTA>
DPFHE_HD void hoistg_phase2(CTA &cta, u64 *buf, const HoistGArgs &A, const GroupConsts &G, const LimbParams &p, size_t ct, u32 i, u32 g,
                            const u64 *t_rows, size_t t_stride) {
    constexpr size_t N = (size_t)1 << LOGN;
    const Twiddle *tw = A.tw + (size_t)i * N;
    const u32 lo = g * G.K, hi = lo + G.K < G.Lq ? lo + G.K : G.Lq, L = G.Lq + G.K;
    auto get = [&](int c) {
        U64x2 r;
        r.x = r.y = 0;
        for (u32 j = lo; j < hi; ++j) {   // bounds as in ks_phase2_group
            const U64x2 v = ld_cg(reinterpret_cast<const U64x2 *>(t_rows + (size_t)j * t_stride) + c);
            r.x += shoup_lazy(v.x, G.up[j][i], G.up_s[j][i], p);
            r.y += shoup_lazy(v.y, G.up[j][i], G.up_s[j][i], p);
        }
        if (hi - lo > 2) {
            r.x = csub(r.x, p.q8);
            r.y = csub(r.y, p.q8);
        }
        r.x = csub(r.x, p.q4);
        r.y = csub(r.y, p.q4);
        return r;
    };
    auto load = [&](int h) {
        cta.par([&](int tid) {
            if constexpr (LOGN <= 13) fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, get);
            else fwd_load_stage_half<LOGN, NT, false>(buf, tw, p, tid, get, h);
        });
    };
    hoist_phase2_core<LOGN, NT, 4>(cta, buf, tw, p, load, A.U + ((ct * G.dnum + g) * L + i) * N);
}

// CB ciphertexts ct0 .. ct0+n_ct-1 (n_ct <= CB) share every key chunk they multiply with.  PF: the operands of digit
// j + 1 (gathered transforms and key chunks) are requested before the arithmetic of digit j, which is what this
// latency-bound loop needs (measured: sharing key chunks between ciphertexts does not help, more loads in flight do).
template <int CB>
struct RotOperands {
    U64x2 vb, vbs, va, vas, u[CB];
};

// one rotation applied to the shared lifts: acc[ct][c][i] = [i < Lq, c = 0] P * perm(c0[i]) + sum_g perm(U[ct][g][i]) o key[g][c][i]
// for all L limbs, canonical; the division by P (md_tau / md_limb kernels) then yields (perm(c0) + ks0, ks1).
struct RotApplyGArgs {
    const u64 *ct;       // [batch][2][Lq][N]
    const u64 *U;        // [batch][dnum][L][N]
    const u64 *key;      // [dnum][2][L][N] Galois key of this rotation
    const u64 *key_s;    // its Shoup companions
    u64 *acc;            // [batch][2][L][N]
    u32 galois;
};

// LV (DESIGN.md §4.18): the key is a top-level key, key_shift rows longer than the view's per (digit, component), read through
// ks_key_row with its companions, as in rot_sum_grouped_rows; the lifted digits U keep the view's layout.
template <int LOGN, int NT, int CB, bool LV = false, class CTA>
DPFHE_HD void rot_apply_grouped_rows(CTA &cta, const RotApplyGArgs &A, const GroupConsts &G, const MsConsts &K, const LimbParams &p, size_t ct0,
                                     u32 n_ct, u32 i, int c_lo = 0, int c_hi = 1 << (LOGN - 1), u32 key_shift = 0) {
    constexpr int N = 1 << LOGN;
    const u32 L = G.Lq + G.K, D = G.dnum, g = A.galois;
    const size_t P = (size_t)L * N, Pq = (size_t)G.Lq * N;
    const bool limb = i < G.Lq;
    const u64 pm = limb ? K.qlm[i] : 0, pm_s = limb ? K.qlm_s[i] : 0;   // P mod q_i: the c0 term is carried through the division
    cta.par([&](int tid) {
#pragma unroll 1
        for (int c = c_lo + tid; c < c_hi; c += NT) {
            const int pi0 = galois_index<LOGN>(2 * c, g);
            const int pc = pi0 >> 1;
            const bool swap = (pi0 & 1) != 0;
            auto gather = [&](const u64 *row) {
                const U64x2 v = ld_stream(reinterpret_cast<const U64x2 *>(row) + pc);
                U64x2 r;
                r.x = swap ? v.y : v.x;
                r.y = swap ? v.x : v.y;
                return r;
            };
            // the operands of digit d + 1 (key chunks and gathered rows) are requested before the arithmetic of digit d: the loop
            // is bound by the latency of the gathers (ncu: long-scoreboard stalls), as in rot_apply_rows
            auto fetch = [&](u32 d, RotOperands<CB> &o) {
                size_t kb, ka;
                if constexpr (LV) {
                    const size_t PK = (size_t)(L + key_shift) * N, kr = ks_key_row(i, G.Lq, key_shift);
                    kb = ((size_t)d * 2 + 0) * PK + kr * N;
                    ka = ((size_t)d * 2 + 1) * PK + kr * N;
                } else {
                    kb = ((size_t)d * 2 + 0) * P + (size_t)i * N;
                    ka = ((size_t)d * 2 + 1) * P + (size_t)i * N;
                }
                o.vb = ld_keep(reinterpret_cast<const U64x2 *>(A.key + kb) + c);
                o.vbs = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s + kb) + c);
                o.va = ld_keep(reinterpret_cast<const U64x2 *>(A.key + ka) + c);
                o.vas = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s + ka) + c);
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    const size_t ct = ct0 + ((u32)b < n_ct ? (u32)b : n_ct - 1);   // rows past the end repeat the last one, not stored
                    o.u[b] = gather(A.U + ((ct * D + d) * L + i) * N);
                }
            };
            U64x2 r0[CB], r1[CB];
            auto mac = [&](const RotOperands<CB> &o, bool trim) {
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    r0[b].x += shoup_lazy(o.u[b].x, o.vb.x, o.vbs.x, p);
                    r0[b].y += shoup_lazy(o.u[b].y, o.vb.y, o.vbs.y, p);
                    r1[b].x += shoup_lazy(o.u[b].x, o.va.x, o.vas.x, p);
                    r1[b].y += shoup_lazy(o.u[b].y, o.va.y, o.vas.y, p);
                    if (trim) {
                        r0[b].x = csub(r0[b].x, p.q8); r0[b].y = csub(r0[b].y, p.q8);
                        r1[b].x = csub(r1[b].x, p.q8); r1[b].y = csub(r1[b].y, p.q8);
                    }
                }
            };
            RotOperands<CB> oa, ob;
            fetch(0, oa);
#pragma unroll
            for (int b = 0; b < CB; ++b) {
                r0[b].x = r0[b].y = r1[b].x = r1[b].y = 0;
                if (limb) {
                    const size_t ct = ct0 + ((u32)b < n_ct ? (u32)b : n_ct - 1);
                    const U64x2 s0 = gather(A.ct + ct * 2 * Pq + (size_t)i * N);
                    // LV: read from the parameter block here rather than held across the loop, as rot_sum_grouped_rows does: the
                    // generic variant's level instance fits its 80 registers that way
                    const u64 m = LV ? K.qlm[i] : pm, m_s = LV ? K.qlm_s[i] : pm_s;
                    r0[b].x = shoup_lazy(s0.x, m, m_s, p);   // < SB*q
                    r0[b].y = shoup_lazy(s0.y, m, m_s, p);
                }
            }
            for (u32 d = 0; d < D; d += 2) {
                if (d + 1 < D) fetch(d + 1, ob);
                mac(oa, d + 1 < D && acc_trim_after(SB, (int)d));   // no trim after the last digit: canon takes any value below 16q
                if (d + 1 < D) {
                    if (d + 2 < D) fetch(d + 2, oa);
                    mac(ob, d + 2 < D && acc_trim_after(SB, (int)d + 1));
                }
            }
#pragma unroll
            for (int b = 0; b < CB; ++b) {
                if ((u32)b < n_ct) {
                    U64x2 o0, o1;
                    o0.x = canon(r0[b].x, p); o0.y = canon(r0[b].y, p);
                    o1.x = canon(r1[b].x, p); o1.y = canon(r1[b].y, p);
                    st_stream(reinterpret_cast<U64x2 *>(A.acc + (ct0 + b) * 2 * P + (size_t)i * N) + c, o0);
                    st_stream(reinterpret_cast<U64x2 *>(A.acc + (ct0 + b) * 2 * P + P + (size_t)i * N) + c, o1);
                }
            }
        }
    });
}

// ---- summed rotations with grouped hybrid keys (DESIGN.md §2.17) --------------------------------------
// The key-switch accumulators of n_rot rotations of the same ciphertexts, summed before ONE division by P:
//   acc[ct][0][i] = [i < Lq] P * (c0[i] + sum_m perm_m(c0[i])) + sum_m sum_g perm_m(U[ct][g][i]) o key_m[g][0][i]
//   acc[ct][1][i] = [i < Lq] P * c1[i]                         + sum_m sum_g perm_m(U[ct][g][i]) o key_m[g][1][i]
// for all L limbs, canonical; md_tau / md_limb then yield (c0 + sum_m perm_m(c0) + ks0, c1 + ks1).  The carried terms are
// multiples of P, so they pass the division exactly (their special residues are 0).
struct RotSumGArgs {
    const u64 *ct;                     // [batch][2][Lq][N]
    const u64 *U;                      // [batch][dnum][L][N]
    const u64 *key[ROT_SUM_MAX];       // [dnum][2][L][N] Galois key of rotation m
    const u64 *key_s[ROT_SUM_MAX];     // its Shoup companions
    u64 *acc;                          // [batch][2][L][N]
    u32 galois[ROT_SUM_MAX];
    u32 n_rot;
};

// The trim schedule of a lazy accumulator row that starts below SB*q and gains one Shoup product (< SB*q) per add(): the running
// bound b (multiples of q) never passes 16; add() returns whether the row takes csub(8q) right after the addition, which it does
// whenever the next addition could pass 16q (the rule of acc_trim_after, kept incrementally).
struct LazyBound {
    int b = SB;
    DPFHE_HD bool add() {
        b += SB;
        const bool t = b + SB > 16;
        if (t) b = 8;
        return t;
    }
};

// The rotation loop runs inside the per-chunk loop on the same register accumulators and the operands of rot_apply_grouped_rows
// (RotOperands): the registers do not grow with n_rot.  On a ciphertext limb every rotation has one more "digit" after its dnum
// digits: its gathered c0 times the constant P mod q_i (key row 1: zero), which carries P * perm_m(c0) into r0.
// Lazy bound: both rows start below SB*q (P * c0 and P * c1, ciphertext limbs) and gain one Shoup product (< SB*q) per pair,
// n_rot * (dnum + 1) <= 15 (dnum + 1) of them; a row takes csub(8q) after a pair whenever the next addition could pass 16q (the
// rule of acc_trim_after, kept as a running bound), so every value stays below 16q, what canon accepts.
// LV (DESIGN.md §4.17): the keys are top-level keys, key_shift rows longer than the view's per (digit, component), read through
// ks_key_row; the lifted digits U keep the view's layout.
template <int LOGN, int NT, int CB, bool LV = false, class CTA>
DPFHE_HD void rot_sum_grouped_rows(CTA &cta, const RotSumGArgs &A, const GroupConsts &G, const MsConsts &K, const LimbParams &p, size_t ct0,
                                   u32 n_ct, u32 i, int c_lo = 0, int c_hi = 1 << (LOGN - 1), u32 key_shift = 0) {
    constexpr int N = 1 << LOGN;
    const u32 L = G.Lq + G.K, D = G.dnum;
    const size_t P = (size_t)L * N, Pq = (size_t)G.Lq * N;
    const bool limb = i < G.Lq;
    const u32 DM = D + (limb ? 1u : 0u), T = A.n_rot * DM;   // pairs per rotation; T (rotation, digit) pairs, rotation-major
    // P mod q_i and its companion are read from the parameter block where they are used (K.qlm[i], K.qlm_s[i]; ciphertext limbs
    // only) rather than held in registers across the loop: the generic variant's body fits its 80 registers that way
    cta.par([&](int tid) {
#pragma unroll 1
        for (int c = c_lo + tid; c < c_hi; c += NT) {
            auto ct_of = [&](int b) { return ct0 + ((u32)b < n_ct ? (u32)b : n_ct - 1); };   // rows past the end repeat the last one, not stored
            // the operands of pair k + 1 (key chunks and gathered rows) are requested before the arithmetic of pair k, as in
            // rot_apply_grouped_rows; the gather positions of a pair are those of its rotation
            auto fetch = [&](u32 k, RotOperands<CB> &o) {
                const u32 m = k / DM, d = k - m * DM;
                const int pi0 = galois_index<LOGN>(2 * c, A.galois[m]);
                const int pc = pi0 >> 1;
                const bool swap = (pi0 & 1) != 0;
                auto gather = [&](const u64 *row) {
                    const U64x2 v = ld_stream(reinterpret_cast<const U64x2 *>(row) + pc);
                    U64x2 r;
                    r.x = swap ? v.y : v.x;
                    r.y = swap ? v.x : v.y;
                    return r;
                };
                if (d < D) {
                    size_t kb, ka;
                    if constexpr (LV) {
                        const size_t PK = (size_t)(L + key_shift) * N, kr = ks_key_row(i, G.Lq, key_shift);
                        kb = ((size_t)d * 2 + 0) * PK + kr * N;
                        ka = ((size_t)d * 2 + 1) * PK + kr * N;
                    } else {
                        kb = ((size_t)d * 2 + 0) * P + (size_t)i * N;
                        ka = ((size_t)d * 2 + 1) * P + (size_t)i * N;
                    }
                    o.vb = ld_keep(reinterpret_cast<const U64x2 *>(A.key[m] + kb) + c);
                    o.vbs = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s[m] + kb) + c);
                    o.va = ld_keep(reinterpret_cast<const U64x2 *>(A.key[m] + ka) + c);
                    o.vas = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s[m] + ka) + c);
#pragma unroll
                    for (int b = 0; b < CB; ++b) o.u[b] = gather(A.U + ((ct_of(b) * D + d) * L + i) * N);
                } else {   // the carried term perm_m(c0) * P
                    o.vb.x = o.vb.y = K.qlm[i];
                    o.vbs.x = o.vbs.y = K.qlm_s[i];
                    o.va.x = o.va.y = o.vas.x = o.vas.y = 0;
#pragma unroll
                    for (int b = 0; b < CB; ++b) o.u[b] = gather(A.ct + ct_of(b) * 2 * Pq + (size_t)i * N);
                }
            };
            U64x2 r0[CB], r1[CB];
            LazyBound bnd;   // running bound of both rows
            auto mac = [&](const RotOperands<CB> &o) {
                const bool trim = bnd.add();
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    r0[b].x += shoup_lazy(o.u[b].x, o.vb.x, o.vbs.x, p);
                    r0[b].y += shoup_lazy(o.u[b].y, o.vb.y, o.vbs.y, p);
                    r1[b].x += shoup_lazy(o.u[b].x, o.va.x, o.vas.x, p);
                    r1[b].y += shoup_lazy(o.u[b].y, o.va.y, o.vas.y, p);
                    if (trim) {
                        r0[b].x = csub(r0[b].x, p.q8); r0[b].y = csub(r0[b].y, p.q8);
                        r1[b].x = csub(r1[b].x, p.q8); r1[b].y = csub(r1[b].y, p.q8);
                    }
                }
            };
            RotOperands<CB> oa, ob;
            fetch(0, oa);
#pragma unroll
            for (int b = 0; b < CB; ++b) {
                r0[b].x = r0[b].y = r1[b].x = r1[b].y = 0;
                if (limb) {   // the unrotated ciphertext, times P
                    const size_t row = ct_of(b) * 2 * Pq + (size_t)i * N;
                    const U64x2 v0 = ld_stream(reinterpret_cast<const U64x2 *>(A.ct + row) + c);
                    const U64x2 v1 = ld_stream(reinterpret_cast<const U64x2 *>(A.ct + row + Pq) + c);
                    const u64 pm = K.qlm[i], pm_s = K.qlm_s[i];
                    r0[b].x = shoup_lazy(v0.x, pm, pm_s, p);   // < SB*q
                    r0[b].y = shoup_lazy(v0.y, pm, pm_s, p);
                    r1[b].x = shoup_lazy(v1.x, pm, pm_s, p);
                    r1[b].y = shoup_lazy(v1.y, pm, pm_s, p);
                }
            }
            for (u32 k = 0; k < T; k += 2) {
                if (k + 1 < T) fetch(k + 1, ob);
                mac(oa);
                if (k + 1 < T) {
                    if (k + 2 < T) fetch(k + 2, oa);
                    mac(ob);
                }
            }
#pragma unroll
            for (int b = 0; b < CB; ++b) {
                if ((u32)b < n_ct) {
                    U64x2 o0, o1;
                    o0.x = canon(r0[b].x, p); o0.y = canon(r0[b].y, p);
                    o1.x = canon(r1[b].x, p); o1.y = canon(r1[b].y, p);
                    st_stream(reinterpret_cast<U64x2 *>(A.acc + (ct0 + b) * 2 * P + (size_t)i * N) + c, o0);
                    st_stream(reinterpret_cast<U64x2 *>(A.acc + (ct0 + b) * 2 * P + P + (size_t)i * N) + c, o1);
                }
            }
        }
    });
}

// one (ciphertext, limb i) row pair of one rotation: out = (perm(c0) + ks0, ks1) with the switched pair assembled from the
// shared transforms.  pi(2c + 1) = pi(2c) ^ 1 (flipping the lowest index bit flips the highest exponent bit, and g is odd),
// so the two coefficients of an output chunk come from one 16-byte chunk of the source row.
struct RotApplyArgs {
    const u64 *ct;       // [batch][2][L][N]
    const u64 *U;        // [batch][L][L][N] (diagonal = c1 limbs); nullptr when L == 1: the only digit is c1[0] itself
    const u64 *key;      // [L][2][L][N] Galois key of this rotation
    const u64 *key_s;    // its Shoup companions
    const u64 *kprime;   // [2][L][N] canonical: NTT_i(negmask_g) o sum_{j != i} (q_j mod q_i) * key[j][c][i]
    u64 *out;            // [batch][2][L][N]
    u32 L, galois;
};


template <int LOGN, int NT, int CB, bool PF, class CTA>
DPFHE_HD void rot_apply_rows(CTA &cta, const RotApplyArgs &A, const LimbParams &p, size_t ct0, u32 n_ct, u32 i, int c_lo = 0,
                             int c_hi = 1 << (LOGN - 1)) {
    constexpr int N = 1 << LOGN;
    const u32 L = A.L, g = A.galois;
    const size_t P = (size_t)L * N;
    const U64x2 *kp0 = reinterpret_cast<const U64x2 *>(A.kprime + (size_t)i * N), *kp1 = reinterpret_cast<const U64x2 *>(A.kprime + P + (size_t)i * N);
    cta.par([&](int tid) {
#pragma unroll 1
        for (int c = c_lo + tid; c < c_hi; c += NT) {   // chunk range [c_lo, c_hi) of the row
            const int pi0 = galois_index<LOGN>(2 * c, g);
            const int pc = pi0 >> 1;
            const bool swap = (pi0 & 1) != 0;
            auto gather = [&](const u64 *row) {
                const U64x2 v = ld_stream(reinterpret_cast<const U64x2 *>(row) + pc);
                U64x2 r;
                r.x = swap ? v.y : v.x;
                r.y = swap ? v.x : v.y;
                return r;
            };
            auto fetch = [&](u32 j, RotOperands<CB> &o) {
                const size_t kb = ((size_t)j * 2 + 0) * P + (size_t)i * N, ka = ((size_t)j * 2 + 1) * P + (size_t)i * N;
                o.vb = ld_keep(reinterpret_cast<const U64x2 *>(A.key + kb) + c);
                o.vbs = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s + kb) + c);
                o.va = ld_keep(reinterpret_cast<const U64x2 *>(A.key + ka) + c);
                o.vas = ld_keep(reinterpret_cast<const U64x2 *>(A.key_s + ka) + c);
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    const size_t ct = ct0 + ((u32)b < n_ct ? (u32)b : n_ct - 1);   // rows past the end repeat the last one, not stored
                    o.u[b] = gather(A.U != nullptr ? A.U + ((ct * L + j) * L + i) * N : A.ct + ct * 2 * P + P);
                }
            };
            U64x2 r0[CB], r1[CB];
            auto mac = [&](const RotOperands<CB> &o, bool trim) {
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    r0[b].x += shoup_lazy(o.u[b].x, o.vb.x, o.vbs.x, p);
                    r0[b].y += shoup_lazy(o.u[b].y, o.vb.y, o.vbs.y, p);
                    r1[b].x += shoup_lazy(o.u[b].x, o.va.x, o.vas.x, p);
                    r1[b].y += shoup_lazy(o.u[b].y, o.va.y, o.vas.y, p);
                    if (trim) {   // + SB*q per digit from below 2q: csub(8q) whenever the next digit could pass 16q
                        r0[b].x = csub(r0[b].x, p.q8); r0[b].y = csub(r0[b].y, p.q8);
                        r1[b].x = csub(r1[b].x, p.q8); r1[b].y = csub(r1[b].y, p.q8);
                    }
                }
            };
            RotOperands<CB> oa, ob;   // two operand sets used alternately: the loads of one fly during the arithmetic of the other
            fetch(0, oa);
            {
                const U64x2 k0 = ld_keep(kp0 + c), k1 = ld_keep(kp1 + c);
#pragma unroll
                for (int b = 0; b < CB; ++b) {
                    const size_t ct = ct0 + ((u32)b < n_ct ? (u32)b : n_ct - 1);
                    const U64x2 s0 = gather(A.ct + ct * 2 * P + (size_t)i * N);
                    r0[b].x = k0.x + s0.x;   // < 2q
                    r0[b].y = k0.y + s0.y;
                    r1[b] = k1;
                }
            }
            for (u32 j = 0; j < L; j += 2) {
                if (PF && j + 1 < L) fetch(j + 1, ob);
                mac(oa, j + 1 < L && acc_trim_after(2, (int)j));   // no trim after the last digit: canon takes any value below 16q
                if (j + 1 < L) {
                    if (!PF) fetch(j + 1, ob);
                    if (PF && j + 2 < L) fetch(j + 2, oa);
                    mac(ob, j + 2 < L && acc_trim_after(2, (int)j + 1));
                    if (!PF && j + 2 < L) fetch(j + 2, oa);
                }
            }
#pragma unroll
            for (int b = 0; b < CB; ++b) {
                if ((u32)b < n_ct) {
                    U64x2 o0, o1;
                    o0.x = canon(r0[b].x, p); o0.y = canon(r0[b].y, p);
                    o1.x = canon(r1[b].x, p); o1.y = canon(r1[b].y, p);
                    st_stream(reinterpret_cast<U64x2 *>(A.out + (ct0 + b) * 2 * P + (size_t)i * N) + c, o0);
                    st_stream(reinterpret_cast<U64x2 *>(A.out + (ct0 + b) * 2 * P + P + (size_t)i * N) + c, o1);
                }
            }
        }
    });
}

// ---- plaintext inner products: out[g] = sum_b steps[b] o pts[g][b]  (baby-step/giant-step inner loop, DESIGN.md §4.7) ----
// One CTA owns a tile of PTI_COEFFS coefficients of one limb for a block of giant steps: the plaintext tile
// [gcnt][nb][16] stays in shared memory while the whole batch streams through, so every ciphertext row is read once
// and every output row written once (instead of one read-modify-write pass over the batch per diagonal).
// Operands are pre-split into 30-bit halves when they are staged, so a multiply-accumulate is four IMAD.WIDE with
// 64-bit accumulators and no carry handling: 16 products of two values below 2^30 fit in 64 bits.
struct PtInnerArgs {
    const u64 *steps;   // [nb][batch][2][L][N] ciphertext batches (e.g. the baby-step rotations)
    const u64 *pts;     // [ng][nb][L][N] plaintexts, evaluation form, shared by the batch
    u64 *out;           // [ng][batch][2][L][N]
    size_t batch;
    u32 L, nb, ng;
};
constexpr int PTI_COEFFS = 16;   // coefficients per tile: one 128-byte segment of a row
constexpr int PTI_GBLK = 3;      // outputs a thread accumulates together (15 64-bit accumulators)
constexpr int PTI_FLUSH = 16;    // products per accumulator before it is folded: 16 * 2^60 = 2^64

// acc += a * b, one IMAD.WIDE (written as PTX: nvcc's u32 -> u64 promotion leaves a dead add on the high word)
DPFHE_HD void mad_wide(u64 &acc, u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(a), "r"(b));
#else
    acc += (u64)a * b;
#endif
}
DPFHE_HD u64 pti_split(u64 x) { return (x & 0x3fffffffull) | ((x >> 30) << 32); }   // low / high 30-bit halves in the two words

DPFHE_HD void st_stream64(u64 *p, u64 v) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
    *p = v;
#endif
}

// z = a0 + (a1a + a1b) * 2^30 + a2 * 2^60 < 16 q^2  ->  [0, 3q)   (barrett_lazy's own bound is z < 2^(s+64) ~ 4 q^2)
DPFHE_HD u64 pti_fold(u64 a0, u64 a1a, u64 a1b, u64 a2, const LimbParams &p) {
    const u64 m = a1a + a1b, mc = m < a1a ? 1ull : 0ull;   // 65-bit middle sum
    u64 lo = a0, hi, t = m << 30;
    lo += t;
    hi = (lo < t ? 1ull : 0ull) + (m >> 34) + (mc << 30);
    t = a2 << 60;
    lo += t;
    hi += (lo < t ? 1ull : 0ull) + (a2 >> 4);
    return word_reduce(barrett_lazy_long(hi, lo, p), p);
}

// shared memory: (gcnt * nb + 4 * nb) * 16 words (plaintext tile + two ciphertext-row buffers)
template <int LOGN, int NT, class CTA>
DPFHE_HD void pt_inner_tile(CTA &cta, u64 *smem, const PtInnerArgs &A, const LimbParams &p, u32 limb, u32 tile, u32 g0, u32 gcnt) {
    constexpr size_t N = (size_t)1 << LOGN;
    constexpr int NW = NT / 32;
    static_assert(PTI_COEFFS == 16 && NT % 32 == 0, "a half-warp covers one tile row");
    const size_t P = (size_t)A.L * N, col = (size_t)limb * N + (size_t)tile * PTI_COEFFS;
    const u32 nb = A.nb;
    u64 *ps = smem;                                       // [gcnt][nb][16] split plaintext values
    u64 *xs = smem + (size_t)gcnt * nb * PTI_COEFFS;      // 2 x [nb][2][16] split ciphertext values (double buffer)
    cta.par([&](int tid) {
        for (u32 idx = (u32)tid; idx < gcnt * nb * 8; idx += NT) {
            const u32 r = idx >> 3, ch = idx & 7, g = r / nb, b = r % nb;
            const U64x2 v = ld_keep(reinterpret_cast<const U64x2 *>(A.pts + ((size_t)(g0 + g) * nb + b) * P + col) + ch);
            ps[r * 16 + ch * 2] = pti_split(v.x);
            ps[r * 16 + ch * 2 + 1] = pti_split(v.y);
        }
    });
    // x rows of batch element k -> split halves in buffer xs + (k & 1) * nb * 32; a thread moves chunks tid, tid + NT, ...
    auto x_src = [&](size_t k, u32 idx) {
        const u32 r = idx >> 3, ch = idx & 7, b = r >> 1, comp = r & 1;
        return reinterpret_cast<const U64x2 *>(A.steps + (((size_t)b * A.batch + k) * 2 + comp) * P + col) + ch;
    };
    const u32 n_chunks = nb * 2 * 8;
    cta.par([&](int tid) {
        for (u32 idx = (u32)tid; idx < n_chunks; idx += NT) {
            const U64x2 v = ld_stream(x_src(0, idx));
            xs[idx * 2] = pti_split(v.x);
            xs[idx * 2 + 1] = pti_split(v.y);
        }
    });
    for (size_t k = 0; k < A.batch; ++k) {
        const u64 *xcur = xs + (k & 1) * (size_t)nb * 32;
        u64 *xnext = xs + ((k + 1) & 1) * (size_t)nb * 32;
        cta.par([&](int tid) {
            const u32 lane = (u32)tid & 31u, c = lane & 15u, comp = lane >> 4, w = (u32)tid >> 5;
            // the next batch element's rows are requested before this one's arithmetic and parked in the other buffer
            // after it: one barrier per batch element, global latency hidden behind the multiply-accumulates
            constexpr int PF = 4;   // 16-byte chunks a thread keeps in flight: covers nb <= 64; larger nb loads after the arithmetic
            U64x2 nx[PF];
            const bool more = k + 1 < A.batch, fits = n_chunks <= (u32)NT * PF;
            if (more && fits) {
#pragma unroll
                for (int u = 0; u < PF; ++u)
                    if ((u32)tid + (u32)u * NT < n_chunks) nx[u] = ld_stream(x_src(k + 1, (u32)tid + (u32)u * NT));
            }
            const u64 *xrow = xcur + comp * 16 + c;   // + b * 32
            for (u32 gb = w; gb < gcnt; gb += NW * PTI_GBLK) {   // this thread's outputs: g = gb + j * NW (warp-uniform)
                // rows past the end of the block are computed on a clamped index and not stored: no branches in the loop
                const u64 *prow[PTI_GBLK];
                u64 a0[PTI_GBLK], a1a[PTI_GBLK], a1b[PTI_GBLK], a2[PTI_GBLK], sum[PTI_GBLK];
#pragma unroll
                for (int j = 0; j < PTI_GBLK; ++j) {
                    const u32 g = gb + (u32)j * NW;
                    prow[j] = ps + (size_t)(g < gcnt ? g : gcnt - 1) * nb * 16 + c;   // + b * 16
                    a0[j] = a1a[j] = a1b[j] = a2[j] = sum[j] = 0;
                }
                for (u32 b0 = 0; b0 < nb; b0 += PTI_FLUSH) {
                    const u32 b1 = b0 + PTI_FLUSH < nb ? b0 + PTI_FLUSH : nb;
                    auto step = [&](u32 b) {
                        const u64 xv = xrow[b * 32];
                        const u32 x0 = (u32)xv, x1 = (u32)(xv >> 32);
#pragma unroll
                        for (int j = 0; j < PTI_GBLK; ++j) {
                            const u64 pv = prow[j][b * 16];
                            const u32 p0 = (u32)pv, p1 = (u32)(pv >> 32);
                            mad_wide(a0[j], x0, p0);
                            mad_wide(a1a[j], x0, p1);
                            mad_wide(a1b[j], x1, p0);
                            mad_wide(a2[j], x1, p1);
                        }
                    };
                    // ptxas lowers the accumulation to IMAD.WIDE (no addend) + one three-input IADD3 / IADD3.X pair per two
                    // products; it does not keep a loop-carried 64-bit addend in the multiplier in any formulation tried.
                    if (b1 - b0 == PTI_FLUSH) {
#pragma unroll
                        for (u32 u = 0; u < PTI_FLUSH; ++u) step(b0 + u);   // full group: shared-memory offsets become immediates
                    } else {
#pragma unroll 4
                        for (u32 b = b0; b < b1; ++b) step(b);
                    }
#pragma unroll
                    for (int j = 0; j < PTI_GBLK; ++j) {
                        sum[j] = csub(sum[j] + pti_fold(a0[j], a1a[j], a1b[j], a2[j], p), p.q4);   // stays below 4q
                        a0[j] = a1a[j] = a1b[j] = a2[j] = 0;
                    }
                }
#pragma unroll
                for (int j = 0; j < PTI_GBLK; ++j) {
                    const u32 g = gb + (u32)j * NW;
                    if (g < gcnt) st_stream64(A.out + (((size_t)(g0 + g) * A.batch + k) * 2 + comp) * P + col + c, canon4(sum[j], p));
                }
            }
            if (more) {
                if (fits) {
#pragma unroll
                    for (int u = 0; u < PF; ++u) {
                        const u32 idx = (u32)tid + (u32)u * NT;
                        if (idx < n_chunks) {
                            xnext[idx * 2] = pti_split(nx[u].x);
                            xnext[idx * 2 + 1] = pti_split(nx[u].y);
                        }
                    }
                } else {
                    for (u32 idx = (u32)tid; idx < n_chunks; idx += NT) {
                        const U64x2 v = ld_stream(x_src(k + 1, idx));
                        xnext[idx * 2] = pti_split(v.x);
                        xnext[idx * 2 + 1] = pti_split(v.y);
                    }
                }
            }
        });
    }
}

// ---- CKKS slot encoding (DESIGN.md §2.12) ------------------------------------------------------------------------
// Floating point with one fixed operation order: every product and sum is rounded on its own.  nvcc never contracts the
// __d*_rn intrinsics into FMAs; host builds of these bodies (tests/emu) compile with -ffp-contract=off.
DPFHE_HD double f_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
DPFHE_HD double f_sub(double a, double b) { return f_add(a, -b); }
DPFHE_HD double f_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
DPFHE_HD double f_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
DPFHE_HD double f_rint(double a) {   // nearest integer, ties to even
#if defined(__CUDA_ARCH__)
    return rint(a);
#else
    return __builtin_rint(a);
#endif
}
DPFHE_HD double f_from_u64(u64 a) {
#if defined(__CUDA_ARCH__)
    return __ull2double_rn(a);
#else
    return (double)a;
#endif
}
DPFHE_HD u64 f_bits(double a) {
#if defined(__CUDA_ARCH__)
    return (u64)__double_as_longlong(a);
#else
    u64 b;
    __builtin_memcpy(&b, &a, 8);
    return b;
#endif
}
// (ar br - ai bi, ar bi + ai br)
DPFHE_HD Cplx c_mul(const Cplx &a, const Cplx &b) {
    return Cplx{f_sub(f_mul(a.re, b.re), f_mul(a.im, b.im)), f_add(f_mul(a.re, b.im), f_mul(a.im, b.re))};
}
DPFHE_HD Cplx c_conj(const Cplx &a) { return Cplx{a.re, -a.im}; }

// Radix-2 decimation in time over S = N/2 points in bit-reversed order: Y[t] = sum_k a[k] W^(+-tk), W = exp(2 pi i / S) = tw[4].
// The twiddle of butterfly j at stage s (span h = 2^s) is W^(j S / 2h) = tw[j N / h]; `inverse` conjugates it.
template <int LOGN, int NT, class CTA>
DPFHE_HD void ckks_fft_stages(CTA &cta, Cplx *a, const Cplx *tw, bool inverse) {
    constexpr int S = 1 << (LOGN - 1);
#pragma unroll 1
    for (int s = 0; s < LOGN - 1; ++s) {
        cta.par([&](int tid) {
#pragma unroll 1
            for (int b = tid; b < S / 2; b += NT) {
                const int j = b & ((1 << s) - 1), i0 = ((b >> s) << (s + 1)) + j, i1 = i0 + (1 << s);
                Cplx w = tw[j << (LOGN - s)];
                if (inverse) w = c_conj(w);
                const Cplx x = a[i0], y = c_mul(a[i1], w);
                a[i0] = Cplx{f_add(x.re, y.re), f_add(x.im, y.im)};
                a[i1] = Cplx{f_sub(x.re, y.re), f_sub(x.im, y.im)};
            }
        });
    }
}

// encode, one vector: z [N/2] slots -> x [N] rounded coefficients rint(sc * m_k), sc = scale * 2/N.  a: N/2 complex of
// shared memory.
template <int LOGN, int NT, class CTA>
DPFHE_HD void ckks_enc_fft_body(CTA &cta, Cplx *a, const Cplx *z, double *x, const Cplx *tw, const u32 *tj, double sc) {
    constexpr int S = 1 << (LOGN - 1);
    cta.par([&](int tid) {
        for (int j = tid; j < S; j += NT) a[bitrev_n(tj[j], LOGN - 1)] = z[j];
    });
    ckks_fft_stages<LOGN, NT>(cta, a, tw, true);
    cta.par([&](int tid) {
        for (int k = tid; k < S; k += NT) {
            const Cplx u = c_mul(a[k], c_conj(tw[k]));
            x[k] = f_rint(f_mul(sc, u.re));
            x[k + S] = f_rint(f_mul(sc, u.im));
        }
    });
}

// the exact residue of an integral double x modulo q_l: x = +-M 2^e, M < 2^53, so x mod q = +-(M mod q)(2^e mod q).
// pow2: the limb's 2^e mod q table.  Non-finite values give some residue (the table index stays in range).
DPFHE_HD u64 ckks_reduce(double x, const LimbParams &p, const u64 *pow2) {
    const u64 b = f_bits(x);
    const int ex = (int)((b >> 52) & 0x7ff);
    const u64 m = (b & ((1ull << 52) - 1)) | (ex ? 1ull << 52 : 0);
    const int e = (ex ? ex : 1) - 1075;
    const u64 v = e >= 0 ? m : (e > -64 ? m >> -e : 0);
    const int pe = e < 0 ? 0 : (e < CKKS_POW2_E ? e : CKKS_POW2_E - 1);
    const u64 r = mulmod(canon(v, p), pow2[pe], p);
    return (b >> 63) && r ? p.q - r : r;
}

// Garner, shared by the CKKS and BGV decoders: the residues col[l * stride], l < L (canonical), are overwritten by the
// mixed-radix digits of X = d_0 + d_1 q_0 + d_2 q_0 q_1 + ...; returns X > (Q-1)/2 (the digits of (Q-1)/2 in `half`, compared
// lexicographically from the most significant one)
DPFHE_HD bool garner_digits(u64 *col, size_t stride, u32 L, const LimbParams *lp, const u64 (&ginv)[16][16], const u64 *half) {
#pragma unroll 1
    for (u32 i = 1; i < L; ++i) {
        const LimbParams &p = lp[i];
        u64 t = col[i * stride];
#pragma unroll 1
        for (u32 j = 0; j < i; ++j) {
            const u64 d = canon(col[j * stride], p);
            t = mulmod(t >= d ? t - d : t + p.q - d, ginv[j][i], p);
        }
        col[i * stride] = t;
    }
    int cmp = 0;
#pragma unroll 1
    for (u32 i = L; i-- > 0 && cmp == 0;) {
        const u64 d = col[i * stride];
        cmp = d > half[i] ? 1 : (d < half[i] ? -1 : 0);
    }
    return cmp > 0;
}

// decode, one coefficient: the residues col[l * stride], l < L (canonical), are overwritten by the mixed-radix digits of X
// (Garner); returns centred(X) / scale as a double: Horner from the most significant digit, then one division.
DPFHE_HD double ckks_crt_double(u64 *col, size_t stride, u32 L, const LimbParams *lp, const CkksConsts &K) {
    const bool neg = garner_digits(col, stride, L, lp, K.ginv, K.half);
    // digits of Q - X: 0 below the lowest non-zero digit p of X, q_p - d_p at p, q_i - 1 - d_i above
    u32 low = 0;
    if (neg)
        while (col[low * stride] == 0) ++low;
    double r = 0.0;
#pragma unroll 1
    for (u32 i = L; i-- > 0;) {
        const u64 d = col[i * stride], q = lp[i].q;
        const u64 f = !neg ? d : (i > low ? q - 1 - d : (i == low ? q - d : 0));
        r = i == L - 1 ? f_from_u64(f) : f_add(f_mul(r, K.qd[i]), f_from_u64(f));
    }
    return f_div(neg ? -r : r, K.scale);
}

// decode, one vector: col [L][N] coefficients (inverse-transformed, canonical; overwritten) -> z [N/2] slots
template <int LOGN, int NT, class CTA>
DPFHE_HD void ckks_dec_fft_body(CTA &cta, Cplx *a, u64 *col, Cplx *z, const Cplx *tw, const u32 *tj, const LimbParams *lp, const CkksConsts &K,
                                u32 L) {
    constexpr int S = 1 << (LOGN - 1);
    constexpr size_t N = (size_t)1 << LOGN;
    cta.par([&](int tid) {
        for (int k = tid; k < S; k += NT) {
            const Cplx u{ckks_crt_double(col + k, N, L, lp, K), ckks_crt_double(col + k + S, N, L, lp, K)};
            a[bitrev_n((u32)k, LOGN - 1)] = c_mul(u, tw[k]);
        }
    });
    ckks_fft_stages<LOGN, NT>(cta, a, tw, false);
    cta.par([&](int tid) {
        for (int j = tid; j < S; j += NT) z[j] = a[tj[j]];
    });
}

// ---- BGV slot encoding (DESIGN.md §2.13) ---------------------------------------------------------------------------
// The negacyclic transform of N values mod t (32-bit arithmetic) in shared memory, radix-2 stages with CTA barriers and the
// conventions of §2.3 with psi = zeta: stage s has 2^s groups of span N / 2^(s+1), the twiddle of group i is tw[2^s + i].
// Forward: Cooley-Tukey, natural in, bit-reversed out, a[i] -> m(zeta^(2 br(i) + 1)).  Inverse: Gentleman-Sande, bit-reversed
// in, natural out, WITHOUT the factor N^-1.  Every value stays canonical, so the result is an exact integer.
template <int LOGN, int NT, class CTA>
DPFHE_HD void bgv_ntt_stages(CTA &cta, u32 *a, const u32 *tw, u32 t, bool inverse) {
    constexpr int N = 1 << LOGN;
#pragma unroll 1
    for (int k = 0; k < LOGN; ++k) {
        const int s = inverse ? LOGN - 1 - k : k, hs = LOGN - 1 - s;   // 2^s groups of span 2^hs
        const u32 *w = tw + (inverse ? 2 * N : 0), *ws = w + N;
        cta.par([&](int tid) {
#pragma unroll 1
            for (int b = tid; b < N / 2; b += NT) {
                const int g = (1 << s) + (b >> hs), i0 = ((b >> hs) << (hs + 1)) + (b & ((1 << hs) - 1)), i1 = i0 + (1 << hs);
                const u32 x = a[i0], y = a[i1];
                if (!inverse) {
                    const u32 v = shoup32(y, w[g], ws[g], t);
                    a[i0] = add32(x, v, t);
                    a[i1] = sub32(x, v, t);
                } else {
                    a[i0] = add32(x, y, t);
                    a[i1] = shoup32(x + t - y, w[g], ws[g], t);   // x + t - y < 2t < 2^32: shoup32 takes any 32-bit word
                }
            }
        });
    }
}

// floor-mod of any int64 by t (numpy's %).  INT64_MIN included: the magnitude 0 - (u64)v of a negative v is exact.
DPFHE_HD u32 bgv_reduce_slot(int64_t v, const Mod32 &m) {
    if (v >= 0) return reduce64_32((u64)v, m);
    const u32 r = reduce64_32(0 - (u64)v, m);
    return r ? m.t - r : 0u;
}

// the centred lift of a coefficient c in [0, t) into a limb: c <= floor(t/2) stays, above it is c - t, i.e. q - (t - c)
DPFHE_HD u64 bgv_lift(u32 c, u32 t, const LimbParams &p) { return c > (t >> 1) ? p.q - (t - c) : (u64)c; }

// encode, one vector: z [2][N/2] slots -> x [N] coefficients in [0, t).  a: N words of shared memory.
template <int LOGN, int NT, class CTA>
DPFHE_HD void bgv_enc_body(CTA &cta, u32 *a, const int64_t *z, u32 *x, const BgvTables &T) {
    constexpr int N = 1 << LOGN;
    cta.par([&](int tid) {
        for (int j = tid; j < N; j += NT) a[T.pos[j]] = bgv_reduce_slot(z[j], T.m);
    });
    bgv_ntt_stages<LOGN, NT>(cta, a, T.tw, T.m.t, true);
    cta.par([&](int tid) {
        for (int k = tid; k < N; k += NT) x[k] = shoup32(a[k], T.ninv, T.ninv_s, T.m.t);
    });
}

// decode, one coefficient: Garner digits of X (written over the residues col[l * stride]), then centred(X) mod t by Horner from
// the most significant digit, r = r (q_i mod t) + (d_i mod t), minus Q mod t when X > (Q-1)/2
DPFHE_HD u32 bgv_crt_mod_t(u64 *col, size_t stride, u32 L, const LimbParams *lp, const BgvConsts &K) {
    const bool neg = garner_digits(col, stride, L, lp, K.ginv, K.half);
    const u32 t = K.m.t;
    u32 r = reduce64_32(col[(L - 1) * stride], K.m);
#pragma unroll 1
    for (u32 i = L - 1; i-- > 0;) r = add32(shoup32(r, K.qt[i], K.qt_s[i], t), reduce64_32(col[i * stride], K.m), t);
    return neg ? sub32(r, K.Qt, t) : r;
}

// decode, one vector: col [L][N] coefficients (inverse-transformed, canonical; overwritten) -> z [2][N/2] slots in [0, t)
template <int LOGN, int NT, class CTA>
DPFHE_HD void bgv_dec_body(CTA &cta, u32 *a, u64 *col, u64 *z, const BgvTables &T, const LimbParams *lp, const BgvConsts &K, u32 L) {
    constexpr int N = 1 << LOGN;
    cta.par([&](int tid) {
        for (int k = tid; k < N; k += NT) a[k] = bgv_crt_mod_t(col + k, N, L, lp, K);
    });
    bgv_ntt_stages<LOGN, NT>(cta, a, T.tw, T.m.t, false);
    cta.par([&](int tid) {
        for (int j = tid; j < N; j += NT) z[j] = a[T.pos[j]];
    });
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
