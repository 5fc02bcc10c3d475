// ntt_core.cuh — the in-shared-memory negacyclic NTT of one limb (DESIGN.md §4.2).
//
// A limb of N = 2^LOGN coefficients lives in shared memory in the TMA SWIZZLE_128B
// layout (16-byte chunk index XOR row index mod 8, rows of 128 B = 16 coefficients), so
// that every access pattern below is bank-conflict free:
//   - "column" accesses (32 lanes -> 32 consecutive coefficients, 8 B each),
//   - "row" accesses (each lane owns one whole 128-B row, 16 B at a time).
//
// The transform is split as  [K = LOGN-12 outer stages, fused into the global load/store]
//                          + [three radix-16 register passes A, B, C over shared memory].
// Forward = Cooley-Tukey butterflies, natural -> bit-reversed order, twist merged (Harvey);
// inverse = Gentleman-Sande, bit-reversed -> natural, N^-1 folded into the last stage.
//
// All functions are __host__ __device__: tests/emu runs the identical code on the CPU
// thread-by-thread to check the index algebra against the oracle (test infrastructure only).
#pragma once
#include "modarith.cuh"

namespace dpfhe {
namespace DPFHE_VNS {

// ---- shared-memory layout -------------------------------------------------------------
// coefficient index -> u64 slot (TMA SWIZZLE_128B: chunk ^= row & 7)
DPFHE_HD int swz(int idx) { return idx ^ (((idx >> 4) & 7) << 1); }
// 16-byte chunk index (two coefficients) -> chunk slot
DPFHE_HD int swz_chunk(int cg) { return cg ^ ((cg >> 3) & 7); }

// twiddle table layout: tw_pos<LOGN>(stage, group) in types.hpp

// ---- butterflies -----------------------------------------------------------------------
// forward, fully lazy: x' = x + w*y, y' = x - w*y + SB*q; bound grows by SB per stage (SB*q: bound of shoup_lazy).
DPFHE_HD void ct_bfly(u64 &x, u64 &y, const Twiddle &w, const LimbParams &p) {
    u64 t = shoup_lazy_cc(y, w.x, w.y, p);
    u64 a = x;
    x = a + t;
    y = a + p.qsb - t;
}
// inverse, Harvey: inputs and outputs in [0, SB*q)
DPFHE_HD void gs_bfly(u64 &x, u64 &y, const Twiddle &w, const LimbParams &p) {
    u64 a = x, b = y;
    x = csub(a + b, p.qsb);
    y = shoup_lazy(a + p.qsb - b, w.x, w.y, p);
}

// ---- lazy-bound schedule of the forward transform ------------------------------------------
// Values are tracked as "< B*q".  A forward stage maps X-inputs below B*q to outputs below
// (B+SB)*q (shoup_lazy yields < SB*q for any 64-bit input).  16*q < 2^64, so when B + SB would
// exceed 16 the X inputs of that stage first take one conditional subtraction of 8q
// (B <= 16 -> 8).  Everything is resolved at compile time from the bound at entry.
DPFHE_HD constexpr bool fwd_needs_csub(int bin, int stage) {
    int b = bin;
    for (int s = 0; s < stage; ++s) b = (b + SB > 16 ? 8 : b) + SB;
    return b + SB > 16;
}
DPFHE_HD constexpr int fwd_bound_after(int bin, int stages) {
    int b = bin;
    for (int s = 0; s < stages; ++s) b = (b + SB > 16 ? 8 : b) + SB;
    return b;
}
// fwd_needs_csub(bin, u) for u < 4 as bit u.  Kernels take the schedule from a constexpr mask: called per butterfly inside an
// unrolled pass, fwd_needs_csub is left as a runtime loop (one per butterfly of stages 2 and 3) that selects the subtraction
// at run time and cuts the pass into basic blocks the scheduler cannot interleave.
DPFHE_HD constexpr unsigned fwd_csub_mask16(int bin) {
    unsigned m = 0;
    for (int u = 0; u < 4; ++u) m |= fwd_needs_csub(bin, u) ? 1u << u : 0u;
    return m;
}

// 16-point register kernels.  `x[k]` holds element k of a radix-16 group; stage u pairs
// k with k + (8 >> u).  tw(u, j) returns the twiddle of sub-group j at local stage u.
template <int BIN, class TW>
DPFHE_HD void fwd16(u64 (&x)[16], const LimbParams &p, TW tw) {
    // constant trip counts, as in inv16 below
    constexpr unsigned CSUB = fwd_csub_mask16(BIN);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int half = 8 >> u;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < (1 << u)) {
                const Twiddle w = tw(u, j);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    if (i < half) {
                        if ((CSUB >> u) & 1u) x[j * 2 * half + i] = csub(x[j * 2 * half + i], p.q8);
                        ct_bfly(x[j * 2 * half + i], x[j * 2 * half + half + i], w, p);
                    }
                }
            }
        }
    }
}
template <class TW>
DPFHE_HD void inv16(u64 (&x)[16], const LimbParams &p, TW tw) {
    // Every loop has a constant trip count and the stage-dependent bounds are conditions that fold once all loops are
    // unrolled: with trip counts that depend on u, the compute_90a front end leaves inner loops rolled, indexes x[]
    // dynamically and moves it to local memory.
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const int u = 3 - s;
        const int half = 8 >> u;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < (1 << u)) {
                const Twiddle w = tw(u, j);
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (i < half) gs_bfly(x[j * 2 * half + i], x[j * 2 * half + half + i], w, p);
            }
        }
    }
}

// ---- register passes over shared memory ----------------------------------------------
// A pass covers stages [S0, S0+4).  Group p in [0, N/16) splits as (hi, lo) with
// lo = p mod 2^NLO, NLO = LOGN-S0-4; its 16 elements are idx = hi*2^(LOGN-S0) + k*2^NLO + lo.
// Thread `tid` of NT handles groups p = tid + g*NT.
// BIN: lazy bound (in units of q) of the values at entry; the pass leaves fwd_bound_after(BIN, 4).

// BLKS / blk0: the buffer holds BLKS consecutive 4096-coefficient blocks of the limb starting at block blk0
// (the whole limb when BLKS = 2^K, blk0 = 0).  Every pass with S0 >= K stays inside one block, so twiddles use
// the global group index while shared-memory indices are relative to the first resident block.
template <int LOGN, int S0, int NT, int BIN, int BLKS>
DPFHE_HD void fwd_pass(u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, int blk0) {
    constexpr int NLO = LOGN - S0 - 4;
    constexpr int NGROUPS = BLKS * 256;
    static_assert(NLO == 0 || NLO >= 4, "pass split must keep column accesses row-aligned");
    static_assert(S0 >= LOGN - 12, "register passes operate inside 4096-coefficient blocks");
#pragma unroll 1
    for (int lg = tid; lg < NGROUPS; lg += NT) {
        const int g = (blk0 << 8) + lg;
        const int lo = g & ((1 << NLO) - 1), hi = g >> NLO;
        const int base = (hi << (LOGN - S0)) + lo - (blk0 << 12);
        u64 x[16];
        if (NLO == 0) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                U64x2 v = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lg * 8 + c)];
                x[2 * c] = v.x;
                x[2 * c + 1] = v.y;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) x[k] = buf[swz(base + (k << NLO))];
        }
        fwd16<BIN>(x, p, [&](int u, int j) { return tw[tw_pos<LOGN>(S0 + u, (hi << u) + j)]; });
        if (NLO == 0) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                U64x2 v;
                v.x = x[2 * c];
                v.y = x[2 * c + 1];
                reinterpret_cast<U64x2 *>(buf)[swz_chunk(lg * 8 + c)] = v;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) buf[swz(base + (k << NLO))] = x[k];
        }
    }
}

template <int LOGN, int S0, int NT, int BLKS>
DPFHE_HD void inv_pass(u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, int blk0) {
    constexpr int NLO = LOGN - S0 - 4;
    constexpr int NGROUPS = BLKS * 256;
    static_assert(NLO == 0 || NLO >= 4, "pass split must keep column accesses row-aligned");
    static_assert(S0 >= LOGN - 12, "register passes operate inside 4096-coefficient blocks");
#pragma unroll 1
    for (int lg = tid; lg < NGROUPS; lg += NT) {
        const int g = (blk0 << 8) + lg;
        const int lo = g & ((1 << NLO) - 1), hi = g >> NLO;
        const int base = (hi << (LOGN - S0)) + lo - (blk0 << 12);
        u64 x[16];
        if (NLO == 0) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                U64x2 v = reinterpret_cast<const U64x2 *>(buf)[swz_chunk(lg * 8 + c)];
                x[2 * c] = v.x;
                x[2 * c + 1] = v.y;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) x[k] = buf[swz(base + (k << NLO))];
        }
        inv16(x, p, [&](int u, int j) { return tw[tw_pos<LOGN>(S0 + u, (hi << u) + j)]; });
        if (NLO == 0) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                U64x2 v;
                v.x = x[2 * c];
                v.y = x[2 * c + 1];
                reinterpret_cast<U64x2 *>(buf)[swz_chunk(lg * 8 + c)] = v;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) buf[swz(base + (k << NLO))] = x[k];
        }
    }
}

// ---- outer stages fused with the global <-> shared copies -----------------------------
// K = LOGN-12 outer stages (radix 2^K across the limb).  Work item c in [0, N/2/2^K) names a
// 16-byte chunk column: coefficients n = 2c, 2c+1 of each of the 2^K blocks of size N/2^K.

// SRC(chunk_index) -> U64x2 loads the 16-byte chunk `chunk_index` of the source limb.
// IN_REDUCE: the source is not canonical for this modulus (key-switch digit lift): word_reduce it.
template <int LOGN, int NT, bool IN_REDUCE, class SRC>
DPFHE_HD void fwd_load_stage(u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, SRC src) {
    constexpr int K = LOGN - 12;
    constexpr int NB = 1 << K;                  // blocks
    constexpr int CPB = (1 << (LOGN - 1)) / NB; // chunks per block
    U64x2 nxt[NB];   // loads of the next iteration are issued before this iteration's butterflies
#pragma unroll
    for (int b = 0; b < NB; ++b) nxt[b] = src(b * CPB + tid);
#pragma unroll 1
    for (int c = tid; c < CPB; c += NT) {
        u64 x[NB][2];
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const U64x2 v = nxt[b];
            x[b][0] = IN_REDUCE ? word_reduce(v.x, p) : v.x;
            x[b][1] = IN_REDUCE ? word_reduce(v.y, p) : v.y;
        }
        if (c + NT < CPB) {
#pragma unroll
            for (int b = 0; b < NB; ++b) nxt[b] = src(b * CPB + c + NT);
        }
        // entry bound is at most 4; K <= 2 stages never need a csub (static_assert in fwd_passes_blk)
#pragma unroll
        for (int u = 0; u < K; ++u) {
            const int half = NB >> (u + 1);
#pragma unroll
            for (int j = 0; j < (1 << u); ++j) {
                const Twiddle w = tw[tw_pos<LOGN>(u, j)];
#pragma unroll
                for (int i = 0; i < half; ++i) {
                    ct_bfly(x[j * 2 * half + i][0], x[j * 2 * half + half + i][0], w, p);
                    ct_bfly(x[j * 2 * half + i][1], x[j * 2 * half + half + i][1], w, p);
                }
            }
        }
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            U64x2 v;
            v.x = x[b][0];
            v.y = x[b][1];
            reinterpret_cast<U64x2 *>(buf)[swz_chunk(b * CPB + c)] = v;
        }
    }
}

// canonical product of the last inverse stage: exact quotient + one conditional subtraction.  -DDPFHE_INV_FINAL_LAZY=1 selects the
// quotient estimate (one IMAD.WIDE less) + two conditional subtractions; measured slower (15.72 -> 15.37 M NTT/s, DESIGN.md §6 table)
#ifndef DPFHE_INV_FINAL_LAZY
#define DPFHE_INV_FINAL_LAZY 0
#endif
DPFHE_HD u64 inv_final_product(u64 x, u64 w, u64 ws, const LimbParams &p) {
#if DPFHE_INV_FINAL_LAZY && DPFHE_SHOUP_APPROX
    return canon4(shoup_lazy(x, w, ws, p), p);   // < SB*q = 4q  ->  [0, q)
#else
    return csub(shoup_exact(x, w, ws, p), p.q);
#endif
}

// Inverse counterpart: SRC(chunk_index) yields the chunks left by the register passes (values in [0,SB*q));
// applies the K outermost Gentleman-Sande stages with N^-1 folded into the very last one, and hands
// canonical chunks to DST(chunk_index, U64x2) (the last stage uses the exact product so that one csub finishes).
// [c_lo, c_hi): the chunk columns this call handles (all of them by default; a CTA pair splits them, ntt_inv_half_outer).
template <int LOGN, int NT, class SRC, class DST>
DPFHE_HD void inv_outer_stage(const Twiddle *__restrict__ tw, const LimbParams &p, int tid, SRC src, DST dst, int c_lo = 0,
                              int c_hi = (1 << (LOGN - 1)) >> (LOGN - 12)) {
    constexpr int K = LOGN - 12;
    constexpr int NB = 1 << K;
    constexpr int CPB = (1 << (LOGN - 1)) / NB;
#pragma unroll 1
    for (int c = c_lo + tid; c < c_hi; c += NT) {
        u64 x[NB][2];
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            U64x2 v = src(b * CPB + c);
            x[b][0] = v.x;
            x[b][1] = v.y;
        }
#pragma unroll
        for (int u = K - 1; u >= 1; --u) {
            const int half = NB >> (u + 1);
#pragma unroll
            for (int j = 0; j < (1 << u); ++j) {
                const Twiddle w = tw[tw_pos<LOGN>(u, j)];
#pragma unroll
                for (int i = 0; i < half; ++i) {
                    gs_bfly(x[j * 2 * half + i][0], x[j * 2 * half + half + i][0], w, p);
                    gs_bfly(x[j * 2 * half + i][1], x[j * 2 * half + half + i][1], w, p);
                }
            }
        }
        if (K >= 1) {
            // stage 0: x' = (x + y) * N^-1, y' = (x - y) * (w * N^-1)
#pragma unroll
            for (int i = 0; i < NB / 2; ++i) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    u64 a = x[i][e], b = x[NB / 2 + i][e];
                    x[i][e] = inv_final_product(a + b, p.ninv, p.ninv_s, p);
                    x[NB / 2 + i][e] = inv_final_product(a + p.qsb - b, p.wninv, p.wninv_s, p);
                }
            }
        } else {
#pragma unroll
            for (int e = 0; e < 2; ++e) x[0][e] = inv_final_product(x[0][e], p.ninv, p.ninv_s, p);
        }
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            U64x2 v;
            v.x = x[b][0];
            v.y = x[b][1];
            dst(b * CPB + c, v);
        }
    }
}

template <int LOGN, int NT, class DST>
DPFHE_HD void inv_store_stage(const u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, DST dst) {
    inv_outer_stage<LOGN, NT>(tw, p, tid, [&](int c) { return reinterpret_cast<const U64x2 *>(buf)[swz_chunk(c)]; }, dst);
}

// Half-limb variant of fwd_load_stage for N = 16384 (K = 2, four blocks): reads all four input blocks but keeps
// only the two output blocks {2h, 2h+1} of the outer radix-4 step (3 multiplications per column instead of 4),
// so the register passes run on 64 KiB of shared memory and three CTAs fit an SM.
template <int LOGN, int NT, bool IN_REDUCE, class SRC>
DPFHE_HD void fwd_load_stage_half(u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, SRC src, int h) {
    static_assert(LOGN == 14, "the half-limb load stage is written for K = 2");
    constexpr int CPB = 1 << (LOGN - 3);   // chunks per block: (N/2) / 4
    const Twiddle w0 = tw[tw_pos<LOGN>(0, 0)], w1 = tw[tw_pos<LOGN>(1, h)];
#pragma unroll 1
    for (int c = tid; c < CPB; c += NT) {
        u64 x[4][2];
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const U64x2 v = src(b * CPB + c);
            x[b][0] = IN_REDUCE ? word_reduce(v.x, p) : v.x;
            x[b][1] = IN_REDUCE ? word_reduce(v.y, p) : v.y;
        }
        U64x2 o0, o1;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            // stage 0 pairs (0,2) and (1,3); half 0 keeps the sums, half 1 the differences
            const u64 t02 = shoup_lazy(x[2][e], w0.x, w0.y, p), t13 = shoup_lazy(x[3][e], w0.x, w0.y, p);
            const u64 a = h == 0 ? x[0][e] + t02 : x[0][e] + p.qsb - t02;
            const u64 b = h == 0 ? x[1][e] + t13 : x[1][e] + p.qsb - t13;
            // stage 1 pairs (2h, 2h+1) with the twiddle of group h
            const u64 t = shoup_lazy(b, w1.x, w1.y, p);
            (e == 0 ? o0.x : o0.y) = a + t;
            (e == 0 ? o1.x : o1.y) = a + p.qsb - t;
        }
        reinterpret_cast<U64x2 *>(buf)[swz_chunk(c)] = o0;
        reinterpret_cast<U64x2 *>(buf)[swz_chunk(CPB + c)] = o1;
    }
}

// Block variant of fwd_load_stage (fused key switch at N <= 8192, one 4096-point block per CTA): at N = 8192 (K = 1) it reads
// both input blocks and keeps output block h of the outer radix-2 step (the same products as the whole stage); at N = 4096 the
// block is the limb.
template <int LOGN, int NT, bool IN_REDUCE, class SRC>
DPFHE_HD void fwd_load_stage_blk(u64 *buf, const Twiddle *__restrict__ tw, const LimbParams &p, int tid, SRC src, int h) {
    if constexpr (LOGN == 12) {
        fwd_load_stage<LOGN, NT, IN_REDUCE>(buf, tw, p, tid, src);
    } else {
        static_assert(LOGN == 13, "the block load stage is written for K <= 1");
        constexpr int CPB = 1 << (LOGN - 2);   // chunks per block
        const Twiddle w = tw[tw_pos<LOGN>(0, 0)];
        U64x2 nx = src(tid), ny = src(CPB + tid);   // loads of the next iteration are issued before this iteration's butterflies
#pragma unroll 1
        for (int c = tid; c < CPB; c += NT) {
            const U64x2 vx = nx, vy = ny;
            if (c + NT < CPB) {
                nx = src(c + NT);
                ny = src(CPB + c + NT);
            }
            U64x2 o;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const u64 x = IN_REDUCE ? word_reduce(e ? vx.y : vx.x, p) : (e ? vx.y : vx.x);
                const u64 y = IN_REDUCE ? word_reduce(e ? vy.y : vy.x, p) : (e ? vy.y : vy.x);
                const u64 t = shoup_lazy_cc(y, w.x, w.y, p);
                (e ? o.y : o.x) = h == 0 ? x + t : x + p.qsb - t;
            }
            reinterpret_cast<U64x2 *>(buf)[swz_chunk(c)] = o;
        }
    }
}

// ---- whole-limb drivers --------------------------------------------------------------
// The CTA policy provides three barrier scopes (all of them "run f(tid) for every thread, then sync"):
//   cta.par(f)       whole CTA                     (__syncthreads)
//   cta.par_dom(f)   256-thread domain tid >> 8    (named barrier): after the outer stages the limb is
//                    2^K independent 4096-point blocks and pass A of block b only involves the threads
//                    g >> 8 == b (mod NT/256), so the two halves of a 512-thread CTA run decoupled;
//   cta.par_warp(f)  one warp                      (__syncwarp): passes B and C of a 256-coefficient
//                    sub-block touch only the 16 groups g with equal g >> 4, i.e. 16 lanes of one warp.
// The host emulator runs every segment for all threads in order, whatever the scope.

// forward: buf already holds the output of fwd_load_stage, whose inputs were below BIN*q
// (BIN = 1 canonical, 3 word-reduced).  Returns with values below fwd_out_bound<LOGN,BIN>()*q <= 16q.
template <int LOGN, int BIN>
DPFHE_HD constexpr int fwd_out_bound() {
    return fwd_bound_after(BIN, LOGN);
}
template <int LOGN, int NT, int BIN, int BLKS, class CTA>
DPFHE_HD void fwd_passes_blk(CTA &cta, u64 *buf, const Twiddle *tw, const LimbParams &p, int blk0) {
    constexpr int K = LOGN - 12;
    constexpr int B0 = fwd_bound_after(BIN, K), B1 = fwd_bound_after(BIN, K + 4), B2 = fwd_bound_after(BIN, K + 8);
    static_assert(BIN + SB * K <= 16, "load stage applies no conditional subtraction");
    static_assert(NT % 32 == 0 && (NT >= 256 ? NT % 256 == 0 : true), "thread count must tile the barrier domains");
    static_assert(BLKS == (1 << K) || NT <= 256, "partial-limb buffers use whole-CTA barriers");
    cta.par_dom([&](int tid) { fwd_pass<LOGN, K, NT, B0, BLKS>(buf, tw, p, tid, blk0); });
    cta.par_warp([&](int tid) { fwd_pass<LOGN, K + 4, NT, B1, BLKS>(buf, tw, p, tid, blk0); });
    cta.par([&](int tid) { fwd_pass<LOGN, K + 8, NT, B2, BLKS>(buf, tw, p, tid, blk0); });
}
template <int LOGN, int NT, int BIN, class CTA>
DPFHE_HD void fwd_passes(CTA &cta, u64 *buf, const Twiddle *tw, const LimbParams &p) {
    fwd_passes_blk<LOGN, NT, BIN, (1 << (LOGN - 12))>(cta, buf, tw, p, 0);
}
// inverse: buf holds [0,SB*q) values in bit-reversed order; afterwards run inv_store_stage / inv_outer_stage
template <int LOGN, int NT, int BLKS, class CTA>
DPFHE_HD void inv_passes_blk(CTA &cta, u64 *buf, const Twiddle *itw, const LimbParams &p, int blk0) {
    constexpr int K = LOGN - 12;
    static_assert(BLKS == (1 << K) || NT <= 256, "partial-limb buffers use whole-CTA barriers");
    cta.par_warp([&](int tid) { inv_pass<LOGN, K + 8, NT, BLKS>(buf, itw, p, tid, blk0); });
    cta.par_dom([&](int tid) { inv_pass<LOGN, K + 4, NT, BLKS>(buf, itw, p, tid, blk0); });
    cta.par([&](int tid) { inv_pass<LOGN, K, NT, BLKS>(buf, itw, p, tid, blk0); });
}
template <int LOGN, int NT, class CTA>
DPFHE_HD void inv_passes(CTA &cta, u64 *buf, const Twiddle *itw, const LimbParams &p) {
    inv_passes_blk<LOGN, NT, (1 << (LOGN - 12))>(cta, buf, itw, p, 0);
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
