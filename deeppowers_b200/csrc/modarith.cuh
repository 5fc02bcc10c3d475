// modarith.cuh — 64-bit modular arithmetic for moduli 2^33 < q < 2^60 (DESIGN.md §2.2, §4.1).
//
// Everything is __host__ __device__ so the same code is exercised by the host emulator
// in tests/emu (test infrastructure; never part of libdpfhe.so's product path).
//
// The functions live in namespace dpfhe::gen or dpfhe::fast (types.hpp: DPFHE_FAST).  In the fast variant every
// modulus is q = qh * 2^32 + 1, so k*q = k + ((k*qh) << 32): subtracting a multiple of q takes one 32-bit multiply-add
// instead of one IMAD.WIDE and two IMAD.  What bounds these kernels is the integer multiplier (IMAD.WIDE issues at a
// fraction of the rate of the other integer instructions), so both variants also use quotient
// ESTIMATES that skip partial products (DPFHE_SHOUP_APPROX): the result stays congruent, only the lazy range widens.
//
// Lazy-range conventions ("bound B" means value < B*q; 16q < 2^64 because q < 2^60), SB = 4 (2 with exact quotients):
//   shoup_lazy(x, w)      any 64-bit x        -> [0, SB*q)
//   shoup_exact(x, w)     any 64-bit x        -> [0, 2q)
//   word_reduce(x)        any 64-bit x        -> [0, 3q)
//   barrett_lazy(a*b)     a*b <= 4 q^2        -> [0, (SB+1) q), [0, SB*q) for canonical factors
//   barrett_lazy_long(z)  z < 2^(2b+4)        -> [0, 15q)  (b = bit length of q; sums of up to 16 products)
//   canon(x)              x < 16q             -> [0, q)
#pragma once
#include "types.hpp"

namespace dpfhe {
namespace DPFHE_VNS {

DPFHE_HD u64 umulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

DPFHE_HD u32 umulhi32(u32 a, u32 b) {
    // high half of a 32x32 wide multiply (IMAD.WIDE, not the much slower IMAD.HI)
    return (u32)(((u64)a * b) >> 32);
}

// 32 x 32 -> 64 product that stays one IMAD.WIDE: opaque to the optimiser, so that the sums built around it keep their shape
DPFHE_HD u64 mul_wide(u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    u64 r;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(r) : "r"(a), "r"(b));
    return r;
#else
    return (u64)a * b;
#endif
}

// hi64(x * y) minus 0, 1 or 2.  Three IMAD.WIDE: the low partial product xl*yl only matters through a carry (<= 1) and
// so does the sum of the low words of the two middle products (<= 1).
DPFHE_HD u64 mulhi_approx(u64 x, u64 y) {
#if DPFHE_SHOUP_APPROX == 0
    return umulhi64(x, y);
#else
    // Written with plain sums on purpose.  Pinning the shape in one asm block (no register-pair moves, 21.7 instead of 21.4
    // instructions per butterfly but fewer of them on the multiplier pipe) was SLOWER, and so was keeping the carry
    // additions off IMAD.X with an opaque third addend: ptxas' own split of the adds and moves between the ALU and the
    // multiplier pipe is the better one when both pipes are close to full.
    const u32 xl = (u32)x, xh = (u32)(x >> 32), yl = (u32)y, yh = (u32)(y >> 32);
    const u64 a = mul_wide(xh, yl), b = mul_wide(xl, yh);
    const u64 m = (u64)(u32)(a >> 32) + (u32)(b >> 32);
    return (u64)xh * yh + m;
#endif
}

// mulhi_approx, the same value, with the middle sum pinned as a 32-bit add with carry that is the addend of the xh*yh
// multiply-add (IADD3, one carry instruction, IMAD.WIDE).  Where a product feeds several sums while its operand stays live (the
// forward butterfly: x + t and x + SB*q - t; the Barrett quotient of the tensor), ptxas folds the plain sums the other way,
// xh*yh + hi(a) through a zero-extended register pair and then + hi(b), which costs two IMAD.MOV on the multiplier pipe per
// product.  The inverse butterfly keeps mulhi_approx: there the plain sums compile to fewer instructions than this block.
DPFHE_HD u64 mulhi_approx_cc(u64 x, u64 y) {
#if DPFHE_SHOUP_APPROX == 0 || !defined(__CUDA_ARCH__)
    return mulhi_approx(x, y);
#else
    const u32 xl = (u32)x, xh = (u32)(x >> 32), yl = (u32)y, yh = (u32)(y >> 32);
    const u64 a = mul_wide(xh, yl), b = mul_wide(xl, yh);
    u64 r;
    asm("{\n\t"
        ".reg .u32 ml, mh;\n\t"
        ".reg .u64 m;\n\t"
        "add.cc.u32 ml, %1, %2;\n\t"
        "addc.u32 mh, 0, 0;\n\t"
        "mov.b64 m, {ml, mh};\n\t"
        "mad.wide.u32 %0, %3, %4, m;\n\t"
        "}"
        : "=l"(r)
        : "r"((u32)(a >> 32)), "r"((u32)(b >> 32)), "r"(xh), "r"(yh));
    return r;
#endif
}

// x >= m ? x - m : x, branch-free.  Correct for every 64-bit x when m <= 2^63.
// Device: subtract with borrow and select on the borrow (IADD3, IADD3.X, 2x SEL).
DPFHE_HD u64 csub(u64 x, u64 m) {
#if defined(__CUDA_ARCH__)
    u32 xl = (u32)x, xh = (u32)(x >> 32), ml = (u32)m, mh = (u32)(m >> 32), tl, th, b;
    asm("sub.cc.u32 %0, %3, %5;\n\tsubc.cc.u32 %1, %4, %6;\n\tsubc.u32 %2, 0, 0;"
        : "=&r"(tl), "=&r"(th), "=&r"(b)
        : "r"(xl), "r"(xh), "r"(ml), "r"(mh));
    const u32 rl = b ? xl : tl, rh = b ? xh : th;
    return ((u64)rh << 32) | rl;
#else
    u64 t = x - m;
    return t < x ? t : x;   // unsigned wrap makes t > x exactly when x < m
#endif
}

// c + a*b mod 2^64 as ONE multiply-add chain (IMAD.WIDE + 2 IMAD, no separate adds)
DPFHE_HD u64 mad_lo64(u64 a, u64 b, u64 c) {
#if defined(__CUDA_ARCH__)
    u64 t;
    asm("{\n\t"
        ".reg .u32 al, ah, bl, bh, t0, t1;\n\t"
        ".reg .u64 T;\n\t"
        "mov.b64 {al, ah}, %1;\n\t"
        "mov.b64 {bl, bh}, %2;\n\t"
        "mad.wide.u32 T, al, bl, %3;\n\t"
        "mov.b64 {t0, t1}, T;\n\t"
        "mad.lo.u32 t1, al, bh, t1;\n\t"
        "mad.lo.u32 t1, ah, bl, t1;\n\t"
        "mov.b64 %0, {t0, t1};\n\t"
        "}"
        : "=l"(t)
        : "l"(a), "l"(b), "l"(c));
    return t;
#else
    return c + a * b;
#endif
}

// x - k*q mod 2^64
DPFHE_HD u64 sub_mul_q(u64 x, u64 k, const LimbParams &p) {
#if DPFHE_FAST
    return x - k + ((u64)((u32)k * p.nqh) << 32);   // k*q = k + ((k*qh) << 32)
#else
    return mad_lo64(k, p.nq, x);
#endif
}

// One-word quotient estimate: k = floor(x_hi * mu32 / 2^32) <= floor(x/q), off by at most 2.
DPFHE_HD u64 word_reduce(u64 x, const LimbParams &p) {
    const u32 k = umulhi32((u32)(x >> 32), p.mu32);
    return sub_mul_q(x, (u64)k, p);   // x - k*q, in [0, 3q)
}

// shoup_tail: low 64 bits of x*w - h*q.
// gen:  one multiply-add chain t = xl*wl + hl*nql (2 IMAD.WIDE), t.hi += xl*wh + xh*wl + hl*nqh + hh*nql (4 IMAD) with
//       nq = 2^64 - q, which avoids the negation and the split adds nvcc otherwise emits.
// fast: the chain is xl*wl (1 IMAD.WIDE), t.hi += xl*wh + xh*wl + hl*(-qh) (3 IMAD), minus h.
DPFHE_HD u64 shoup_tail(u64 x, u64 w, u64 h, const LimbParams &p) {
#if defined(__CUDA_ARCH__)
    u64 t;
#if DPFHE_FAST
    asm("{\n\t"
        ".reg .u32 xl, xh, wl, wh, hl, hh, t0, t1;\n\t"
        ".reg .u64 T;\n\t"
        "mov.b64 {xl, xh}, %1;\n\t"
        "mov.b64 {wl, wh}, %2;\n\t"
        "mov.b64 {hl, hh}, %3;\n\t"
        "mul.wide.u32 T, xl, wl;\n\t"
        "mov.b64 {t0, t1}, T;\n\t"
        "mad.lo.u32 t1, xl, wh, t1;\n\t"
        "mad.lo.u32 t1, xh, wl, t1;\n\t"
        "mad.lo.u32 t1, hl, %4, t1;\n\t"
        "mov.b64 %0, {t0, t1};\n\t"
        "}"
        : "=l"(t)
        : "l"(x), "l"(w), "l"(h), "r"(p.nqh));
    return t - h;
#else
    asm("{\n\t"
        ".reg .u32 xl, xh, wl, wh, hl, hh, nl, nh, t0, t1;\n\t"
        ".reg .u64 T;\n\t"
        "mov.b64 {xl, xh}, %1;\n\t"
        "mov.b64 {wl, wh}, %2;\n\t"
        "mov.b64 {hl, hh}, %3;\n\t"
        "mov.b64 {nl, nh}, %4;\n\t"
        "mul.wide.u32 T, xl, wl;\n\t"
        "mad.wide.u32 T, hl, nl, T;\n\t"
        "mov.b64 {t0, t1}, T;\n\t"
        "mad.lo.u32 t1, xl, wh, t1;\n\t"
        "mad.lo.u32 t1, xh, wl, t1;\n\t"
        "mad.lo.u32 t1, hl, nh, t1;\n\t"
        "mad.lo.u32 t1, hh, nl, t1;\n\t"
        "mov.b64 %0, {t0, t1};\n\t"
        "}"
        : "=l"(t)
        : "l"(x), "l"(w), "l"(h), "l"(p.nq));
    return t;
#endif
#else
    return x * w - h * p.q;
#endif
}

// Shoup multiplication by a fixed w < q with ws = floor(w * 2^64 / q): valid for ANY 64-bit x.
// r = x*w - h*q (mod 2^64) with h = floor(x*ws / 2^64) - e:  r in [0, (2 + e) q).
//   shoup_exact: e = 0 (ptxas' own mul.hi.u64 expansion, 4 IMAD.WIDE with carry predicates), r in [0, 2q)
//   shoup_lazy:  e <= 2 (mulhi_approx, 3 IMAD.WIDE), r in [0, SB*q)
DPFHE_HD u64 shoup_exact(u64 x, u64 w, u64 ws, const LimbParams &p) { return shoup_tail(x, w, umulhi64(x, ws), p); }
DPFHE_HD u64 shoup_lazy(u64 x, u64 w, u64 ws, const LimbParams &p) { return shoup_tail(x, w, mulhi_approx(x, ws), p); }
// shoup_lazy with mulhi_approx_cc: the same value
DPFHE_HD u64 shoup_lazy_cc(u64 x, u64 w, u64 ws, const LimbParams &p) { return shoup_tail(x, w, mulhi_approx_cc(x, ws), p); }

// The Shoup factor w < q from its companion ws = floor(w * 2^64 / q) alone, exactly: ws*q lies in (w 2^64 - q, w 2^64], so
// ws*q + q - 1 lies in [w 2^64, w 2^64 + q - 1] and w = hi64(ws*q + q - 1).  A kernel that reads only the companions of a key
// row reads half the bytes (DESIGN.md §4.4).
// fast: q - 1 = qh 2^32, so ws*q + q - 1 = wl + 2^32 (wh + qh + wl qh) + 2^64 wh qh (ws = wh:wl): two IMAD.WIDE (wl qh, wh qh)
//       and a carry chain; of the middle sum only the carry out of its low word matters.
// gen:  the full 128-bit product (not used on the device's hot path).
DPFHE_HD u64 shoup_w_from_companion(u64 ws, const LimbParams &p) {
#if defined(__CUDA_ARCH__)
#if DPFHE_FAST
    const u32 qh = 0u - p.nqh;
    u64 w;
    asm("{\n\t"
        ".reg .u32 wl, wh, sl, sh, bl, bh;\n\t"
        ".reg .u64 S, B;\n\t"
        "mov.b64 {wl, wh}, %1;\n\t"
        "mul.wide.u32 S, wl, %2;\n\t"
        "mul.wide.u32 B, wh, %2;\n\t"
        "mov.b64 {sl, sh}, S;\n\t"
        "add.cc.u32 sl, sl, wh;\n\t"
        "addc.u32 sh, sh, 0;\n\t"
        "add.cc.u32 sl, sl, %2;\n\t"
        "addc.u32 sh, sh, 0;\n\t"
        "mov.b64 {bl, bh}, B;\n\t"
        "add.cc.u32 bl, bl, sh;\n\t"
        "addc.u32 bh, bh, 0;\n\t"
        "mov.b64 %0, {bl, bh};\n\t"
        "}"
        : "=l"(w)
        : "l"(ws), "r"(qh));
    return w;
#else
    const u64 hi = umulhi64(ws, p.q), lo = ws * p.q;
    const u64 s = lo + (p.q - 1);
    return hi + (s < lo ? 1u : 0u);
#endif
#else
    return (u64)(((unsigned __int128)ws * p.q + (p.q - 1)) >> 64);
#endif
}

// 128-bit product (hi:lo) of two 64-bit words.  Device: four IMAD.WIDE partial products combined once
// (nvcc's separate a*b and __umul64hi(a,b) would recompute the low partial product: 5 IMAD.WIDE + 2 IMAD).
DPFHE_HD void mul128(u64 a, u64 b, u64 &hi, u64 &lo) {
#if defined(__CUDA_ARCH__)
    asm("{\n\t"
        ".reg .u32 al, ah, bl, bh, p0l, p0h, ml, mh, cy;\n\t"
        ".reg .u64 p0, p1, p2, p3, m, t;\n\t"
        "mov.b64 {al, ah}, %2;\n\t"
        "mov.b64 {bl, bh}, %3;\n\t"
        "mul.wide.u32 p0, al, bl;\n\t"
        "mul.wide.u32 p1, al, bh;\n\t"
        "mul.wide.u32 p2, ah, bl;\n\t"
        "mul.wide.u32 p3, ah, bh;\n\t"
        "mov.b64 {p0l, p0h}, p0;\n\t"
        "add.cc.u64 m, p1, p2;\n\t"
        "addc.u32 cy, 0, 0;\n\t"
        "cvt.u64.u32 t, p0h;\n\t"
        "add.cc.u64 m, m, t;\n\t"
        "addc.u32 cy, cy, 0;\n\t"
        "mov.b64 {ml, mh}, m;\n\t"
        "mov.b64 %1, {p0l, ml};\n\t"
        "mov.b64 t, {mh, cy};\n\t"
        "add.u64 %0, p3, t;\n\t"
        "}"
        : "=l"(hi), "=l"(lo)
        : "l"(a), "l"(b));
#else
    unsigned __int128 z = (unsigned __int128)a * b;
    lo = (u64)z;
    hi = (u64)(z >> 64);
#endif
}

// (hi:lo) -= (bh:bl), no borrow out expected
DPFHE_HD void sub128(u64 &hi, u64 &lo, u64 bh, u64 bl) {
#if defined(__CUDA_ARCH__)
    asm("sub.cc.u64 %0, %0, %2;\n\tsubc.u64 %1, %1, %3;" : "+l"(lo), "+l"(hi) : "l"(bl), "l"(bh));
#else
    const unsigned __int128 z = (((unsigned __int128)hi << 64) | lo) - (((unsigned __int128)bh << 64) | bl);
    lo = (u64)z;
    hi = (u64)(z >> 64);
#endif
}

// Barrett reduction of z = hi:lo.  Requires z < 2^(s+64), s = bitlen(q) - 2, i.e. z <= 4 q^2 (factor bounds Ba*Bb <= 4:
// the shifted value must fit one word).  With the exact quotient the result is in [0, 3q) ([0, 2q) for canonical
// factors); the estimate of mulhi_approx adds at most 2q: [0, (SB+1) q) and [0, SB*q).
DPFHE_HD u64 barrett_lazy(u64 hi, u64 lo, const LimbParams &p) {
    const u32 s = p.bar_shift;                       // 32 <= s <= 58 because 2^33 < q < 2^60
#if defined(__CUDA_ARCH__)
    // floor(z / 2^s) with two funnel shifts over the three upper words of z
    const u32 w1 = (u32)(lo >> 32), w2 = (u32)hi, w3 = (u32)(hi >> 32);
    const u32 zl = __funnelshift_r(w1, w2, s - 32), zh = __funnelshift_r(w2, w3, s - 32);
    const u64 zt = ((u64)zh << 32) | zl;
#else
    const u64 zt = (hi << (64 - s)) | (lo >> s);     // floor(z / 2^s) < 2^64
#endif
    return sub_mul_q(lo, mulhi_approx_cc(zt, p.bar_mu), p);   // lo - qhat*q
}

// Barrett reduction of a longer sum z = hi:lo < 2^(2b+4), b = bit length of q (e.g. 16 products of canonical factors):
// the quotient is estimated from z / 2^(s+2) so that the shifted value still fits one word; 4*qh is within 14 of
// floor(z/q), so the result is in [0, 15q) (and 15q < 2^64).  Exact high product: once per 16 multiply-accumulates.
DPFHE_HD u64 barrett_lazy_long(u64 hi, u64 lo, const LimbParams &p) {
    const u32 s = p.bar_shift + 2;                   // 34 <= s <= 60
#if defined(__CUDA_ARCH__)
    const u32 w1 = (u32)(lo >> 32), w2 = (u32)hi, w3 = (u32)(hi >> 32);
    const u32 zl = __funnelshift_r(w1, w2, s - 32), zh = __funnelshift_r(w2, w3, s - 32);
    const u64 zt = ((u64)zh << 32) | zl;
#else
    const u64 zt = (hi << (64 - s)) | (lo >> s);     // floor(z / 2^s) < 2^64
#endif
    const u64 qh = umulhi64(zt, p.bar_mu);
    return sub_mul_q(lo, qh << 2, p);                // lo - 4*qh*q
}

// product of two values whose bounds multiply to at most 4: [0, (SB+1) q); canonical factors: [0, SB*q)
DPFHE_HD u64 mulmod_lazy(u64 a, u64 b, const LimbParams &p) {
    u64 hi, lo;
    mul128(a, b, hi, lo);
    return barrett_lazy(hi, lo, p);
}

// x < 16q  ->  [0, q)
DPFHE_HD u64 canon(u64 x, const LimbParams &p) {
    u64 r = word_reduce(x, p);   // < 3q
    r = csub(r, p.q2);
    return csub(r, p.q);
}
// canon for a modulus with floor(2^64 / q) == 16, i.e. q > 2^64 / 17 (the default basis and any other modulus within 6 % of 2^60):
// the quotient estimate is then k = x >> 60 without a multiplication, and x/q - x/2^60 = x (2^60 - q) / (q 2^60) < 16 (2^60 - q) / q
// < 1, so floor(x/q) - k is 0 or 1: x - k q < 2q for ANY 64-bit x and ONE conditional subtraction finishes.  Used by the store loop
// of the forward transform, where the uniform branch is hoisted out of the loop (+2.5 % on the transform); inside the fused
// kernels the second code path costs more in register pressure than it saves (DESIGN.md §6 table).
DPFHE_HD bool canon_near60_applies(const LimbParams &p) { return p.mu32 == 16u; }
DPFHE_HD u64 canon_near60(u64 x, const LimbParams &p) { return csub(sub_mul_q(x, x >> 60, p), p.q); }
// uniform branch per value (the limb constants sit in the constant bank)
DPFHE_HD u64 canon_store(u64 x, const LimbParams &p) { return canon_near60_applies(p) ? canon_near60(x, p) : canon(x, p); }
// x < 4q -> [0, q)
DPFHE_HD u64 canon4(u64 x, const LimbParams &p) { return csub(csub(x, p.q2), p.q); }

// canonical factors -> canonical product
DPFHE_HD u64 mulmod(u64 a, u64 b, const LimbParams &p) { return canon4(mulmod_lazy(a, b, p), p); }

// ---- 32-bit arithmetic modulo a prime t < 2^31 (the BGV plaintext modulus, DESIGN.md §2.13) ----
DPFHE_HD u32 mulhi32(u32 a, u32 b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);   // IMAD.HI
#else
    return (u32)(((u64)a * b) >> 32);
#endif
}
DPFHE_HD u32 csub32(u32 x, u32 t) { return x >= t ? x - t : x; }
// Shoup multiplication by a fixed w < t with ws = floor(w * 2^32 / t), canonical result for ANY 32-bit x: h = hi32(x * ws) is
// floor(x w / t) or one less, so x w - h t lies in [0, 2t) and 2t < 2^32: the low words give it exactly (one IMAD.HI, two IMAD)
DPFHE_HD u32 shoup32(u32 x, u32 w, u32 ws, u32 t) { return csub32(x * w - mulhi32(x, ws) * t, t); }
DPFHE_HD u32 add32(u32 a, u32 b, u32 t) { return csub32(a + b, t); }   // canonical operands
DPFHE_HD u32 sub32(u32 a, u32 b, u32 t) { return a >= b ? a - b : a + t - b; }
// any 64-bit x -> x mod t: x = xh 2^32 + xl, reduced as xh (2^32 mod t) + xl * 1 with two Shoup products
DPFHE_HD u32 reduce64_32(u64 x, const Mod32 &m) {
    return add32(shoup32((u32)(x >> 32), m.r32, m.r32_s, m.t), shoup32((u32)x, 1u, m.one_s, m.t), m.t);
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
