// compact.cuh — compact ciphertexts (DESIGN.md §2.24): the switch of a level-1 ciphertext from q0 to the power-of-two modulus 2^b,
// the bit packing of its coefficients, and the client's way back to a level-1 plaintext.
//
// __host__ __device__ like every kernel body, so that the host emulator (tests/emu/emu_compact.cpp) runs the product's code.  A
// polynomial of N b-bit coefficients is packed as a little-endian bit stream: coefficient i takes bits [i b, (i + 1) b), so a tile of
// 64 coefficients is exactly b words.  A work item is one tile, run by one warp: a lane computes coefficients lane and lane + 32, and
// lane k < b reads or writes word k of the tile, so that a tile's words move as one coalesced run.
#pragma once
#include "kernel_bodies.cuh"
#include "modarith.cuh"

namespace dpfhe {

DPFHE_HD u64 compact_mask(u32 bits) { return ((u64)1 << bits) - 1; }

// word k of a tile whose 64 coefficients y[0 .. 63] are below 2^bits
DPFHE_HD u64 compact_pack_word(const u64 *y, u32 bits, u32 k) {
    const u32 lo = 64 * k;
    u64 w = 0;
    for (u32 i = lo / bits; i < 64 && i * bits < lo + 64; ++i) {
        const int s = (int)(i * bits) - (int)lo;
        w |= s < 0 ? y[i] >> -s : y[i] << s;
    }
    return w;
}

// coefficient i of a tile of `bits` words w
DPFHE_HD u64 compact_unpack(const u64 *w, u32 bits, u32 i) {
    const u32 o = i * bits, k = o >> 6, s = o & 63;
    u64 v = w[k] >> s;
    if (s + bits > 64) v |= w[k + 1] << (64 - s);
    return v & compact_mask(bits);
}

namespace DPFHE_VNS {

// x w mod m in [0, 2m) for any 64-bit x, with w < m < 2^62 and ws = floor(w 2^64 / m)
DPFHE_HD u64 compact_shoup(u64 x, u64 w, u64 ws, u64 m) { return x * w - umulhi64(x, ws) * m; }

// The switch of one coefficient x in [0, q0) to 2^bits.  u = 2^bits x, z = u mod q0 (a Shoup product by 2^bits mod q0) and
// floor(u / q0) = (u - z) q0^-1 mod 2^64, an exact division whose quotient is below 2^bits.  CKKS rounds to nearest (z > (q0 - 1) / 2;
// no ties, q0 is odd); BGV subtracts the representative j in [-(t-1)/2, (t-1)/2] of -z q0^-1 mod t, so that y = lambda x (mod t).
DPFHE_HD u64 compact_scale(u64 x, const CompactArgs &A) {
    const u64 z = csub(compact_shoup(x, A.r, A.r_s, A.q), A.q);
    const u64 Q = ((x << A.bits) - z) * A.qinv64;
    u64 y;
    if (A.t == 0) {
        y = Q + (z > (A.q >> 1) ? 1 : 0);
    } else {
        const u64 jr = csub(compact_shoup(z, A.c, A.c_s, A.t), A.t);   // j mod t
        y = jr > (A.t >> 1) ? Q - jr + A.t : Q - jr;
    }
    return y & compact_mask(A.bits);
}

// c1' in [0, 2^bits) lifted centred into Z_q0
DPFHE_HD u64 compact_lift(u64 c1, const CompactArgs &A) { return c1 >> (A.bits - 1) ? c1 - ((u64)1 << A.bits) + A.q : c1; }

// One coefficient of the level-1 plaintext (coefficient form) from c0' and prod = c1' s mod q0: phi = c0' + centred(prod) mod 2^bits,
// taken centred in [-2^(bits-1), 2^(bits-1)).  BGV: (phi mod t) lambda^-1 mod t, lifted centred into Z_q0.  CKKS:
// floor(phi q0 / 2^bits + 1/2) mod q0, computed from psi = phi + 2^(bits-1) in [0, 2^bits) as floor(psi q0 / 2^bits) - (q0 - 1) / 2.
DPFHE_HD u64 compact_finish(u64 c0, u64 prod, const CompactArgs &A) {
    const u64 half = (u64)1 << (A.bits - 1);
    const u64 v = prod > (A.q >> 1) ? prod - A.q : prod;   // two's complement of the centred product
    const u64 phi = (c0 + v) & compact_mask(A.bits);
    if (A.t == 0) {
        const u64 psi = phi ^ half;
        const u64 R = (psi * A.q) >> A.bits | umulhi64(psi, A.q) << (64 - A.bits);
        const u64 h = A.q >> 1;
        return R >= h ? R - h : R + h + 1;
    }
    const bool neg = phi >= half;
    const u64 a = neg ? ((u64)1 << A.bits) - phi : phi;
    u64 m = csub(compact_shoup(a, A.mu, A.mu_s, A.t), A.t);
    if (neg && m) m = A.t - m;
    return m > (A.t >> 1) ? A.q - (A.t - m) : m;
}

// ---- the tile bodies: lane 0 .. 31 of the warp of one tile; the warp synchronises between a tile's phases

// scale-and-pack, phase 1: the switched coefficients of the tile x [64] (coefficient form, [0, q0)) into y [64] (shared memory)
DPFHE_HD void compact_pack_values(const u64 *x, u64 *y, const CompactArgs &A, int lane) {
    y[lane] = compact_scale(x[lane], A);
    y[lane + 32] = compact_scale(x[lane + 32], A);
}
// phase 2: the tile's bits words into out
DPFHE_HD void compact_pack_store(const u64 *y, u64 *out, const CompactArgs &A, int lane) {
    for (u32 k = (u32)lane; k < A.bits; k += 32) out[k] = compact_pack_word(y, A.bits, k);
}

// the bits words of a packed tile src into w (shared memory)
DPFHE_HD void compact_load_words(const u64 *src, u64 *w, const CompactArgs &A, int lane) {
    for (u32 k = (u32)lane; k < A.bits; k += 32) w[k] = src[k];
}
// unpack-and-lift: the tile of c1' (its words w) lifted centred into Z_q0, coefficient form, into dst [64]
DPFHE_HD void compact_lift_tile(const u64 *w, u64 *dst, const CompactArgs &A, int lane) {
    dst[lane] = compact_lift(compact_unpack(w, A.bits, (u32)lane), A);
    dst[lane + 32] = compact_lift(compact_unpack(w, A.bits, (u32)lane + 32), A);
}
// unpack-and-finish: the tile of c0' (its words w) and of prod = c1' s mod q0 (coefficient form) into the plaintext tile dst [64]
DPFHE_HD void compact_finish_tile(const u64 *w, const u64 *prod, u64 *dst, const CompactArgs &A, int lane) {
    dst[lane] = compact_finish(compact_unpack(w, A.bits, (u32)lane), prod[lane], A);
    dst[lane + 32] = compact_finish(compact_unpack(w, A.bits, (u32)lane + 32), prod[lane + 32], A);
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
