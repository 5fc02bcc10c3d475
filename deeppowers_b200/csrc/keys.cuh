// keys.cuh — key generation, encryption and decryption sampled from a ChaCha20 stream (DESIGN.md §2.14, §4.10).
//
// Everything here is __host__ __device__, like the CKKS and BGV bodies.  The ChaCha20 quarter-round is 32-bit add, xor and
// rotate only: it does not touch the integer multiplier that bounds the transforms.
#pragma once
#include "kernel_bodies.cuh"

namespace dpfhe {

// nonce word n0 = domain | K << 8 | digit << 16 | limb << 24 (DESIGN.md §2.14)
enum KeyDomain : u32 {
    KD_SECRET = 1, KD_KEY_A = 2, KD_KEY_E = 3, KD_ENC_A = 4, KD_ENC_E = 5,
    KD_PK_A = 6, KD_PK_E = 7,                          // public key (the key owner's seed)
    KD_PENC_U = 8, KD_PENC_E0 = 9, KD_PENC_E1 = 10,    // public-key encryption (the encryptor's seed)
    KD_PUBLIC_SEED = 11,                               // the public seed a_seed (the key owner's seed; DESIGN.md §2.23)
    KD_SENC_A = 12, KD_SENC_E = 13,                    // seeded encryption: a from a_seed, e from the key owner's seed
    KD_SKEY_A = 14, KD_SKEY_E = 15                     // seeded switch keys: likewise
};
DPFHE_HD u32 key_nonce0(u32 domain, u32 K, u32 digit, u32 limb) { return domain | K << 8 | digit << 16 | limb << 24; }
// the ChaCha20 key of the `a` rows: the public seed of a seeded mode (whose launch passes SeededKeyArgs), else the seed
template <bool SEEDED>
DPFHE_HD const u32 *key_a_seed(const KeyArgs &A) {
    if constexpr (SEEDED) return static_cast<const SeededKeyArgs &>(A).a_seed;
    else return A.seed;
}
// the unseeded mode whose formula a seeded mode shares
DPFHE_HD constexpr int key_base_mode(int mode) { return mode == KM_ENC_SEEDED ? KM_ENC : mode == KM_RELIN_SEEDED ? KM_RELIN : mode == KM_GALOIS_SEEDED ? KM_GALOIS : mode; }

namespace DPFHE_VNS {

DPFHE_HD u32 rotl32(u32 x, int n) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(x, x, n);
#else
    return (x << n) | (x >> (32 - n));
#endif
}

// ChaCha20 block function (RFC 8439 §2.3): key = seed, word 12 = counter, words 13..15 = nonce
DPFHE_HD void chacha20_block(const u32 key[8], u32 ctr, u32 n0, u32 n1, u32 n2, u32 out[16]) {
    u32 x[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
                 key[4],      key[5],      key[6],      key[7],      ctr,    n0,     n1,     n2};
    u32 y[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) y[i] = x[i];
#define DPFHE_QR(a, b, c, d)                   \
    y[a] += y[b]; y[d] = rotl32(y[d] ^ y[a], 16); \
    y[c] += y[d]; y[b] = rotl32(y[b] ^ y[c], 12); \
    y[a] += y[b]; y[d] = rotl32(y[d] ^ y[a], 8);  \
    y[c] += y[d]; y[b] = rotl32(y[b] ^ y[c], 7);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        DPFHE_QR(0, 4, 8, 12) DPFHE_QR(1, 5, 9, 13) DPFHE_QR(2, 6, 10, 14) DPFHE_QR(3, 7, 11, 15)
        DPFHE_QR(0, 5, 10, 15) DPFHE_QR(1, 6, 11, 12) DPFHE_QR(2, 7, 8, 13) DPFHE_QR(3, 4, 9, 14)
    }
#undef DPFHE_QR
#pragma unroll
    for (int i = 0; i < 16; ++i) out[i] = y[i] + x[i];
}

// ternary secret coefficient from one word: floor(3 w / 2^32) - 1
DPFHE_HD int ternary_from_word(u32 w) { return (int)(((u64)3 * w) >> 32) - 1; }
// centred binomial, eta = 21, from two words (the oracle's xo_cbd of r = lo | hi << 32)
DPFHE_HD int cbd_from_words(u32 lo, u32 hi) {
    const u64 r = (u64)lo | (u64)hi << 32;
#if defined(__CUDA_ARCH__)
    return __popcll(r & 0x1FFFFFull) - __popcll((r >> 21) & 0x1FFFFFull);
#else
    return __builtin_popcountll(r & 0x1FFFFFull) - __builtin_popcountll((r >> 21) & 0x1FFFFFull);
#endif
}
// the 128-bit integer hi 2^64 + lo reduced exactly mod q: hi (2^64 mod q) by shoup_exact ([0, 2q)) plus word_reduce(lo)
// ([0, 3q)), then canon (< 5q < 16q)
DPFHE_HD u64 uniform_reduce(u64 lo, u64 hi, u64 r64, u64 r64_s, const LimbParams &p) {
    return canon(shoup_exact(hi, r64, r64_s, p) + word_reduce(lo, p), p);
}
// a small signed value v times t (tq = t mod q, canonical) as a canonical residue
DPFHE_HD u64 small_lift(int v, u64 tq, const LimbParams &p) {
    const u64 m = mulmod((u64)(v < 0 ? -v : v), tq, p);
    return v < 0 && m ? p.q - m : m;
}

// Samples the item's small polynomial (the secret's ternary coefficients, or the noise) into `small` [N] int8, NT threads.
template <int LOGN, int NT>
DPFHE_HD void sample_small(signed char *small, const u32 seed[8], bool ternary, u32 n0, u64 item, int tid) {
    constexpr int N = 1 << LOGN;
    const int per = ternary ? 16 : 8;
    for (int b = tid; b < N / per; b += NT) {
        u32 w[16];
        chacha20_block(seed, (u32)b, n0, (u32)item, (u32)(item >> 32), w);
        if (ternary) {
#pragma unroll
            for (int i = 0; i < 16; ++i) small[b * 16 + i] = (signed char)ternary_from_word(w[i]);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) small[b * 8 + i] = (signed char)cbd_from_words(w[2 * i], w[2 * i + 1]);
        }
    }
}

// Output rows of one (item, limb) from the forward transform `buf` of t * small: the store stage.  Coefficient pair chunks
// [c_lo, c_hi) of the limb, two chunks (one ChaCha20 block of uniform values) per step; buf chunk = chunk - c_lo.
//   SECRET: out row = the transform.
//   ENC / KEY / PUBLIC_KEY: a from its stream, c0 / b = transform - a s + (plaintext | gadget term | nothing), c1 / a = a.
//   seeded ENC / KEY: a from the stream of A.a_seed in the seeded domains, only c0 / b stored ([item][L][N]).

template <int LOGN, int NT, int MODE_>
DPFHE_HD void keys_store(const u64 *buf, const KeyArgs &A, const LimbParams &p, u32 l, u32 L, size_t item, int c_lo, int c_hi, int tid) {
    constexpr int MODE = key_base_mode(MODE_);
    constexpr bool SEEDED = MODE != MODE_;
    constexpr bool SWITCH_KEY = MODE == KM_RELIN || MODE == KM_GALOIS;
    constexpr size_t N = (size_t)1 << LOGN;
    const U64x2 *sb = reinterpret_cast<const U64x2 *>(buf);
    if (MODE == KM_SECRET) {
        U64x2 *dst = reinterpret_cast<U64x2 *>(A.out + (size_t)l * N);
        for (int c = c_lo + tid; c < c_hi; c += NT) {
            U64x2 v = sb[swz_chunk(c - c_lo)];
            v.x = canon_store(v.x, p);
            v.y = canon_store(v.y, p);
            st_stream(dst + c, v);
        }
        return;
    }
    // item numbering: encryption: ciphertext item; public key: 0; switch keys: item = e * ndig + digit
    u32 digit = 0;
    u64 item_no;
    u32 g = 0;
    if (MODE == KM_ENC) {
        item_no = A.item0 + item;
    } else if (MODE == KM_PUBLIC_KEY) {
        item_no = 0;
    } else {
        digit = (u32)(item % A.ndig);
        const size_t e = item / A.ndig;
        item_no = MODE == KM_GALOIS ? A.galois[e] : 0;
        g = (u32)item_no;
    }
    const u32 n0 = key_nonce0(SEEDED ? (MODE == KM_ENC ? KD_SENC_A : KD_SKEY_A)
                                     : MODE == KM_ENC ? KD_ENC_A : MODE == KM_PUBLIC_KEY ? KD_PK_A : KD_KEY_A, A.K, digit, l);
    const bool in_digit = SWITCH_KEY && (A.K == 0 ? l == digit : (l < A.Lq && l / A.K == digit));
    const u64 r64 = A.r64[l], r64_s = A.r64_s[l], fac = A.fac[l];
    const u64 *srow = A.s + (size_t)l * N;
    U64x2 *ob = reinterpret_cast<U64x2 *>(A.out + (item * (SEEDED ? 1 : 2) + 0) * L * N + (size_t)l * N);
    U64x2 *oa = reinterpret_cast<U64x2 *>(A.out + (item * 2 + 1) * L * N + (size_t)l * N);
    const U64x2 *pt = MODE == KM_ENC ? reinterpret_cast<const U64x2 *>(A.pt + (item * L + l) * N) : nullptr;
    for (int c = c_lo + 2 * tid; c < c_hi; c += 2 * NT) {
        u32 w[16];
        chacha20_block(key_a_seed<SEEDED>(A), (u32)(c >> 1), n0, (u32)item_no, (u32)(item_no >> 32), w);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int cc = c + h;
            const U64x2 v = sb[swz_chunk(cc - c_lo)];
            const U64x2 s = ld_keep(reinterpret_cast<const U64x2 *>(srow) + cc);
            U64x2 a, b;
            a.x = uniform_reduce((u64)w[8 * h + 0] | (u64)w[8 * h + 1] << 32, (u64)w[8 * h + 2] | (u64)w[8 * h + 3] << 32, r64, r64_s, p);
            a.y = uniform_reduce((u64)w[8 * h + 4] | (u64)w[8 * h + 5] << 32, (u64)w[8 * h + 6] | (u64)w[8 * h + 7] << 32, r64, r64_s, p);
            u64 add[2] = {0, 0};
            if (MODE == KM_ENC) {
                const U64x2 m = ld_stream(pt + cc);
                add[0] = m.x;
                add[1] = m.y;
            } else if (in_digit) {
                u64 tg[2];
                if (MODE == KM_RELIN) {
                    tg[0] = mulmod(s.x, s.x, p);
                    tg[1] = mulmod(s.y, s.y, p);
                } else {
                    tg[0] = srow[galois_index<LOGN>(2 * cc, g)];
                    tg[1] = srow[galois_index<LOGN>(2 * cc + 1, g)];
                }
                add[0] = mulmod(tg[0], fac, p);
                add[1] = mulmod(tg[1], fac, p);
            }
            const u64 ev[2] = {canon_store(v.x, p), canon_store(v.y, p)};
            const u64 as[2] = {mulmod(a.x, s.x, p), mulmod(a.y, s.y, p)};
            u64 r[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const u64 d = csub(ev[e] + p.q - as[e], p.q);   // t e - a s
                r[e] = csub(d + add[e], p.q);
            }
            b.x = r[0];
            b.y = r[1];
            st_stream(ob + cc, b);
            if (!SEEDED) st_stream(oa + cc, a);
        }
    }
}

// the noise (or ternary) row of an item: nonce and domain
template <int MODE_>
DPFHE_HD void keys_small_nonce(const KeyArgs &A, size_t item, u32 &n0, u64 &item_no) {
    constexpr int MODE = key_base_mode(MODE_);
    constexpr bool SEEDED = MODE != MODE_;
    if (MODE == KM_SECRET) {
        n0 = key_nonce0(KD_SECRET, 0, 0, 0);
        item_no = 0;
    } else if (MODE == KM_ENC) {
        n0 = key_nonce0(SEEDED ? KD_SENC_E : KD_ENC_E, 0, 0, 0);
        item_no = A.item0 + item;
    } else if (MODE == KM_PUBLIC_KEY) {
        n0 = key_nonce0(KD_PK_E, 0, 0, 0);
        item_no = 0;
    } else {
        const u32 digit = (u32)(item % A.ndig);
        n0 = key_nonce0(SEEDED ? KD_SKEY_E : KD_KEY_E, A.K, digit, 0);
        item_no = MODE == KM_GALOIS ? A.galois[item / A.ndig] : 0;
    }
}

// one (item, limb) at N <= 8192: sample, forward transform with the lift in the load stage, output rows in the store stage
template <int LOGN, int NT, int MODE, class CTA>
DPFHE_HD void keys_limb_body(CTA &cta, u64 *buf, signed char *small, const KeyArgs &A, const Twiddle *tw, const LimbParams &p, u32 l, u32 L,
                             size_t item) {
    u32 n0;
    u64 item_no;
    keys_small_nonce<MODE>(A, item, n0, item_no);
    cta.par([&](int tid) { sample_small<LOGN, NT>(small, A.seed, MODE == KM_SECRET, n0, item_no, tid); });
    const u64 tq = A.tq[l];
    auto src = [&](int c) {
        U64x2 r;
        r.x = small_lift(small[2 * c], tq, p);
        r.y = small_lift(small[2 * c + 1], tq, p);
        return r;
    };
    cta.par([&](int tid) { fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, src); });
    fwd_passes<LOGN, NT, 1>(cta, buf, tw, p);
    cta.par([&](int tid) { keys_store<LOGN, NT, MODE>(buf, A, p, l, L, item, 0, 1 << (LOGN - 1), tid); });
}

// N = 16384: CTA h of a pair keeps output blocks {2h, 2h+1} (as ckks_enc_ntt_pair_kernel); both regenerate the whole small row
template <int NT, int MODE, class CTA>
DPFHE_HD void keys_half_body(CTA &cta, u64 *buf, signed char *small, const KeyArgs &A, const Twiddle *tw, const LimbParams &p, u32 l, u32 L,
                             size_t item, int h) {
    constexpr int LOGN = NTT_PAIR_LOGN, HC = 1 << (LOGN - 2);
    u32 n0;
    u64 item_no;
    keys_small_nonce<MODE>(A, item, n0, item_no);
    cta.par([&](int tid) { sample_small<LOGN, NT>(small, A.seed, MODE == KM_SECRET, n0, item_no, tid); });
    const u64 tq = A.tq[l];
    auto src = [&](int c) {
        U64x2 r;
        r.x = small_lift(small[2 * c], tq, p);
        r.y = small_lift(small[2 * c + 1], tq, p);
        return r;
    };
    ntt_fwd_half_load_src<NT>(cta, buf, src, tw, p, h);
    fwd_passes_blk<LOGN, NT, 1, 2>(cta, buf, tw, p, 2 * h);
    cta.par([&](int tid) { keys_store<LOGN, NT, MODE>(buf, A, p, l, L, item, h * HC, (h + 1) * HC, tid); });
}

// Public-key encryption (KM_ENC_PUBLIC): ct = (b U + t E0 + pt, a U + t E1) with U = NTT(u), E0 = NTT(e0), E1 = NTT(e1) and the
// public key (b, a) at A.s / A.s + A.pk_a.  One limb buffer: pass 0 (buf = U) writes c0 = b U + pt and c1 = a U, pass 1 (buf = t E0)
// adds into c0, pass 2 (buf = t E1) into c1.  A thread owns the same chunks in every pass, so it reads back only its own stores
// (through L2: .cg); the rows it finishes in a pass are written with st_stream.
template <int LOGN, int NT, int PASS>
DPFHE_HD void pub_enc_store(const u64 *buf, const KeyArgs &A, const LimbParams &p, u32 l, u32 L, size_t item, int c_lo, int c_hi, int tid) {
    constexpr size_t N = (size_t)1 << LOGN;
    const U64x2 *sb = reinterpret_cast<const U64x2 *>(buf);
    U64x2 *o0 = reinterpret_cast<U64x2 *>(A.out + (item * 2 + 0) * L * N + (size_t)l * N);
    U64x2 *o1 = reinterpret_cast<U64x2 *>(A.out + (item * 2 + 1) * L * N + (size_t)l * N);
    const U64x2 *pkb = reinterpret_cast<const U64x2 *>(A.s + (size_t)l * N);
    const U64x2 *pka = reinterpret_cast<const U64x2 *>(A.s + A.pk_a + (size_t)l * N);
    const U64x2 *pt = reinterpret_cast<const U64x2 *>(A.pt + (item * L + l) * N);
    for (int c = c_lo + tid; c < c_hi; c += NT) {
        const U64x2 v = sb[swz_chunk(c - c_lo)];
        const u64 ev[2] = {canon_store(v.x, p), canon_store(v.y, p)};
        if (PASS == 0) {
            const U64x2 b = ld_keep(pkb + c), a = ld_keep(pka + c), m = ld_stream(pt + c);
            U64x2 r0, r1;
            r0.x = csub(mulmod(ev[0], b.x, p) + m.x, p.q);
            r0.y = csub(mulmod(ev[1], b.y, p) + m.y, p.q);
            r1.x = mulmod(ev[0], a.x, p);
            r1.y = mulmod(ev[1], a.y, p);
            st_cg(o0 + c, r0);
            st_cg(o1 + c, r1);
        } else {
            U64x2 *o = PASS == 1 ? o0 : o1;
            U64x2 r = ld_cg(o + c);
            r.x = csub(r.x + ev[0], p.q);
            r.y = csub(r.y + ev[1], p.q);
            st_stream(o + c, r);
        }
    }
}

// one pass of public-key encryption: sample u (ternary; PASS 0), e0 or e1 (noise), the forward transform with the lift (u by 1,
// the noise by t) in the load stage, then the pass's store stage.  N <= 8192: the whole limb (h unused); N = 16384: CTA h of the
// pair keeps output blocks {2h, 2h+1} and regenerates the whole small row, as keys_half_body
template <int LOGN, int NT, int PASS, class CTA>
DPFHE_HD void pub_enc_pass(CTA &cta, u64 *buf, signed char *small, const KeyArgs &A, const Twiddle *tw, const LimbParams &p, u32 l, u32 L,
                           size_t item, int h) {
    const u32 n0 = key_nonce0(KD_PENC_U + PASS, 0, 0, 0);
    cta.par([&](int tid) { sample_small<LOGN, NT>(small, A.seed, PASS == 0, n0, A.item0 + item, tid); });
    const u64 tq = PASS == 0 ? 1 : A.tq[l];
    auto src = [&](int c) {
        U64x2 r;
        r.x = small_lift(small[2 * c], tq, p);
        r.y = small_lift(small[2 * c + 1], tq, p);
        return r;
    };
    if constexpr (LOGN == NTT_PAIR_LOGN) {
        constexpr int HC = 1 << (LOGN - 2);
        ntt_fwd_half_load_src<NT>(cta, buf, src, tw, p, h);
        fwd_passes_blk<LOGN, NT, 1, 2>(cta, buf, tw, p, 2 * h);
        cta.par([&](int tid) { pub_enc_store<LOGN, NT, PASS>(buf, A, p, l, L, item, h * HC, (h + 1) * HC, tid); });
    } else {
        cta.par([&](int tid) { fwd_load_stage<LOGN, NT, false>(buf, tw, p, tid, src); });
        fwd_passes<LOGN, NT, 1>(cta, buf, tw, p);
        cta.par([&](int tid) { pub_enc_store<LOGN, NT, PASS>(buf, A, p, l, L, item, 0, 1 << (LOGN - 1), tid); });
    }
}

// one (item, limb) of public-key encryption (h: the CTA of the pair at N = 16384, else 0)
template <int LOGN, int NT, class CTA>
DPFHE_HD void pub_enc_body(CTA &cta, u64 *buf, signed char *small, const KeyArgs &A, const Twiddle *tw, const LimbParams &p, u32 l, u32 L,
                           size_t item, int h) {
    pub_enc_pass<LOGN, NT, 0>(cta, buf, small, A, tw, p, l, L, item, h);
    pub_enc_pass<LOGN, NT, 1>(cta, buf, small, A, tw, p, l, L, item, h);
    pub_enc_pass<LOGN, NT, 2>(cta, buf, small, A, tw, p, l, L, item, h);
}

// Expansion of seeded rows (DESIGN.md §2.23), one ChaCha20 block w of [n][L][N / 4]: the four `a` values of coefficients 4b .. 4b + 3
// of limb l of row item, and the matching c0 / b words.  KEYS: row item = e * ndig + digit of [n_keys][ndig], item number
// A.galois[e] (0 for the relinearisation key); else ciphertext item, item number A.item0 + item.  src = nullptr: the c0 / b words
// are already in place (the upload writes them straight into dst).  dst [n][2][L][N].
template <int LOGN, bool KEYS>
DPFHE_HD void expand_block(const U64x2 *src, U64x2 *dst, const SeededKeyArgs &A, const LimbParams &p, u32 L, size_t w) {
    constexpr size_t NB = (size_t)1 << (LOGN - 2);
    const size_t b = w % NB, row = w / NB;
    const u32 l = (u32)(row % L);
    const size_t item = row / L;
    u32 digit = 0;
    u64 item_no;
    if (KEYS) {
        digit = (u32)(item % A.ndig);
        item_no = A.galois[item / A.ndig];
    } else {
        item_no = A.item0 + item;
    }
    u32 x[16];
    chacha20_block(A.a_seed, (u32)b, key_nonce0(KEYS ? KD_SKEY_A : KD_SENC_A, A.K, digit, l), (u32)item_no, (u32)(item_no >> 32), x);
    const u64 r64 = A.r64[l], r64_s = A.r64_s[l];
    U64x2 a[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        a[h].x = uniform_reduce((u64)x[8 * h + 0] | (u64)x[8 * h + 1] << 32, (u64)x[8 * h + 2] | (u64)x[8 * h + 3] << 32, r64, r64_s, p);
        a[h].y = uniform_reduce((u64)x[8 * h + 4] | (u64)x[8 * h + 5] << 32, (u64)x[8 * h + 6] | (u64)x[8 * h + 7] << 32, r64, r64_s, p);
    }
    const size_t in_row = (size_t)l << (LOGN - 1), c = 2 * b;   // 16-byte chunks: limb offset, first chunk of the block
    U64x2 *o0 = dst + item * 2 * L * (NB * 2) + in_row + c;
    U64x2 *o1 = o0 + L * (NB * 2);
    if (src) {
        const U64x2 *s0 = src + row * (NB * 2) + c;
        const U64x2 v0 = ld_stream(s0), v1 = ld_stream(s0 + 1);
        st_stream(o0, v0);
        st_stream(o0 + 1, v1);
    }
    st_stream(o1, a[0]);
    st_stream(o1 + 1, a[1]);
}

// decryption, one 16-byte chunk c of [n][L][N]: c0 + c1 s (+ c2 s^2)
DPFHE_HD U64x2 decrypt_chunk(const U64x2 *ct, const U64x2 *s, size_t pc, u32 n_comp, const LimbParams &p) {
    const U64x2 c0 = ld_stream(ct), c1 = ld_stream(ct + pc), sv = ld_keep(s);
    U64x2 r;
    r.x = csub(c0.x + mulmod(c1.x, sv.x, p), p.q);
    r.y = csub(c0.y + mulmod(c1.y, sv.y, p), p.q);
    if (n_comp == 3) {
        const U64x2 c2 = ld_stream(ct + 2 * pc);
        r.x = csub(r.x + mulmod(c2.x, mulmod(sv.x, sv.x, p), p), p.q);
        r.y = csub(r.y + mulmod(c2.y, mulmod(sv.y, sv.y, p), p), p.q);
    }
    return r;
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
