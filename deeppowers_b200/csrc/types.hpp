// types.hpp — plain data types shared by every translation unit of libdpfhe.so (host code, both arithmetic variants).
//
// The device arithmetic exists in two compile-time variants (DESIGN.md §4.1):
//   gen   any modulus 2^33 < q < 2^60, q = 1 (mod 2N)
//   fast  every modulus of the context is q = qh * 2^32 + 1: a multiplication by q costs one 32-bit multiply-add
// kernels.cu is compiled once per variant (-DDPFHE_FAST=0 / 1); functions whose code depends on the variant live in
// namespace dpfhe::gen / dpfhe::fast (DPFHE_VNS), the types below are common to both.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define DPFHE_HD __host__ __device__ __forceinline__
#else
#define DPFHE_HD inline
#endif

#ifndef DPFHE_FAST
#define DPFHE_FAST 0
#endif
#if DPFHE_FAST
#define DPFHE_VNS fast
#else
#define DPFHE_VNS gen
#endif
// 0: exact Shoup / Barrett quotients; 2: the quotient estimates drop the low partial product and the carry of the
// middle ones (hi64 - {0,1,2}): one IMAD.WIDE and one add less per product, lazy bounds grow by 4q instead of 2q
#ifndef DPFHE_SHOUP_APPROX
#define DPFHE_SHOUP_APPROX 2
#endif

// 1: the ct x ct tensor product forms a0 b1 + a1 b0 from three 128-bit products (Karatsuba) instead of four
#ifndef DPFHE_TENSOR_KARATSUBA
#define DPFHE_TENSOR_KARATSUBA 1
#endif

namespace dpfhe {

typedef uint64_t u64;
typedef uint32_t u32;

struct alignas(16) U64x2 {
    u64 x, y;
};

// (w, floor(w*2^64/q)) pairs, 16 B each, so one 128-bit load fetches a twiddle.
typedef U64x2 Twiddle;

// bound (in units of q) of a lazy Shoup product, and of a lazy Barrett reduction of a product of canonical factors
constexpr int SB = DPFHE_SHOUP_APPROX == 0 ? 2 : 4;

// Per-limb constants (host-built in host_params.cpp; passed by value in the kernel parameter block).
struct alignas(16) LimbParams {
    u64 q;           // modulus
    u64 q2;          // 2q
    u64 qsb;         // SB * q: keeps the differences of lazy butterflies positive
    u64 q4;          // 4q
    u64 q8;          // 8q  (< 2^63)
    u64 nq;          // 2^64 - q: adding h*nq subtracts h*q without a separate negation
    u64 bar_mu;      // floor(2^(bar_shift+64) / q)
    u64 ninv;        // N^-1 mod q                    } folded into the last inverse stage
    u64 ninv_s;      // Shoup companion of ninv
    u64 wninv;       // psi^-bitrev(1) * N^-1 mod q
    u64 wninv_s;     // Shoup companion of wninv
    u32 bar_shift;   // bitlen(q) - 2
    u32 mu32;        // floor(2^64 / q)  (< 2^31 because q > 2^33)
    u32 nqh;         // fast moduli (q = qh * 2^32 + 1): -qh mod 2^32; 0 for any other modulus
    u32 pad_;
};

struct LimbTable {
    LimbParams lp[16];
};

// Modulus switching / special-prime division (DESIGN.md §2.9, §2.10): constants of one call, built on the host
// (host_params.cpp:build_ms_consts) and passed by value in the kernel parameter block.
struct MsConsts {
    u64 inv[16], inv_s[16];     // q_last^-1 mod q_i and its Shoup companion
    u64 sinv[16], sinv_s[16];   // s * q_last^-1 mod q_i (s = t_plain, or 1 for plain rounding)
    u64 qlm[16], qlm_s[16];     // q_last mod q_i and its Shoup companion (hybrid key switching scales by it)
    u64 tinv, tinv_s;           // t_plain^-1 mod q_last (BGV correction), used when has_t
    u64 half;                   // floor(q_last / 2)
    u32 has_t;
};

// Grouped hybrid key switching (DESIGN.md §2.11): the last K limbs of the context are special primes (P = their product), the
// Lq = L - K ciphertext limbs form dnum = ceil(Lq / K) digits of K consecutive limbs.  Constants of one call, built on the
// host (host_params.cpp:build_group_consts) and passed by value in the kernel parameter block, so that every use is a
// constant-bank operand with a CTA-uniform index.  The MsConsts of such a call describe the division by P (inv = P^-1 ...).
constexpr int KS_MAX_SPECIAL = 4;
constexpr int ROT_SUM_MAX = 15;   // rotations of one summed-rotation call (DESIGN.md §2.17)
struct GroupConsts {
    u32 Lq, K, dnum, pad_;
    // limb parameters whose N^-1 (ninv, wninv) carries the factor that the basis conversion wants on the inverse transform's
    // output: Qhat_j^-1 mod q_j for a ciphertext limb j (Qhat_j = product of the other moduli of its group), and
    // (t * Phat_k)^-1 mod p_k for special limb Lq + k (Phat_k = P / p_k; t = 1 for plain rounding)
    LimbParams lp_up[16];
    u64 up[16][16], up_s[16][16];                                // [j][i]: Qhat_j mod q_i, with its Shoup companion (j < Lq, i < L)
    u64 dn[KS_MAX_SPECIAL][16], dn_s[KS_MAX_SPECIAL][16];      // [k][i]: Phat_k mod q_i (i < Lq)
    u64 neg_p[16];                                               // q_i - (P mod q_i): adding it subtracts P
    u64 half[KS_MAX_SPECIAL];                                    // floor(p_k / 2)
};

// Multiply-and-rescale (DESIGN.md §2.19, §4.16): the division by P' = P * qbar, qbar = q_{Lq-1} the dropped ciphertext limb.  The
// GroupConsts of such a call describe P' for the K special rows (lp_up, dn, neg_p), its MsConsts divide by P'; this block is the
// divided set's fifth row, kept apart so that the parameter blocks of the other grouped kernels keep their layout
// (host_params.cpp:build_rescale_consts).
struct RescaleConsts {
    LimbParams lp_drop;   // limb Lq-1 with N^-1 scaled by (t * P)^-1 mod qbar: its inverse transform yields y_qbar
    u64 dn[16], dn_s[16]; // [i]: P mod q_i (= P' / qbar), with its Shoup companion (i < Lq - 1)
    u64 half;             // floor(qbar / 2)
    u64 *tau;             // [groups][2 parities][2][N]: y_qbar of the dropped limb's CTA, double-buffered by round parity
    u32 *tau_flag;        // [groups]: round tag of the last y_qbar published
    u32 pad_[2];
};

// ---- twiddle table layout (host_params.cpp writes it, ntt_core.cuh reads it) -----------------------------
// natural index of the twiddle of group i at stage s is 2^s + i.  Stages of the last
// register pass (s >= LOGN-4) are stored transposed so that lane-consecutive rows read
// consecutive table entries:  i = row * 2^u + j  ->  2^s + j * (N/16) + row,  u = s - (LOGN-4).
template <int LOGN>
DPFHE_HD int tw_pos(int s, int i) {
    if (s < LOGN - 4) return (1 << s) + i;
    const int u = s - (LOGN - 4);
    const int row = i >> u, j = i & ((1 << u) - 1);
    return (1 << s) + j * (1 << (LOGN - 4)) + row;
}

// CKKS slot encoding (DESIGN.md §2.12).  A complex double, laid out as the (re, im) pairs of the slot arrays.
struct alignas(16) Cplx {
    double re, im;
};
constexpr int CKKS_POW2_E = 1024;   // 2^e mod q_l is tabulated for 0 <= e < 1024, every exponent a finite double can carry
// device tables of one context, built on first use (host_params.cpp:build_ckks_tables)
struct CkksTables {
    const Cplx *tw = nullptr;       // [N]   (cos, sin)(pi k / N), correctly rounded
    const u32 *tj = nullptr;        // [N/2] t_j = (5^j mod 2N - 1) / 4: slot j is the DFT output t_j
    const u64 *pow2 = nullptr;      // [L][CKKS_POW2_E] 2^e mod q_l
};
// decoding constants of one context (host_params.cpp:build_ckks_consts), passed by value in the kernel parameter block
struct CkksConsts {
    u64 ginv[16][16];   // [j][i] q_j^-1 mod q_i (j < i): Garner's mixed-radix digits
    u64 half[16];       // mixed-radix digits of (Q - 1) / 2, Q = q_0 ... q_{L-1}
    double qd[16];      // q_l rounded to double
    double scale;       // the divisor of the decoded coefficients
};

// BGV slot encoding (DESIGN.md §2.13).  A prime plaintext modulus t < 2^31 and the constants of its 32-bit arithmetic
// (modarith.cuh: shoup32, reduce64_32)
struct Mod32 {
    u32 t;
    u32 r32, r32_s;   // 2^32 mod t and its Shoup companion floor(r32 * 2^32 / t)
    u32 one_s;        // floor(2^32 / t), the Shoup companion of 1
};
// device tables of the plaintext modulus last used (host_params.cpp:build_bgv_tables), cached by the context
struct BgvTables {
    const u32 *tw = nullptr;    // [4][N] zeta^br(k), their Shoup companions, zeta^-br(k), their companions (br over log2 N bits)
    const u32 *pos = nullptr;   // [2][N/2] slot (r, c) -> position of its value in the bit-reversed evaluation order
    Mod32 m{};
    u32 ninv = 0, ninv_s = 0;   // N^-1 mod t and its Shoup companion
};
// decoding constants of one context and t (host_params.cpp:build_bgv_consts), passed by value in the kernel parameter block
struct BgvConsts {
    u64 ginv[16][16];       // Garner's inverses, as CkksConsts
    u64 half[16];           // mixed-radix digits of (Q - 1) / 2
    u32 qt[16], qt_s[16];   // q_i mod t and its Shoup companion
    u32 Qt;                 // Q mod t
    Mod32 m;
};

// Key generation and encryption (DESIGN.md §2.14): what one launch of the key / encryption kernels (keys.cu) produces, built in
// abi.cu and passed by value in the kernel parameter block
// the seeded modes (DESIGN.md §2.23) are KM_ENC / KM_RELIN / KM_GALOIS with `a` drawn from a_seed and only c0 / b stored
enum KeyMode { KM_SECRET = 0, KM_ENC = 1, KM_RELIN = 2, KM_GALOIS = 3, KM_PUBLIC_KEY = 4, KM_ENC_PUBLIC = 5,
               KM_ENC_SEEDED = 6, KM_RELIN_SEEDED = 7, KM_GALOIS_SEEDED = 8 };
constexpr int KEYS_MAX_ELTS = 64;   // Galois elements per launch (abi.cu splits longer lists)
struct KeyArgs {
    u32 seed[8];                  // the 32-byte seed as little-endian words (the ChaCha20 key)
    u32 K, Lq, ndig;              // special primes (0: per-limb digits), limbs the digits cover, digits per key
    u32 pk_a;                     // public-key encryption: the words from the public key's b to its a (L N of the key's context)
    u64 item0;                    // item number of the first item (encryption: first_index)
    u64 galois[KEYS_MAX_ELTS];    // item number and automorphism of Galois key e of the launch
    u64 r64[16], r64_s[16];       // 2^64 mod q_l and its Shoup companion (exact uniform reduction)
    u64 tq[16];                   // t mod q_l (1 for t = 0, and for the secret): the factor of the small row
    u64 fac[16];                  // gadget factor on the limbs of a digit: 1 (K = 0) or P mod q_l
    const u64 *s;                 // secret [L][N], evaluation form (public-key encryption: the public key, b at s, a at s + pk_a)
    const u64 *pt;                // encryption: plaintexts [n][L][N]
    u64 *out;                     // secret [L][N], keys [n_elts][ndig][2][L][N], public key [2][L][N], ciphertexts [n][2][L][N]
                                  // (seeded: keys [n_elts][ndig][L][N], ciphertexts [n][L][N])
};
// the seeded modes and the expansion of seeded rows (DESIGN.md §2.23): KeyArgs and the public seed of the `a` rows.  A type of its own,
// so that the parameter block of every unseeded instance keeps its layout (a longer KeyArgs would move the kernel parameters after it)
struct SeededKeyArgs : KeyArgs {
    u32 a_seed[8];                // the public seed as little-endian words (the ChaCha20 key of the `a` rows)
};
DPFHE_HD constexpr bool key_mode_seeded(int mode) { return mode >= KM_ENC_SEEDED; }

// Compact ciphertexts (DESIGN.md §2.24): the constants of the switch between q0 and 2^bits, built on the host (abi.cu) and passed by
// value in the kernel parameter block of compact.cu.  The "companion" of w modulo m is floor(w 2^64 / m).
struct CompactArgs {
    u64 q;             // q0
    u64 r, r_s;        // 2^bits mod q0 and its companion modulo q0
    u64 qinv64;        // q0^-1 mod 2^64
    u64 t;             // the plaintext modulus; 0: CKKS
    u64 c, c_s;        // BGV: -q0^-1 mod t and its companion modulo t (the correction j of the switch)
    u64 mu, mu_s;      // BGV: lambda^-1 mod t (lambda = 2^bits q0^-1 mod t) and its companion modulo t
    u32 bits;          // 2 <= bits, N 2^bits < q0
    u32 tiles;         // 64-coefficient tiles per polynomial, N / 64
};

// KS_DOT (grouped keys only, DESIGN.md §2.18): the digit is the third component of a SUM of tensor products
enum KsMode { KS_MUL_RELIN = 0, KS_PLAIN = 1, KS_ROTATE = 2, KS_DOT = 3 };
constexpr int DOT_MAX_TERMS = 64;   // pairs of one encrypted inner product
// tau' rows of a hybrid key-switching group are double-buffered by round parity (the division step runs one round late)
constexpr int KS_HYB_ROWS = 6;

// splitmix64 finaliser, the synthetic-data hash of DESIGN.md §5
DPFHE_HD u64 splitmix64(u64 x) {
    u64 z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

}  // namespace dpfhe
