/*
 * dpfhe_compact.h — compact ciphertexts (DESIGN.md §2.24).  Included by dpfhe.h; the types and conventions are dpfhe.h's.
 *
 * A compact ciphertext is a level-1 ciphertext switched from q0 to the power-of-two modulus 2^bits and bit-packed: (c0', c1') with
 * coefficients in [0, 2^bits), coefficient form, natural order, coefficient i of a polynomial in bits [i bits, (i + 1) bits) of a
 * little-endian stream of N bits / 64 words.  The layout is [n][2][N bits / 64] words, so a compact ciphertext is N bits / 4 bytes
 * against 16 l N for a full one at level l.  It carries the plaintext and its noise only: results leave the server in it.
 *
 * Compaction of level-l ciphertexts [n][2][l][N] (evaluation form): down to q0 (BGV, t_plain odd: the composition of l - 1 modulus
 * switches with t_plain; CKKS, t_plain = 0: limb 0 alone, which decrypts when |phase| < q0 / 2), the inverse transform, then
 * y = round(2^bits x / q0) mod 2^bits (CKKS) or floor(2^bits x / q0) - j mod 2^bits (BGV, j in (-t/2, t/2] such that
 * y = lambda x mod t with lambda = 2^bits q0^-1 mod t).  Decryption gives a level-1 plaintext [n][1][N] in evaluation form, which
 * dpfhe_bgv_decode_level / dpfhe_ckks_decode_level at level 1 take (BGV with t_plain; CKKS at the caller's scale).  It reads row 0 of
 * the secret [L][N], which must be ternary (dpfhe_secret_keygen's).
 *
 * Checks: 1 <= level <= L; bits >= 2 and N 2^bits < q0; t_plain = 0 or odd with 3 <= t_plain < 2^(bits-1); BGV at level >= 2: the
 * checks of the modulus switches down to q0.  Null and misaligned pointers, and outputs that overlap an input, are rejected.  Every
 * check runs before the first launch or copy; a failed check leaves the output untouched.
 */
#ifndef DPFHE_COMPACT_H
#define DPFHE_COMPACT_H

#include "dpfhe.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- compaction on the device: d_ct [n][2][level][N] -> d_out [n][2][N bits / 64] (asynchronous).  Launches: 2 (CKKS or level 1),
 *      2 level (BGV at level >= 2).  Device scratch, kept by the context until dpfhe_context_trim: 2 n N words (CKKS or level 1), or
 *      2 n N (2 level - 3) words at BGV level >= 2 (the outputs of the modulus switches, in two buffers used in turn), about
 *      (2 level - 3) / level times the input; dpfhe_download_compact_ciphertexts needs it for one chunk only. */
int dpfhe_compact_ciphertexts(dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, const uint64_t *d_ct, uint64_t *d_out,
                              size_t n, void *stream);

/* ---- device ciphertexts to host compact words (synchronous): chunk by chunk, each chunk compacted on the context's stream into
 *      staging and only the packed words copied back.  The first compaction waits for the context's previous call and for the work
 *      queued on the legacy default stream. */
int dpfhe_download_compact_ciphertexts(dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, const uint64_t *d_ct,
                                       uint64_t *h_out, size_t n);

/* ---- decryption of compact ciphertexts d_cct [n][2][N bits / 64] with the secret d_sk [L][N] (row 0 read) into level-1 plaintexts
 *      d_pt [n][1][N], evaluation form (asynchronous; 6 launches).  _host: host buffers, pipelined in chunks (synchronous). */
int dpfhe_decrypt_compact(dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, const uint64_t *d_sk, const uint64_t *d_cct, uint64_t *d_pt,
                          size_t n, void *stream);
int dpfhe_decrypt_compact_host(dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, const uint64_t *h_sk, const uint64_t *h_cct,
                               uint64_t *h_pt, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* DPFHE_COMPACT_H */
