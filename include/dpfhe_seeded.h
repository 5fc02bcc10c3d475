/*
 * dpfhe_seeded.h — seeded ciphertexts and switch keys (DESIGN.md §2.23).  Included by dpfhe.h; the types and conventions are
 * dpfhe.h's.
 *
 * A fresh symmetric ciphertext is (c0, c1) with c1 = a uniform, and a switch key digit is (b_j, a_j) with a_j uniform.  The seeded
 * forms draw every `a` row from the ChaCha20 stream of a public seed, a_seed, that the key owner's seed determines
 * (dpfhe_seeded_public_seed), so that only c0 / b and the 32-byte a_seed need to be stored, sent or copied to the device.  The
 * expansion calls regenerate the `a` rows on the device and give the full ciphertexts [n][2][L][N] and keys [n_keys][dnum][2][L][N]
 * that every other call takes.
 *
 * The seeded rows use nonce domains of their own (DESIGN.md §2.14): a seeded object and an unseeded one of the same key owner never
 * share an `a` or a noise row, and the caller cannot pick a_seed.  The restriction of §2.14 holds: the first l rows of a seeded
 * ciphertext, and of its expansion, are the level-l seeded ciphertext.  Public-key encryption has no seeded form (its c1 = a u + t e1
 * is not a stream output).
 *
 * Every check of a call runs before its first launch or copy; a failed check leaves the output untouched.  Item numbers of keys are
 * 0 (the relinearisation key) or a Galois element (odd, < 2N).  An output must not overlap an input of its call.
 */
#ifndef DPFHE_SEEDED_H
#define DPFHE_SEEDED_H

#include "dpfhe.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The public seed of a key owner: words 0..7 (32 bytes, little-endian) of the ChaCha20 block with key `seed`, counter 0 and nonce
 * (11, 0, 0).  Stateless; needs no context or device. */
int dpfhe_seeded_public_seed(const uint8_t seed[32], uint8_t a_seed[32]);

/* ---- seeded symmetric encryption: d_c0 [n][L][N] = -a s + t NTT(e) + pt with a from the public seed of `seed` (domain 12, item
 *      first_index + k, per limb) and e from `seed` (domain 13).  The arguments, t rules and noise bound are dpfhe_encrypt's.  The
 *      _level forms are the same call on the prefix basis {q_0 .. q_{level-1}} (1 <= level <= L; with special primes encrypt at
 *      level = Lq, as dpfhe_encrypt_level).  The _host forms pipeline host buffers in chunks (synchronous). */
int dpfhe_encrypt_seeded(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                         const uint64_t *d_pt, uint64_t *d_c0, size_t n, void *stream);
int dpfhe_encrypt_seeded_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                              const uint64_t *h_pt, uint64_t *h_c0, size_t n);
int dpfhe_encrypt_seeded_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32],
                               uint64_t first_index, const uint64_t *d_pt, uint64_t *d_c0, size_t n, void *stream);
int dpfhe_encrypt_seeded_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32],
                                    uint64_t first_index, const uint64_t *h_pt, uint64_t *h_c0, size_t n);

/* ---- expansion of seeded ciphertexts: d_c0 [n][L][N] -> d_ct [n][2][L][N] (c0 copied, c1 regenerated from a_seed with item numbers
 *      first_index + k).  One launch.  _level: [n][level][N] -> [n][2][level][N], 1 <= level <= L. */
int dpfhe_expand_ciphertexts(dpfhe_ctx *ctx, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *d_c0, uint64_t *d_ct, size_t n,
                             void *stream);
int dpfhe_expand_ciphertexts_level(dpfhe_ctx *ctx, unsigned level, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *d_c0,
                                   uint64_t *d_ct, size_t n, void *stream);

/* ---- host c0 [n][L][N] -> device ciphertexts d_ct [n][2][L][N] (synchronous).  Each chunk of h_c0 is copied straight into the c0
 *      rows of d_ct and its c1 rows are expanded behind the copy, so that half of the bytes of the ciphertexts cross the bus.
 *      _level: [n][level][N] -> [n][2][level][N]. */
int dpfhe_upload_seeded_ciphertexts(dpfhe_ctx *ctx, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *h_c0, uint64_t *d_ct,
                                    size_t n);
int dpfhe_upload_seeded_ciphertexts_level(dpfhe_ctx *ctx, unsigned level, const uint8_t a_seed[32], uint64_t first_index,
                                          const uint64_t *h_c0, uint64_t *d_ct, size_t n);

/* ---- seeded switch keys: the b rows [dnum][L][N] of dpfhe_relin_keygen's key, and [n_elts][dnum][L][N] of dpfhe_galois_keygen's
 *      keys, with a_j from the public seed of `seed` (domain 14) and e_j from `seed` (domain 15).  n_special = K = 0 .. 4 and the
 *      checks of the unseeded generators; Galois lists longer than 64 take several launches. */
int dpfhe_relin_keygen_seeded(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t *d_b,
                              void *stream);
int dpfhe_relin_keygen_seeded_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32],
                                   uint64_t *h_b);
int dpfhe_galois_keygen_seeded(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, size_t n_elts,
                               const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *d_b, void *stream);
int dpfhe_galois_keygen_seeded_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, size_t n_elts,
                                    const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *h_b);

/* ---- expansion of seeded switch keys: b rows [n_keys][dnum][L][N] -> keys [n_keys][dnum][2][L][N].  items (host array of n_keys):
 *      0 for the relinearisation key, else the key's Galois element.  _expand: device to device, one launch per 64 keys; _upload:
 *      host b to device keys, synchronous, each chunk copied straight into the b rows; _host: host to host, synchronous (for the
 *      object creates, which take full keys). */
int dpfhe_expand_switch_keys(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                             const uint64_t *d_b, uint64_t *d_keys, void *stream);
int dpfhe_upload_seeded_switch_keys(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                                    const uint64_t *h_b, uint64_t *d_keys);
int dpfhe_expand_switch_keys_host(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                                  const uint64_t *h_b, uint64_t *h_keys);

#ifdef __cplusplus
}
#endif
#endif /* DPFHE_SEEDED_H */
