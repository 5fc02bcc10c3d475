/*
 * dpfhe_level.h — the polynomial evaluators and the keyless calls at level l of the modulus chain, on the top-level context
 * (DESIGN.md §2.22).  Included by dpfhe.h; the types and conventions are dpfhe.h's.  With the key-switching calls and objects at a
 * level (dpfhe.h, DESIGN.md §2.20, §2.21) they run a whole network, from encoding to decoding, on one context with one set of
 * top-level keys.
 */
#ifndef DPFHE_LEVEL_H
#define DPFHE_LEVEL_H

#include "dpfhe.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- BGV and CKKS polynomial evaluation (dpfhe_polyeval_create_grouped / _ckks) at level l: bit for bit the top-level object
 *      created on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the top-level key h_relin_key [dnum][2][L][N] restricted to
 *      that basis (its first ceil(l / K) digits, limb rows 0 .. l-1 and the special rows).  Input [batch][2][level][N]; the depth
 *      conditions of the top-level creates hold with l in place of Lq (BGV: D <= l - 1 and D <= l - K + 1, result l - D limbs;
 *      CKKS: D + 2 <= l and D <= l - K + 1, result l - D - 1 limbs).  Valid levels K <= level <= Lq; level = Lq is the top-level object.  A failed create returns no object and
 *      its message names the level.  _apply, _apply_host, _destroy, _result_limbs and _result_scale serve these unchanged. */
int dpfhe_polyeval_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, uint64_t t_plain, const int64_t *coeffs,
                                        size_t degree, const uint64_t *h_relin_key, dpfhe_polyeval **out);
int dpfhe_polyeval_create_ckks_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const double *coeffs, size_t degree, double scale_in,
                                     double scale_out, const uint64_t *h_relin_key, dpfhe_polyeval **out);

/* ---- the keyless calls at level l on the top-level context (DESIGN.md §2.22).  Each call below takes the arguments of the call it
 *      is named after plus `level`, and is, bit for bit, that call on a context over the first l moduli {q_0 .. q_{l-1}}: every
 *      buffer over the limbs ([..][level][N]) is sized by the level, and so are the overlap checks.  Under a context with special
 *      primes this encodes, encrypts, adds and multiplies plaintexts, rescales, decrypts and decodes level-l ciphertexts (l <= Lq)
 *      without a context over the ciphertext moduli.  Keys are the top-level ones: d_sk [L][N], of which the first `level` rows are
 *      read, and the public key d_pk [2][L][N], of whose components the first `level` rows are read.  Valid levels 1 <= level <= L
 *      (mod_switch_down_level: 2 <= level; its output is [n_polys][level-1][N]); level = L is the call itself.  A failed check
 *      leaves the output untouched and names the level.  They run on the context's own tables and scratch: a level call allocates
 *      no device memory the top-level call would not, and launches what it launches.  The *_host forms pipeline host buffers in
 *      chunks (synchronous). ---- */
int dpfhe_ckks_encode_level(dpfhe_ctx *ctx, unsigned level, const double *d_slots, uint64_t *d_pt, size_t n_vec, double scale, void *stream);
int dpfhe_ckks_decode_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_pt, double *d_slots, size_t n_vec, double scale, void *stream);
int dpfhe_ckks_encode_level_host(dpfhe_ctx *ctx, unsigned level, const double *h_slots, uint64_t *h_pt, size_t n_vec, double scale);
int dpfhe_ckks_decode_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_pt, double *h_slots, size_t n_vec, double scale);
int dpfhe_bgv_encode_level(dpfhe_ctx *ctx, unsigned level, const int64_t *d_slots, uint64_t *d_pt, size_t n_vec, uint64_t t_plain, void *stream);
int dpfhe_bgv_decode_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_pt, uint64_t *d_slots, size_t n_vec, uint64_t t_plain, void *stream);
int dpfhe_bgv_encode_level_host(dpfhe_ctx *ctx, unsigned level, const int64_t *h_slots, uint64_t *h_pt, size_t n_vec, uint64_t t_plain);
int dpfhe_bgv_decode_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_pt, uint64_t *h_slots, size_t n_vec, uint64_t t_plain);
int dpfhe_encrypt_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                        const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream);
int dpfhe_encrypt_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                             const uint64_t *h_pt, uint64_t *h_ct, size_t n);
int dpfhe_encrypt_public_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_pk, const uint8_t seed[32], uint64_t first_index,
                               const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream);
int dpfhe_encrypt_public_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_pk, const uint8_t seed[32],
                                    uint64_t first_index, const uint64_t *h_pt, uint64_t *h_ct, size_t n);
int dpfhe_decrypt_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_sk, const uint64_t *d_ct, unsigned n_comp, uint64_t *d_pt, size_t n,
                        void *stream);
int dpfhe_decrypt_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_sk, const uint64_t *h_ct, unsigned n_comp, uint64_t *h_pt,
                             size_t n);
int dpfhe_ct_add_plain_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch,
                             void *stream);
int dpfhe_ct_mul_plain_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch,
                             void *stream);
int dpfhe_ct_lincomb_level(dpfhe_ctx *ctx, unsigned level, size_t n_terms, const uint64_t *const *d_cts, const int64_t *coeffs, int64_t constant,
                           uint64_t *d_out, size_t batch, void *stream);
int dpfhe_mod_switch_down_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain,
                                void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DPFHE_LEVEL_H */
