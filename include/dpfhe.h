/*
 * dpfhe.h — C ABI of the H100-native FHE ciphertext-arithmetic engine (libdpfhe.so).
 *
 * This is the drop-in boundary for the hot path named by BASELINE.json:north_star:
 * RNS negacyclic NTT/INTT, Barrett pointwise multiply, key-switch / relinearise,
 * ct x ct, ct x pt and rotate.  The reference (deeppowers/deeppowers @1cf6449) has NO
 * FFI or operator for this path (SURVEY.md §0, §8a row a-0, §8b "Nothing calls an FHE
 * boundary today"), so each entry point below cites the reference interface whose
 * *conventions* it follows rather than one it replaces:
 *
 *   - device-bound context owning its tables, freed in destroy:
 *       hal::CUDADevice ctor/dtor        src/core/hal/cuda/cuda_device.cpp:18-41
 *   - cudaSetDevice at the top of every call, one default stream per device:
 *       src/core/hal/cuda/cuda_device.cpp:23,64,79
 *   - errors: the reference throws std::runtime_error from CUDA_CHECK
 *       (cuda_device.cpp:9-16); exceptions cannot cross a C ABI, so every call
 *       returns a status and the message is fetched with dpfhe_last_error();
 *       the C++ wrapper (include/deeppowers_fhe.hpp) re-throws std::runtime_error.
 *   - caller-owned data buffers, as hal::Tensor buffers are owned by their creator
 *       src/core/hal/cuda/cuda_tensor.cpp:36-58
 *   - the public API the examples include and that the wrapper attaches to:
 *       src/api/cpp/include/deeppowers.hpp:41-87
 *
 * Layouts (uint64 little-endian, row-major, all residues canonical in [0, q_l)):
 *   polynomial [L][N]; ciphertext [2][L][N] (c0,c1) in evaluation (NTT) form;
 *   batch [batch][2][L][N]; switch key [L digits][2 {b,a}][L limbs][N] evaluation form;
 *   plaintext [L][N] evaluation form.
 * Ring Z_q[X]/(X^N+1); forward NTT natural -> bit-reversed order, inverse the opposite
 * (DESIGN.md §2).  Inputs outside [0,q_l) give unspecified (but memory-safe) results.
 *
 * Threading: a context is bound to one device and is NOT thread-safe; use one context
 * per host thread / GPU (matches the reference's one-default-stream-per-device usage).
 * Different contexts may be used from different threads at the same time (dpfhe_multi_* does).
 * `stream` is a cudaStream_t passed as void* (NULL = the context's own stream).
 * Device-pointer entry points are asynchronous with respect to the host.  All calls on one context share
 * its scratch, so the library orders them itself: a call issued on a different stream than the previous
 * one first waits (on the device) for that previous call.  dpfhe_synchronize() waits for all of them.
 * There is no CPU fallback: without a usable CUDA device dpfhe_context_create fails.
 */
#ifndef DPFHE_H
#define DPFHE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DPFHE_MAX_LIMBS 16

typedef struct dpfhe_ctx dpfhe_ctx;

typedef struct dpfhe_params {
    uint32_t log_n;         /* N = 1 << log_n; supported: 12, 13, 14                       */
    uint32_t n_limbs;       /* L in [1, DPFHE_MAX_LIMBS]                                   */
    const uint64_t *moduli; /* L distinct primes, 2^33 < q < 2^60, q = 1 mod 2N; NULL = the */
                            /* default basis: the L largest primes k*2^32+1 below 2^60      */
                            /* (DESIGN.md §2.1).  Bases made only of k*2^32+1 primes run    */
                            /* the faster kernel variant; any other basis the generic one.  */
} dpfhe_params;

enum {
    DPFHE_OK = 0,
    DPFHE_ERR_INVALID = -1,    /* bad argument / unsupported parameter set */
    DPFHE_ERR_CUDA = -2,       /* CUDA runtime error (message has file:line) */
    DPFHE_ERR_NOMEM = -3,
    DPFHE_ERR_OS = -4          /* the operating system failed a request (dpfhe_random_seed: getrandom) */
};

/* thread-local message of the last failing call on this thread */
const char *dpfhe_last_error(void);
/* library / build identification, e.g. "dpfhe 0.1 sm_90a" */
const char *dpfhe_version(void);

/* ---- context ---- */
int dpfhe_context_create(const dpfhe_params *p, int device_id, dpfhe_ctx **out);
void dpfhe_context_destroy(dpfhe_ctx *ctx);
int dpfhe_get_modulus(const dpfhe_ctx *ctx, uint32_t limb, uint64_t *q);
int dpfhe_get_psi(const dpfhe_ctx *ctx, uint32_t limb, uint64_t *psi);
/* copies psi^bitrev(i), i<N (inverse: psi^-bitrev(i)) in natural table order to a HOST buffer of N words */
int dpfhe_get_root_powers(const dpfhe_ctx *ctx, uint32_t limb, int inverse, uint64_t *h_out);
/* bytes of device scratch the context holds (tables + pipeline scratch), for reporting */
size_t dpfhe_context_device_bytes(const dpfhe_ctx *ctx);
/* releases the scratch that grows with use (up to 4 GiB of hoisted-rotation transforms, host staging, ...) */
int dpfhe_context_trim(dpfhe_ctx *ctx);
/* the CUDA device the context is bound to */
int dpfhe_context_device(const dpfhe_ctx *ctx);
/* number of CUDA devices visible to this process (0 and an error status without a driver) */
int dpfhe_device_count(int *out);
/* waits for everything issued through this context, on whatever stream */
int dpfhe_synchronize(dpfhe_ctx *ctx);

/* ---- transforms: d_data is [n_polys][L][N], in place ---- */
int dpfhe_ntt_fwd(dpfhe_ctx *ctx, uint64_t *d_data, size_t n_polys, void *stream);
int dpfhe_ntt_inv(dpfhe_ctx *ctx, uint64_t *d_data, size_t n_polys, void *stream);

/* ---- pointwise ---- */
/* out[p][l][n] = a*b mod q_l, [n_polys][L][N]; out may BE a or b (or both), any other overlap is rejected */
int dpfhe_poly_mul_pointwise(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out,
                             size_t n_polys, void *stream);
/* out = a + b mod q_l, [n_polys][L][N] (a ciphertext is two polynomials); out may BE a or b (or both), any other overlap is rejected */
int dpfhe_poly_add(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out,
                   size_t n_polys, void *stream);
/* a,b: [batch][2][L][N] -> d: [batch][3][L][N] (d0,d1,d2); d must not overlap a or b */
int dpfhe_ct_tensor(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_d,
                    size_t batch, void *stream);

/* ---- key switching: every work item reads the key for the whole launch, so the output must overlap neither the operands nor
 *      the key (DPFHE_ERR_INVALID); this holds for every key-switching call below, Galois keys of hoisted and summed rotations
 *      included ---- */
/* d: [batch][L][N] (evaluation form) -> out: [batch][2][L][N] = sum_j NTT(INTT(d[j])) o key[j] */
int dpfhe_keyswitch(dpfhe_ctx *ctx, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out,
                    size_t batch, void *stream);
/* out = relinearise(a (x) b); a,b,out: [batch][2][L][N]; out must not alias a or b */
int dpfhe_ct_mul_relin(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk,
                       uint64_t *d_out, size_t batch, void *stream);
/* out = (c0 o pt, c1 o pt); pt [L][N] shared by the batch; out may BE ct, must not otherwise overlap it and must not overlap pt */
int dpfhe_ct_mul_plain(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out,
                       size_t batch, void *stream);
/* acc += (c0 o pt, c1 o pt): fused multiply-accumulate for diagonal-method linear layers; acc [batch][2][L][N], overlapping neither
 * ct nor pt */
int dpfhe_ct_mul_plain_acc(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_acc,
                           size_t batch, void *stream);
/* out = (sigma_g(c0) + ks0, ks1), ks = keyswitch(sigma_g(c1), gk); galois_elt odd in [1,2N);
 * out must not alias ct */
int dpfhe_rotate(dpfhe_ctx *ctx, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk,
                 uint64_t *d_out, size_t batch, void *stream);

/* rotation by k slots (k < 0: the other direction): dpfhe_rotate with the Galois element 5^k mod 2N, which
 * dpfhe_galois_element returns (SURVEY.md §8b declared rotate with an `int k`; the Galois-element form above
 * also covers the conjugation 2N-1) */
int dpfhe_galois_element(const dpfhe_ctx *ctx, int k, uint64_t *galois_elt);
int dpfhe_rotate_steps(dpfhe_ctx *ctx, const uint64_t *d_ct, int k, const uint64_t *d_gk, uint64_t *d_out,
                       size_t batch, void *stream);

/* ---- hoisted rotations (DESIGN.md §2.8b): n_rot rotations of the SAME batch, out[r] = rotate(ct, galois_elts[r], gks[r]).
 *      galois_elts and d_gks are HOST arrays of n_rot entries (d_gks[r] is a device pointer to a key [L][2][L][N]);
 *      d_out is [n_rot][batch][2][L][N].  Bit-identical to n_rot dpfhe_rotate calls, but the digit decomposition and its
 *      L(L-1) forward transforms are computed once per ciphertext.  The context keeps up to 4 GiB of scratch. ---- */
int dpfhe_rotate_hoisted(dpfhe_ctx *ctx, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                         const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, void *stream);

/* ---- plaintext inner products (the inner loop of a baby-step/giant-step matrix-vector product, DESIGN.md §4.7):
 *      out[g][k] = sum_{b < n_steps} steps[b][k] o pts[g][b]   for g < n_groups, k < batch
 *      steps [n_steps][batch][2][L][N] ciphertext batches, pts [n_groups][n_steps][L][N] plaintexts (evaluation form,
 *      shared by the batch), out [n_groups][batch][2][L][N].  Bit-identical to dpfhe_ct_mul_plain followed by
 *      n_steps-1 dpfhe_ct_mul_plain_acc per group, but every ciphertext row is read once. n_steps <= 128.  out must overlap neither
 *      steps nor pts. ---- */
int dpfhe_ct_mul_plain_inner(dpfhe_ctx *ctx, const uint64_t *d_steps, size_t n_steps, const uint64_t *d_pts, size_t n_groups,
                             uint64_t *d_out, size_t batch, void *stream);

/* ---- encrypted linear layer (SURVEY.md §8 row f-4; BASELINE.json config 4): y = W x by baby-step/giant-step diagonals,
 *      y = sum_g rot_{g*baby}( sum_b D[g*baby + b] o rot_b(x) ), a composition of the calls above that runs entirely on
 *      the device.  h_diags [n_diags][L][N]: the diagonal plaintexts in evaluation form, diagonal g*baby + b pre-rotated by
 *      -g*baby (the caller encodes them so); n_diags a multiple of baby (<= 128).  h_gk_baby [baby-1][L][2][L][N]: Galois
 *      keys of the rotations by 1 .. baby-1 slots; h_gk_giant [L][2][L][N]: key of the rotation by `baby` slots.
 *      Weights and keys are uploaded once, at creation.  apply: d_ct, d_out [batch][2][L][N] device buffers (asynchronous);
 *      apply_host: host buffers, the batch pipelined in chunks (upload / compute / download overlapped; synchronous).
 *      Uses (baby-1) + (n_diags/baby - 1) rotations per ciphertext instead of n_diags - 1. ---- */
typedef struct dpfhe_linear dpfhe_linear;
int dpfhe_linear_create(dpfhe_ctx *ctx, const uint64_t *h_diags, size_t n_diags, size_t baby, const uint64_t *h_gk_baby,
                        const uint64_t *h_gk_giant, dpfhe_linear **out);
/*      The same layer with grouped special-prime Galois keys (DESIGN.md §2.11; the context's last n_special limbs are special
 *      primes, ciphertexts carry Lq = L - n_special limbs, dnum = ceil(Lq / n_special)): h_diags [n_diags][Lq][N],
 *      h_gk_baby [baby-1][dnum][2][L][N], h_gk_giant [dnum][2][L][N]; t_plain as dpfhe_rotate_hoisted_grouped (below every
 *      special prime, 0 = plain rounding).  apply / apply_host / destroy serve both kinds; their buffers are [batch][2][Lq][N].
 *      Bit-identical to the composition of dpfhe_rotate_hoisted_grouped, dpfhe_ct_mul_plain_inner on the ciphertext moduli,
 *      dpfhe_rotate_grouped and dpfhe_poly_add; each giant step is one launch (the addition rides on the rotation's store). */
int dpfhe_linear_create_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_diags, size_t n_diags, size_t baby,
                                const uint64_t *h_gk_baby, const uint64_t *h_gk_giant, uint64_t t_plain, dpfhe_linear **out);
void dpfhe_linear_destroy(dpfhe_linear *layer);
int dpfhe_linear_apply(dpfhe_linear *layer, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
int dpfhe_linear_apply_host(dpfhe_linear *layer, const uint64_t *h_ct, uint64_t *h_out, size_t batch);

/* ---- scalar linear combinations (DESIGN.md §2.15): d_out = sum_i (coeffs[i] mod q_l) d_cts[i], plus (constant mod q_l) at every
 *      position of every c0 row; coefficients reduced by floor-mod, results canonical.  d_cts: a HOST array of n_terms (1 .. 64)
 *      device pointers, each [batch][2][L][N] over all L limbs of the context; d_out may be any of them.  One launch.
 *      dpfhe_ct_add_plain: d_out = (c0 + d_pt, c1), d_pt [L][N] shared by the batch (it must not overlap d_out); d_out may BE d_ct,
 *      any other overlap is rejected. ---- */
int dpfhe_ct_lincomb(dpfhe_ctx *ctx, size_t n_terms, const uint64_t *const *d_cts, const int64_t *coeffs, int64_t constant, uint64_t *d_out,
                     size_t batch, void *stream);
int dpfhe_ct_add_plain(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch, void *stream);
/*      host-buffer form: h_pt uploaded once, the batch pipelined in chunks (synchronous) */
int dpfhe_ct_add_plain_host(dpfhe_ctx *ctx, const uint64_t *h_ct, const uint64_t *h_pt, uint64_t *h_out, size_t batch);

/* ---- BGV polynomial evaluation down the modulus chain (DESIGN.md §2.15): slot-wise p(x) = sum_k coeffs[k] x^k mod t_plain,
 *      degree d = 1 .. 64, 2 <= t_plain < 2^31.  The context's last n_special limbs are special primes, ciphertexts come at the
 *      top level Lq = L - n_special; h_relin_key is the grouped relinearisation key [dnum][2][L][N] of the top level (the keys of
 *      the lower levels are restricted from it at creation).  D = ceil(log2 d) must satisfy D <= Lq - 1 and D <= Lq - K + 1.
 *      apply: d_ct [batch][2][Lq][N] -> d_out [batch][2][Lf][N], Lf = Lq - D (dpfhe_polyeval_result_limbs), decrypting under the
 *      first Lf limbs of the secret to p(slots) mod t exactly; asynchronous, d_out must not overlap d_ct.  apply_host: host
 *      buffers, pipelined in chunks (synchronous).  Scratch grows with the batch and counts in dpfhe_context_device_bytes. ---- */
typedef struct dpfhe_polyeval dpfhe_polyeval;
int dpfhe_polyeval_create_grouped(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const int64_t *coeffs, size_t degree,
                                  const uint64_t *h_relin_key, dpfhe_polyeval **out);
unsigned dpfhe_polyeval_result_limbs(const dpfhe_polyeval *pe);
int dpfhe_polyeval_apply(dpfhe_polyeval *pe, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
int dpfhe_polyeval_apply_host(dpfhe_polyeval *pe, const uint64_t *h_ct, uint64_t *h_out, size_t batch);
void dpfhe_polyeval_destroy(dpfhe_polyeval *pe);
/*      CKKS (DESIGN.md §2.16): slot-wise p(z) = sum_k coeffs[k] z^k with real coefficients (finite doubles), inputs at scale
 *      scale_in, the result at scale scale_out (both finite and > 0).  h_relin_key generated with t_plain = 0.  D = ceil(log2 d)
 *      must satisfy D <= Lq - 2 and D <= Lq - K + 1; the result has Lq - D - 1 limbs (dpfhe_polyeval_result_limbs) and decodes
 *      with dpfhe_ckks_decode at dpfhe_polyeval_result_scale (scale_out; 0 for a BGV evaluator).  _apply, _apply_host and
 *      _destroy serve both kinds. */
int dpfhe_polyeval_create_ckks(dpfhe_ctx *ctx, unsigned n_special, const double *coeffs, size_t degree, double scale_in, double scale_out,
                               const uint64_t *h_relin_key, dpfhe_polyeval **out);
double dpfhe_polyeval_result_scale(const dpfhe_polyeval *pe);

/* ---- modulus switching / rescale (DESIGN.md §2.9): drop the last limb of every polynomial.
 *      in [n_polys][L][N] -> out [n_polys][L-1][N] (a ciphertext is two polynomials), evaluation form.
 *      t_plain > 0: BGV modulus switch (the plaintext is scaled by q_last^-1 mod t); t_plain == 0: plain rounding.
 *      The result lives under the first L-1 moduli: evaluate it with a context created for those. ---- */
int dpfhe_mod_switch_down(dpfhe_ctx *ctx, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain,
                          void *stream);

/* ---- hybrid (special-prime) key switching (DESIGN.md §2.10).  The context's LAST limb is the special prime p:
 *      ciphertexts carry L-1 limbs ([batch][2][L-1][N]) and switch keys are [L-1 digits][2][L limbs][N], encrypting
 *      p * g_j * target.  The key-switched pair is accumulated over all L limbs and divided by p (rounding as in
 *      dpfhe_mod_switch_down, t_plain > 0 = BGV correction), which divides the key-switching noise by p.
 *      Same fused persistent kernel family as the calls above; outputs must not alias inputs. ---- */
int dpfhe_keyswitch_hybrid(dpfhe_ctx *ctx, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out, size_t batch,
                           uint64_t t_plain, void *stream);
int dpfhe_ct_mul_relin_hybrid(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk,
                              uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_rotate_hybrid(dpfhe_ctx *ctx, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk,
                        uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);

/* host-buffer forms of the three calls above (synchronous, pipelined like dpfhe_ct_mul_relin_host) */
int dpfhe_ct_mul_relin_hybrid_host(dpfhe_ctx *ctx, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk,
                                   uint64_t *h_out, size_t batch, uint64_t t_plain);
int dpfhe_rotate_hybrid_host(dpfhe_ctx *ctx, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk,
                             uint64_t *h_out, size_t batch, uint64_t t_plain);
int dpfhe_mod_switch_down_host(dpfhe_ctx *ctx, const uint64_t *h_in, uint64_t *h_out, size_t n_polys, uint64_t t_plain);

/* ---- grouped hybrid key switching: digits of several limbs, dnum < L (DESIGN.md §2.11).  The context's last n_special = K
 *      limbs are special primes (P = their product); ciphertexts carry Lq = L-K limbs ([batch][2][Lq][N]), grouped into
 *      dnum = ceil(Lq / K) digits of K consecutive limbs (the last digit may be shorter).  Switch keys are
 *      [dnum][2][L limbs][N] and encrypt P * F_g * target, F_g = 1 on the limbs of digit g and 0 on the others.  Every digit
 *      is raised to all L limbs by fast basis conversion, accumulated against its key, and the pair is divided by P (rounding
 *      as in dpfhe_mod_switch_down, every special residue lifted centred).  Against one special prime this needs fewer
 *      transforms (24 instead of 30 per ct x ct at Lq = 4, K = 2) and keys of dnum instead of Lq digits.
 *      1 <= K <= 4, 2K <= L; K = 1 is the hybrid variant above, bit for bit.  dpfhe_grouped_digits returns dnum.
 *      The reference has no counterpart (SURVEY.md §8 row f-2 widening). ---- */
int dpfhe_grouped_digits(const dpfhe_ctx *ctx, unsigned n_special, unsigned *digits);
int dpfhe_keyswitch_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out,
                            size_t batch, uint64_t t_plain, void *stream);
int dpfhe_ct_mul_relin_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_a, const uint64_t *d_b,
                               const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_rotate_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk,
                         uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
/* n_rot rotations of the SAME ciphertexts with grouped hybrid keys (d_gks[r]: [dnum][2][L][N], Galois key of galois_elts[r]),
 * sharing the basis conversion and the forward transforms of c1 ("hoisting", DESIGN.md §2.11b): one mod-up per ciphertext,
 * then per rotation only multiply-accumulates over the L limbs and the division by P (2K + 2Lq transforms instead of all of
 * them).  d_out: [n_rot][batch][2][L-K][N].  A rotation permutes the lifted digits instead of lifting the permuted digits:
 * the results decrypt to the same plaintexts with the same noise bound as dpfhe_rotate_grouped but are not the same bits
 * (the parity tests check them against the oracle's restatement of exactly this definition).  Works for n_special = 1 (hybrid
 * keys) as well. */
int dpfhe_rotate_hoisted_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                                 const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
/* Summed rotations (DESIGN.md §2.17): d_out = ct + sum_r rot_r(ct) for n_rot = 1 .. 15 rotations of the same ciphertexts,
 * [batch][2][L-K][N].  The key-switch accumulators of all rotations are summed over the L limbs and divided by P ONCE: one
 * mod-up, one summed multiply-accumulate and one division per ciphertext (24 transforms at Lq = 4, K = 2, whatever n_rot is).
 * n_rot = 1 is dpfhe_rotate_hoisted_grouped + dpfhe_poly_add with ct, bit for bit; n_rot >= 2 decrypts to the same plaintext as
 * that composition summed, not the same bits (one rounding instead of n_rot).  Argument checks of dpfhe_rotate_hoisted_grouped;
 * d_out must not overlap d_ct.  The keys' Shoup companions are built per call (n_rot launches), then 4 launches per chunk. */
int dpfhe_rotate_sum_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                             const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
/* host-buffer form: h_gks [n_rot][dnum][2][L][N] back to back, uploaded once; the batch pipelined in chunks (synchronous) */
int dpfhe_rotate_sum_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_ct, size_t n_rot, const uint64_t *galois_elts,
                                  const uint64_t *h_gks, uint64_t *h_out, size_t batch, uint64_t t_plain);
/* Encrypted inner product (DESIGN.md §2.18): d_out = relinearise(sum_i d_as[i] x d_bs[i]) for n_terms = 1 .. 64 pairs of
 * ciphertext batches [batch][2][L-K][N].  The three-component tensor products are summed exactly and key-switched ONCE: 24
 * transforms, one pass over the key and one division by P per output ciphertext at Lq = 4, K = 2, whatever n_terms is.
 * n_terms = 1 is dpfhe_ct_mul_relin_grouped, bit for bit; any n_terms is, bit for bit, dpfhe_ct_tensor per pair summed with
 * dpfhe_poly_add, dpfhe_keyswitch_grouped of the third component, and dpfhe_poly_add of the first two.  It is not the bits of
 * n_terms separate dpfhe_ct_mul_relin_grouped results summed (those round n_terms times) but decrypts to the same plaintext, with
 * one key-switching noise term instead of n_terms.  d_as, d_bs: HOST arrays of n_terms device pointers; d_as[i] and d_bs[i] may be
 * the same buffer (a sum of squares) and a buffer may appear in several pairs; d_out must not overlap any of them.  The sum of the
 * products must still fit the plaintext space (t for BGV, the scale budget for CKKS); the library does not check it.  Argument
 * checks of dpfhe_ct_mul_relin_grouped, plus n_terms and every table entry.  Two launches (key companions + kernel). */
int dpfhe_ct_dot_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                         const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
/* host-buffer form: h_as, h_bs [n_terms][batch][2][L-K][N]; the key uploaded once, the batch pipelined in chunks (synchronous) */
int dpfhe_ct_dot_grouped_host(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs,
                              const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
/* Multiply-and-rescale (DESIGN.md §2.19): the product of dpfhe_ct_mul_relin_grouped (or the inner product of dpfhe_ct_dot_grouped)
 * relinearised and divided by P * q_{Lq-1} in ONE division, Lq = L - K: d_out [batch][2][Lq-1][N] is the ciphertext one level down
 * (the CKKS rescale; BGV's modulus switch, with its factor q_{Lq-1}^-1 mod t on the slots).  It decrypts, under the first Lq - 1 limbs
 * of the secret, to what dpfhe_mod_switch_down of the unrescaled product decrypts to, but is not its bits (one rounding instead of
 * two).  24 transforms per ciphertext at Lq = 4, K = 2, against 32 for the product and a separate rescale, and no round trip of the
 * product through memory.  Same parameters and checks as the unrescaled calls, plus Lq >= 2 and t_plain below q_{Lq-1}; the output
 * must not overlap any operand.  Two launches (key companions + kernel). */
int dpfhe_ct_mul_relin_rescale_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_a, const uint64_t *d_b,
                                       const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_ct_dot_rescale_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                                 const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
/* host-buffer forms: h_a, h_b [batch][2][Lq][N] (h_as, h_bs [n_terms][batch][2][Lq][N]), h_out [batch][2][Lq-1][N]; the key
 * uploaded once, the batch pipelined in chunks (synchronous) */
int dpfhe_ct_mul_relin_rescale_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_a, const uint64_t *h_b,
                                            const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
int dpfhe_ct_dot_rescale_grouped_host(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs,
                                      const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
/* ---- calls at level l on the top-level context (DESIGN.md §2.20).  The context's last K = n_special limbs are special primes and
 *      Lq = L - K; a level-l ciphertext lies over q_0 .. q_{l-1}, [batch][2][level][N].  Each call below takes the arguments of the
 *      call it is named after plus `level`, and is, bit for bit, that call on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with
 *      the key restricted to that basis: digits g < ceil(l / K), rows 0 .. l-1 and Lq .. Lq+K-1 (the last digit is shorter when K
 *      does not divide l).  The keys are the context's TOP-LEVEL grouped keys [dnum][2][L][N], as dpfhe_relin_keygen /
 *      dpfhe_galois_keygen write them; they are read in place, never copied or restricted.  level = Lq is the call itself.
 *      Valid levels: K <= level <= Lq; the rescale forms also need level >= 2 and t_plain below q_{level-1} (their output is
 *      [batch][2][level-1][N]); t_plain below every special prime as always.  A failed check leaves the output untouched and names
 *      the level.  The first call at a (K, level) builds that level's tables on the context (counted in
 *      dpfhe_context_device_bytes, released by dpfhe_context_trim); after that a level call launches what the top-level call
 *      launches and allocates nothing.  Level calls and top-level calls share the context's round numbering and call order. ---- */
int dpfhe_ct_mul_relin_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_a, const uint64_t *d_b,
                                     const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_ct_mul_relin_rescale_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_a, const uint64_t *d_b,
                                             const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_ct_dot_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *const *d_as,
                               const uint64_t *const *d_bs, const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_ct_dot_rescale_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *const *d_as,
                                       const uint64_t *const *d_bs, const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain,
                                       void *stream);
int dpfhe_rotate_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, uint64_t galois_elt,
                               const uint64_t *d_gk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream);
int dpfhe_rotate_sum_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, size_t n_rot,
                                   const uint64_t *galois_elts, const uint64_t *const *d_gks, uint64_t *d_out, size_t batch,
                                   uint64_t t_plain, void *stream);
/* host-buffer forms of the rescale calls: operands [batch][2][level][N] ([n_terms][batch][2][level][N]), h_out
 * [batch][2][level-1][N]; the top-level key uploaded once, the batch pipelined in chunks (synchronous) */
int dpfhe_ct_mul_relin_rescale_grouped_level_host(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *h_a,
                                                  const uint64_t *h_b, const uint64_t *h_evk, uint64_t *h_out, size_t batch,
                                                  uint64_t t_plain);
int dpfhe_ct_dot_rescale_grouped_level_host(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *h_as,
                                            const uint64_t *h_bs, const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
/* ---- slot sums (DESIGN.md §2.17): slot i of the result is sum_{j < count} x[(i + j * stride) mod N/2] in every row, count =
 *      prod radices[t], computed in n_stages (1 .. 16) summed-rotation stages; stage t rotates by m * stride * prod_{u<t} radices[u],
 *      m = 1 .. radices[t] - 1 (2 <= radices[t] <= 16), and stride * count must be at most N/2.
 *      dpfhe_slotsum_steps: the rotation steps, stage by stage and m ascending, which is the order of the keys (stateless, so
 *      that the keys can be generated first); steps may be NULL (then only *n_steps is written), otherwise it holds
 *      sum (radices[t] - 1) entries.  Without a context it checks stride * count <= 8192 (N/2 at N = 16384); creation checks N/2.
 *      dpfhe_slotsum_create_grouped: h_gks [n_steps][dnum][2][L][N], the grouped Galois keys of 5^step in that order (what
 *      dpfhe_galois_keygen writes), uploaded with their Shoup companions once.  apply: d_ct, d_out [batch][2][L-K][N], d_out must
 *      not overlap d_ct; 4 launches per stage (per chunk of the hoisted-rotation scratch); the intermediate stage results are
 *      scratch that grows with the batch and counts in dpfhe_context_device_bytes.  apply_host: host buffers, pipelined in
 *      chunks (synchronous). ---- */
typedef struct dpfhe_slotsum dpfhe_slotsum;
int dpfhe_slotsum_steps(size_t stride, const unsigned *radices, size_t n_stages, int *steps, size_t *n_steps);
int dpfhe_slotsum_create_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t stride, const unsigned *radices, size_t n_stages,
                                 const uint64_t *h_gks, uint64_t t_plain, dpfhe_slotsum **out);
int dpfhe_slotsum_apply(dpfhe_slotsum *ss, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
int dpfhe_slotsum_apply_host(dpfhe_slotsum *ss, const uint64_t *h_ct, uint64_t *h_out, size_t batch);
void dpfhe_slotsum_destroy(dpfhe_slotsum *ss);
/* ---- the objects of a network layer at level l on the top-level context (DESIGN.md §2.21), in the sense of the level calls above:
 *      each is, bit for bit, the same call or object on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the keys restricted to
 *      that basis, and level = Lq is the top-level call or object itself.  The keys are the context's TOP-LEVEL grouped keys, read in
 *      place; their Shoup companions are built once at creation and serve every level.  Valid levels K <= level <= Lq; every other
 *      check is that of the top-level form; a failed check creates nothing and leaves the output untouched.  A level object builds
 *      its level's tables on the context at creation (shared with the level calls at the same (K, level)); after
 *      dpfhe_context_trim its next application builds them again.  An application launches what the top-level object's does.
 *      dpfhe_rotate_hoisted_grouped_level: n_rot hoisted rotations of level-l ciphertexts [batch][2][level][N] with the top-level
 *      keys d_gks[r] [dnum][2][L][N]; d_out [n_rot][batch][2][level][N]. */
int dpfhe_rotate_hoisted_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, size_t n_rot,
                                       const uint64_t *galois_elts, const uint64_t *const *d_gks, uint64_t *d_out, size_t batch,
                                       uint64_t t_plain, void *stream);
/*      the grouped linear layer at level l: h_diags [n_diags][level][N]; keys top-level as dpfhe_linear_create_grouped takes them.
 *      dpfhe_linear_apply / _apply_host / _destroy unchanged, their buffers [batch][2][level][N].  The level is the layer's, fixed at
 *      creation: a layer sits at a fixed depth of a network, and its diagonals take level / Lq of the top-level memory.  Both
 *      encoders (dpfhe_bgv_encode, dpfhe_ckks_encode) put the same integer in every limb, so a diagonal at level l is the first
 *      `level` rows of its top-level encoding: slice it rather than encoding again. */
int dpfhe_linear_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *h_diags, size_t n_diags,
                                      size_t baby, const uint64_t *h_gk_baby, const uint64_t *h_gk_giant, uint64_t t_plain,
                                      dpfhe_linear **out);
/*      the slot sum at level l: h_gks top-level keys in the order of dpfhe_slotsum_steps; apply buffers [batch][2][level][N] */
int dpfhe_slotsum_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t stride, const unsigned *radices,
                                       size_t n_stages, const uint64_t *h_gks, uint64_t t_plain, dpfhe_slotsum **out);
/* division by the product of the last n_special limbs alone (the mod-down half of the calls above; n_special = 1 is
 * dpfhe_mod_switch_down): in [n_polys][L][N] -> out [n_polys][L - n_special][N], 1 <= n_special <= 4, n_special < L */
int dpfhe_mod_down_special(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_in, uint64_t *d_out, size_t n_polys,
                           uint64_t t_plain, void *stream);
int dpfhe_mod_down_special_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_in, uint64_t *h_out, size_t n_polys,
                                uint64_t t_plain);
int dpfhe_ct_mul_relin_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_a, const uint64_t *h_b,
                                    const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
int dpfhe_rotate_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_ct, uint64_t galois_elt,
                              const uint64_t *h_gk, uint64_t *h_out, size_t batch, uint64_t t_plain);

/* ---- CKKS slot encoding (DESIGN.md §2.12).  Slots are N/2 complex doubles stored as interleaved (re, im) pairs,
 *      [n_vec][N/2][2]; plaintexts are [n_vec][L][N] in evaluation form.  Slot j is the value of the plaintext polynomial at
 *      exp(i pi (5^j mod 2N) / N) divided by `scale`, so dpfhe_galois_element(k) moves slot j+k to slot j and 2N-1 conjugates.
 *      encode: coefficients rint(scale * m_k), reduced exactly into every limb, then the forward transform.
 *      decode: inverse transform (into scratch: d_pt is not modified), centred CRT value / scale, then the special FFT.
 *      The results are bit-exact: the floating-point operation order is fixed by the specification.  `scale` must be finite and
 *      positive; non-finite slots, or coefficients beyond the double range, give unspecified (but memory-safe) results.
 *      A plaintext for ciphertexts under a context with special primes is encoded with the context over the ciphertext moduli.
 *      The *_host forms take host buffers and pipeline them in chunks (synchronous).  Outputs must not overlap inputs. ---- */
int dpfhe_ckks_encode(dpfhe_ctx *ctx, const double *d_slots, uint64_t *d_pt, size_t n_vec, double scale, void *stream);
int dpfhe_ckks_decode(dpfhe_ctx *ctx, const uint64_t *d_pt, double *d_slots, size_t n_vec, double scale, void *stream);
int dpfhe_ckks_encode_host(dpfhe_ctx *ctx, const double *h_slots, uint64_t *h_pt, size_t n_vec, double scale);
int dpfhe_ckks_decode_host(dpfhe_ctx *ctx, const uint64_t *h_pt, double *h_slots, size_t n_vec, double scale);

/* ---- BGV slot encoding (DESIGN.md §2.13).  The plaintext modulus t_plain must be a prime below 2^31 with t_plain = 1 (mod 2N);
 *      any other value returns DPFHE_ERR_INVALID.  Slots are [n_vec][2][N/2]: slot (0, c) is m(zeta^e) and slot (1, c) is
 *      m(zeta^(2N-e)), e = 5^c mod 2N, zeta = g^((t-1)/2N) with g the least quadratic non-residue mod t; so
 *      dpfhe_galois_element(k) rolls each row left by k and 2N-1 swaps the rows.  Plaintexts are [n_vec][L][N] in evaluation form.
 *      encode: int64 slots (any value, reduced by floor-mod into [0, t)) -> the polynomial m mod t with those slots, each
 *      coefficient lifted centred (above floor(t/2) it is m_k - t) into every limb, then the forward transform.
 *      decode: inverse transform (into scratch: d_pt is not modified), the centred CRT value mod t, its slots in [0, t).
 *      The results are exact.  The context keeps the tables of the last t_plain used; a call with another t replaces them after
 *      the earlier calls have finished.  A plaintext for ciphertexts under a context with special primes is encoded with the
 *      context over the ciphertext moduli.  The *_host forms take host buffers and pipeline them in chunks (synchronous).  Outputs
 *      must not overlap inputs. ---- */
int dpfhe_bgv_encode(dpfhe_ctx *ctx, const int64_t *d_slots, uint64_t *d_pt, size_t n_vec, uint64_t t_plain, void *stream);
int dpfhe_bgv_decode(dpfhe_ctx *ctx, const uint64_t *d_pt, uint64_t *d_slots, size_t n_vec, uint64_t t_plain, void *stream);
int dpfhe_bgv_encode_host(dpfhe_ctx *ctx, const int64_t *h_slots, uint64_t *h_pt, size_t n_vec, uint64_t t_plain);
int dpfhe_bgv_decode_host(dpfhe_ctx *ctx, const uint64_t *h_pt, uint64_t *h_slots, size_t n_vec, uint64_t t_plain);

/* ---- key generation, encryption and decryption (DESIGN.md §2.14).  Every random value is drawn from a ChaCha20 stream keyed by a
 *      caller-supplied 32-byte seed, one stream per sampled row (its nonce names the row), so the results are reproducible from the
 *      seed.  The seed is the storage form of the secret: keep it as secret as the key.  Encrypting two plaintexts with the same
 *      (seed, index) leaks their difference.  No constant-time or side-channel claim is made.  All results are canonical, in
 *      evaluation form.  t_plain >= 2 scales the noise by t (BGV), t_plain = 0 leaves it unscaled (CKKS).
 *      secret_keygen: d_sk [L][N] over all of the context's limbs, special primes included; its first l rows are the secret of
 *        the context over the first l moduli.
 *      relin_keygen / galois_keygen: switch keys for s o s / sigma_g(s) under d_sk.  n_special = 0: per-limb digits [L][2][L][N]
 *        (dpfhe_ct_mul_relin, dpfhe_rotate); n_special = K in 1 .. 4 with 2K <= L: the grouped key [dnum][2][L][N] of the
 *        *_grouped calls (K = 1: the *_hybrid calls).  galois_keygen writes n_elts keys back to back; every element odd, < 2N.
 *      encrypt: d_pt [n][L][N] plaintexts (as dpfhe_bgv_encode / dpfhe_ckks_encode produce them) -> d_ct [n][2][L][N]; ciphertext
 *        k is drawn with index first_index + k.  Under a context with special primes, encrypt and decrypt with the context over
 *        the ciphertext moduli and the first rows of the secret.
 *      decrypt: d_ct [n][n_comp][L][N], n_comp 2 or 3 -> d_pt [n][L][N] = c0 + c1 o s (+ c2 o s^2), ready for the decoders.
 *      public_keygen: d_pk [2][L][N] = (b, a) = (-a o s + t NTT(e), a), the encryption of zero under the key owner's seed with
 *        nonce domains of its own.  Its first l rows of both components are the public key of the context over the first l
 *        moduli; under a context with special primes, generate it with the context over the ciphertext moduli.
 *      encrypt_public: encryption by anyone who holds d_pk, with the ENCRYPTOR's own seed (not the key owner's): ciphertext k
 *        = (b o NTT(u) + t NTT(e0) + pt_k, a o NTT(u) + t NTT(e1)), drawn with index first_index + k; decrypt as usual with the
 *        secret.  The encryptor's seed must be kept as secret as the plaintexts: (seed, index) and the public key give pt back.
 *        Use a public key with the t_plain it was made with.
 *      The *_host forms take host buffers (encrypt / decrypt pipelined in chunks; synchronous).
 *      dpfhe_random_seed fills 32 bytes from the operating system (getrandom; DPFHE_ERR_OS if that fails).
 *      Outputs must not overlap the secret, the public key, the plaintexts or each other's inputs (decrypt: d_pt neither d_sk nor
 *      d_ct); an overlap is rejected with DPFHE_ERR_INVALID. ---- */
int dpfhe_random_seed(uint8_t seed[32]);
int dpfhe_secret_keygen(dpfhe_ctx *ctx, const uint8_t seed[32], uint64_t *d_sk, void *stream);
int dpfhe_relin_keygen(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32],
                       uint64_t *d_key, void *stream);
int dpfhe_galois_keygen(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, size_t n_elts,
                        const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *d_keys, void *stream);
int dpfhe_encrypt(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                  const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream);
int dpfhe_decrypt(dpfhe_ctx *ctx, const uint64_t *d_sk, const uint64_t *d_ct, unsigned n_comp, uint64_t *d_pt, size_t n,
                  void *stream);
int dpfhe_secret_keygen_host(dpfhe_ctx *ctx, const uint8_t seed[32], uint64_t *h_sk);
int dpfhe_relin_keygen_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32],
                            uint64_t *h_key);
int dpfhe_galois_keygen_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, size_t n_elts,
                             const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *h_keys);
int dpfhe_encrypt_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                       const uint64_t *h_pt, uint64_t *h_ct, size_t n);
int dpfhe_decrypt_host(dpfhe_ctx *ctx, const uint64_t *h_sk, const uint64_t *h_ct, unsigned n_comp, uint64_t *h_pt, size_t n);
int dpfhe_public_keygen(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t *d_pk, void *stream);
int dpfhe_encrypt_public(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_pk, const uint8_t seed[32], uint64_t first_index,
                         const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream);
int dpfhe_public_keygen_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t *h_pk);
int dpfhe_encrypt_public_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_pk, const uint8_t seed[32], uint64_t first_index,
                              const uint64_t *h_pt, uint64_t *h_ct, size_t n);

/* ---- synthetic data (DESIGN.md §5): x[k] = mulhi64(splitmix64(seed + k), q_limb),
 *      k = (first_poly + p)*L*N + l*N + n.  Fills [n_polys][L][N]. ---- */
int dpfhe_fill_uniform(dpfhe_ctx *ctx, uint64_t seed, uint64_t first_poly, uint64_t *d_data,
                       size_t n_polys, void *stream);

/* ---- host-buffer entry points (what a non-CUDA caller of the reference API would bind):
 *      H2D, compute and D2H are pipelined in chunks on the context's streams; synchronous. ---- */
int dpfhe_ntt_fwd_host(dpfhe_ctx *ctx, uint64_t *h_data, size_t n_polys);
int dpfhe_ntt_inv_host(dpfhe_ctx *ctx, uint64_t *h_data, size_t n_polys);
int dpfhe_ct_mul_relin_host(dpfhe_ctx *ctx, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk,
                            uint64_t *h_out, size_t batch);
int dpfhe_ct_mul_plain_host(dpfhe_ctx *ctx, const uint64_t *h_ct, const uint64_t *h_pt, uint64_t *h_out,
                            size_t batch);
int dpfhe_rotate_host(dpfhe_ctx *ctx, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk,
                      uint64_t *h_out, size_t batch);
/* pinned host memory helpers so callers can reach full PCIe bandwidth */
int dpfhe_host_alloc(void **out, size_t bytes);
/* the same, with the pages placed on the NUMA node of the context's GPU (what multi-GPU hosts need: DESIGN.md §7);
 * *placed_node (may be NULL) = that node, or -1 if the placement could not be enforced */
int dpfhe_host_alloc_near(const dpfhe_ctx *ctx, void **out, size_t bytes, int *placed_node);
int dpfhe_host_free(void *p);   /* frees memory of either allocator */
/* NUMA node of the context's GPU (-1: unknown), and a helper that restricts the CALLING thread to that node's CPUs */
int dpfhe_device_numa_node(const dpfhe_ctx *ctx, int *node);
int dpfhe_bind_thread_near(const dpfhe_ctx *ctx, int *n_cpus);

/* ---- device buffers other GPUs can write into.  The output of dpfhe_ct_mul_relin / dpfhe_keyswitch / dpfhe_rotate is
 *      written exactly once, by the kernel's final stores, so `d_out` may be memory of ANOTHER GPU: a peer-mapped
 *      buffer of the same process (dpfhe_multi_*), or, with one process per GPU, a buffer exported by the owning
 *      process and opened here.  That is how a multi-GPU job gathers its result while it computes. ---- */
#define DPFHE_IPC_HANDLE_BYTES 64
int dpfhe_device_alloc(dpfhe_ctx *ctx, void **d_out, size_t bytes);   /* a cudaMalloc of its own on the context's device */
int dpfhe_device_free(dpfhe_ctx *ctx, void *d_ptr);
int dpfhe_ipc_export(dpfhe_ctx *ctx, const void *d_ptr, unsigned char handle[DPFHE_IPC_HANDLE_BYTES]);
int dpfhe_ipc_open(dpfhe_ctx *ctx, const unsigned char handle[DPFHE_IPC_HANDLE_BYTES], void **d_out);
int dpfhe_ipc_close(dpfhe_ctx *ctx, void *d_ptr);

/* ---- several GPUs in one process (SURVEY.md §8e): one context per device, contiguous shards of the batch
 *      (the first batch % n shards hold one ciphertext more), no collective while computing.
 *      device_ids NULL = devices 0..n-1; n_devices <= 0 = all visible devices.  A device may be listed twice
 *      (two logical shards on one GPU).  Contrast with the reference's one-MPI-rank-per-GPU DistributedContext,
 *      src/core/distributed/distributed_context.cpp:242-250. ---- */
typedef struct dpfhe_multi dpfhe_multi;
int dpfhe_multi_create(const dpfhe_params *p, const int *device_ids, int n_devices, dpfhe_multi **out);
void dpfhe_multi_destroy(dpfhe_multi *m);
int dpfhe_multi_device_count(const dpfhe_multi *m);
dpfhe_ctx *dpfhe_multi_context(dpfhe_multi *m, int index);   /* borrowed: shard `index`'s context */
int dpfhe_multi_shard(const dpfhe_multi *m, size_t batch, int index, size_t *first, size_t *count);
/* host buffers [batch][2][L][N]: every device pipelines its own shard (H2D, compute, D2H) — no gather needed */
int dpfhe_multi_ct_mul_relin_host(dpfhe_multi *m, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk,
                                  uint64_t *h_out, size_t batch);
/* the special-prime form (dpfhe_ct_mul_relin_grouped_host) sharded the same way; ciphertexts carry L - n_special limbs */
int dpfhe_multi_ct_mul_relin_grouped_host(dpfhe_multi *m, unsigned n_special, const uint64_t *h_a, const uint64_t *h_b,
                                          const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain);
int dpfhe_multi_rotate_host(dpfhe_multi *m, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk,
                            uint64_t *h_out, size_t batch);
/* device buffers: d_a[r], d_b[r] = shard r of the operands and d_evk[r] = the key, all on device r; the whole result
 * [batch][2][L][N] is gathered on the device of shard `root` (d_out_root), written there directly by every device's
 * kernel through NVLink while it computes.  Synchronous. */
int dpfhe_multi_ct_mul_relin_gather(dpfhe_multi *m, const uint64_t *const *d_a, const uint64_t *const *d_b,
                                    const uint64_t *const *d_evk, uint64_t *d_out_root, int root, size_t batch);

/* ---- diagnostics ---- */
/* number of kernel launches issued through this context since creation */
uint64_t dpfhe_launch_count(const dpfhe_ctx *ctx);
/* per-phase clock64 totals of the fused key-switch kernel (summed over CTAs, then cleared); needs the
 * context to have been created with DPFHE_KS_PROF set in the environment.  out16: 16 words. */
int dpfhe_debug_phase_cycles(dpfhe_ctx *ctx, uint64_t *out16);
/* name + launch geometry of the kernels behind an op, for bench/DESIGN reporting; returns bytes written */
int dpfhe_describe(const dpfhe_ctx *ctx, char *buf, size_t buf_len);

#ifdef __cplusplus
}
#endif

/* the polynomial evaluators and the keyless calls at any level of the modulus chain (DESIGN.md §2.22) */
#include "dpfhe_level.h"
/* seeded ciphertexts and switch keys, their uniform half regenerated on the device from a public seed (DESIGN.md §2.23) */
#include "dpfhe_seeded.h"
/* compact result ciphertexts: switched to a power-of-two modulus and bit-packed on the device (DESIGN.md §2.24) */
#include "dpfhe_compact.h"

#endif /* DPFHE_H */
