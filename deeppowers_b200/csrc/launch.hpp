// launch.hpp — interface between the C ABI (abi.cu) and the kernel launchers (kernels.cu, compiled once per arithmetic
// variant: namespace dpfhe::gen for any moduli, dpfhe::fast for moduli of the form k * 2^32 + 1; types.hpp).
#pragma once
#include <cuda_runtime.h>

#include "types.hpp"

namespace dpfhe {

// device-resident state shared by all launches of one context
struct LaunchCtx {
    int device = 0;
    int num_sms = 0;
    u32 log_n = 0, L = 0;
    bool fast = false;                // every modulus is k * 2^32 + 1: launches go to the dpfhe::fast kernels
    bool lift_reduce = true;          // some modulus is at least twice another: digits are word-reduced when they change limb
    const LimbParams *lp = nullptr;   // [L] device copy (element-wise kernels)
    LimbTable lt;                     // host copy, passed by value to the transform kernels
    int rot_cfg = 0;                  // tuning variant of rot_apply_kernel (DPFHE_ROT_CFG)
    int ntt_cfg = 0;                  // tuning variant of the N=8192 transform kernel (DPFHE_NTT_CFG)
    int ntt_tma = 1;                  // inverse transforms (N <= 8192) fetch their limb with the TMA unit (DPFHE_NTT_TMA=0: thread copies)
    const Twiddle *tw = nullptr;      // [L][N] forward twiddles, device layout (ntt_core.cuh:tw_pos)
    const Twiddle *itw = nullptr;     // [L][N] inverse twiddles
    // fused key-switch pipeline
    u64 *ks_scratch = nullptr;        // [ks_slots][2][N] digit exchange buffers
    u64 *ks_acc = nullptr;            // N = 16384 only: [ks_slots][2][N] lazy accumulator rows of the resident work items (second half of ks_scratch's allocation)
    size_t ks_window_bytes = 0;       // bytes of ks_scratch (+ ks_acc) an L2 access-policy window may cover
    size_t l2_persist_max = 0;        // cudaDevAttrMaxPersistingL2CacheSize
    int l2_persist = 0;               // DPFHE_L2_PERSIST: 1 = mark the fused kernel's scratch as persisting in L2
    u64 *ks_acc_hyb = nullptr;        // hybrid key switching: [ks_slots][2 parities][2][N], allocated at the first hybrid call
    u32 *ks_flags = nullptr;          // [ks_slots] monotonically increasing round counters
    u32 *ks_consumed = nullptr;       // [ks_slots] monotone counters: readers of a single-buffered digit slot that have finished
    int ks_single = 0;                // tuning (DPFHE_KS_SINGLE=1): digit slots single-buffered with consumed counters instead of two per CTA
                                      // (by round parity)
    u32 *ks_ticket = nullptr;         // next ciphertext index (reset per launch)
    u64 *ks_mail = nullptr;           // [ks_slots] per-group mailbox: (round tag << 32) | ciphertext index
    u64 *ks_key_s = nullptr;          // [L][2][L][N] Shoup companions of the current switch key
    u64 *ks_hyb = nullptr;            // hybrid key switching: [ks_slots / 2 + 1][KS_HYB_ROWS][N], allocated at the first hybrid call
    u64 *ks_tau_drop = nullptr;       // multiply-and-rescale: [ks_slots / 3 + 1][2 parities][2][N] rows of the dropped limb, allocated at the first such call
    size_t ks_slots = 0;
    u32 ks_epoch = 0;                 // rounds consumed so far (flag values already used)
    unsigned long long ks_epoch_limit = 1ull << 30;   // the round numbering restarts before it gets here (DPFHE_EPOCH_LIMIT: tests)
    unsigned ks_epoch_restarts = 0;
    int ks_prefetch = 0;              // ciphertexts ahead for the bulk L2 prefetch of inputs (DPFHE_KS_PF), 0 = off
    int ks_occ_cap = 0;               // tuning: cap on resident fused-kernel CTAs per SM (DPFHE_KS_OCC), 0 = no cap
    unsigned long long *ks_prof = nullptr;   // [ks_slots][16] phase cycle counters; non-null selects the profiling build
};

// the launchers, declared once per variant namespace
#define DPFHE_DECLARE_LAUNCHERS \
    cudaError_t launch_ntt(const LaunchCtx &lc, u64 *data, size_t n_polys, bool inverse, cudaStream_t st); \
    cudaError_t launch_ks(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch, \
                          u32 galois, cudaStream_t st, const u32 *only = nullptr, bool key_ready = false, const u64 *key_s = nullptr); \
    cudaError_t launch_hoist(LaunchCtx &lc, const u64 *ct, u64 *U, u32 *zero, size_t batch, cudaStream_t st); \
    cudaError_t launch_rot_prepare(LaunchCtx &lc, const u64 *key, u32 galois, const u64 *delta, u64 *M, u64 *kprime, cudaStream_t st, \
                                   u64 *key_s_out = nullptr); \
    cudaError_t launch_rot_apply(const LaunchCtx &lc, const u64 *ct, const u64 *U, const u64 *key, const u64 *kprime, u32 galois, u64 *out, \
                                 size_t batch, cudaStream_t st, const u64 *key_s = nullptr); \
    cudaError_t launch_ks_hybrid(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch, u32 galois, \
                                 const MsConsts &K, cudaStream_t st, const u64 *key_s = nullptr, u32 key_L = 0); \
    cudaError_t launch_ks_grouped(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch, u32 galois, \
                                  const MsConsts &K, const GroupConsts &G, cudaStream_t st, const u64 *addend = nullptr, \
                                  const u64 *key_s = nullptr); \
    cudaError_t launch_ct_dot_grouped(LaunchCtx &lc, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, u64 *out, size_t batch, \
                                      const MsConsts &K, const GroupConsts &G, cudaStream_t st, const u64 *key_s = nullptr); \
    cudaError_t launch_ks_rescale_grouped(LaunchCtx &lc, bool dot, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, \
                                          u64 *out, size_t batch, const MsConsts &K, const GroupConsts &G, const RescaleConsts &R, \
                                          cudaStream_t st, const u64 *key_s = nullptr); \
    cudaError_t launch_hoist_grouped(LaunchCtx &lc, const u64 *ct, u64 *U, const GroupConsts &G, size_t batch, cudaStream_t st); \
    cudaError_t launch_key_prepare(const LaunchCtx &lc, const u64 *key, u64 *key_s, u32 rows, cudaStream_t st); \
    cudaError_t launch_rot_apply_grouped(LaunchCtx &lc, const u64 *ct, const u64 *U, const u64 *key, const u64 *key_s, u32 galois, u64 *acc, \
                                         const MsConsts &K, const GroupConsts &G, size_t batch, cudaStream_t st, u32 key_shift = 0); \
    cudaError_t launch_rot_sum_grouped(const LaunchCtx &lc, const u64 *ct, const u64 *U, u32 n_rot, const u64 *const *keys, \
                                       const u64 *const *key_s, const u32 *galois, u64 *acc, const MsConsts &K, const GroupConsts &G, \
                                       size_t batch, cudaStream_t st, u32 key_shift = 0); \
    cudaError_t launch_ks_grouped_level(LaunchCtx &lc, int mode, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, \
                                        const u64 *key_s, u32 key_L, u64 *out, size_t batch, u32 galois, const MsConsts &K, \
                                        const GroupConsts &G, const RescaleConsts *R, cudaStream_t st, const u64 *addend = nullptr); \
    cudaError_t launch_pt_inner(const LaunchCtx &lc, const u64 *steps, u32 nb, const u64 *pts, u32 ng, u64 *out, size_t batch, cudaStream_t st, \
                                unsigned *launches); \
    cudaError_t launch_pointwise_mul(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *out, size_t n_polys, cudaStream_t st); \
    cudaError_t launch_mod_switch(const LaunchCtx &lc, const u64 *in, u64 *tau, u64 *out, const MsConsts &K, size_t n_polys, cudaStream_t st); \
    cudaError_t launch_mod_down_special(const LaunchCtx &lc, const u64 *in, u64 *tau, u64 *out, const MsConsts &K, const GroupConsts &G, size_t n_polys, \
                                        cudaStream_t st); \
    cudaError_t launch_poly_add(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *out, size_t n_polys, cudaStream_t st); \
    cudaError_t launch_ct_mul_plain(const LaunchCtx &lc, const u64 *ct, const u64 *pt, u64 *out, size_t batch, cudaStream_t st); \
    cudaError_t launch_ct_mul_plain_acc(const LaunchCtx &lc, const u64 *ct, const u64 *pt, u64 *acc, size_t batch, cudaStream_t st); \
    cudaError_t launch_ct_tensor(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *d, size_t batch, cudaStream_t st); \
    cudaError_t launch_fill_uniform(const LaunchCtx &lc, u64 seed, u64 first_poly, u64 *data, size_t n_polys, cudaStream_t st); \
    cudaError_t launch_ckks_encode(const LaunchCtx &lc, const Cplx *slots, double *coeffs, u64 *pt, const CkksTables &T, double sc, size_t n_vec, \
                                   cudaStream_t st); \
    cudaError_t launch_ckks_decode(const LaunchCtx &lc, u64 *work, Cplx *slots, const CkksTables &T, const CkksConsts &K, size_t n_vec, \
                                   cudaStream_t st); \
    cudaError_t launch_bgv_encode(const LaunchCtx &lc, const int64_t *slots, u32 *coeffs, u64 *pt, const BgvTables &T, size_t n_vec, \
                                  cudaStream_t st); \
    cudaError_t launch_bgv_decode(const LaunchCtx &lc, u64 *work, u64 *slots, const BgvTables &T, const BgvConsts &K, size_t n_vec, \
                                  cudaStream_t st); \
    cudaError_t launch_keys(const LaunchCtx &lc, int mode, const KeyArgs &A, size_t n_items, cudaStream_t st); \
    cudaError_t launch_decrypt(const LaunchCtx &lc, const u64 *ct, const u64 *s, u64 *pt, u32 n_comp, size_t n, cudaStream_t st); \
    cudaError_t launch_expand_seeded(const LaunchCtx &lc, bool keys, const SeededKeyArgs &A, const u64 *src, u64 *dst, size_t n_rows, cudaStream_t st); \
    cudaError_t launch_compact_pack(const LaunchCtx &lc, const CompactArgs &A, const u64 *x, u64 *out, size_t n_polys, cudaStream_t st); \
    cudaError_t launch_compact_unpack(const LaunchCtx &lc, bool finish, const CompactArgs &A, const u64 *cct, const u64 *prod, u64 *dst, size_t n, \
                                      cudaStream_t st); \
    cudaError_t launch_lincomb(const LaunchCtx &lc, const u64 *const *in, const int64_t *coeffs, u32 n_terms, int64_t constant, const u64 *pt, \
                               u64 *out, size_t batch, cudaStream_t st); \
    cudaError_t launch_ckks_comb(const LaunchCtx &lc, const u64 *const *in, const u32 *levels, const double *coeffs, u32 n_terms, \
                                 double constant, const MsConsts &K, u64 *tau, u64 *out, size_t batch, cudaStream_t st);

namespace gen {
DPFHE_DECLARE_LAUNCHERS
}
namespace fast {
DPFHE_DECLARE_LAUNCHERS
}
#undef DPFHE_DECLARE_LAUNCHERS
// launch_ks: `only` = optional [batch] filter (non-zero = process); key_ready: the key's Shoup companions are already in key_s
// (or, with key_s == nullptr, in lc.ks_key_s).  launch_rot_prepare / launch_rot_apply: key_s(_out) == nullptr means lc.ks_key_s.
// launch_ks_grouped: key_s == nullptr builds the companions into lc.ks_key_s (two launches), otherwise one launch; addend (KS_ROTATE
// only) is added to the result in the kernel's final store.
// launch_ct_dot_grouped: a[t] / b[t] of n_terms (1 .. DOT_MAX_TERMS) pairs, host arrays of device pointers; key_s as launch_ks_grouped.
// launch_ks_rescale_grouped: dot = false: a[0] x b[0] (n_terms = 1), dot = true: the pairs as launch_ct_dot_grouped; key_s as
// launch_ks_grouped.
// launch_rot_sum_grouped: keys[m] / key_s[m] / galois[m] of n_rot (1 .. ROT_SUM_MAX) rotations; the companions are required;
// key_shift > 0: lc is a level view and the keys are top-level keys (DESIGN.md §4.17).
// launch_rot_apply_grouped: key_shift > 0 as launch_rot_sum_grouped's, the companions then required (DESIGN.md §4.18).
// launch_ks_hybrid with key_s / launch_ks_grouped_level: the calls at level l on the level's view lc (DESIGN.md §2.20, §4.17), reading
// the top-level key (key_L limbs per row) and its companions key_s, which the caller builds with the context's own launch state;
// launch_ks_grouped_level's addend (KS_ROTATE only) as launch_ks_grouped's: the fused Horner step of a layer at level l (§4.18).
// launch_key_prepare: the Shoup companions of the first `rows` rows [rows][2][L][N] of a switch key into key_s (same layout).

}  // namespace dpfhe
