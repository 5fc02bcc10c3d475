// emu_level_layer.cpp — host emulator of the level layer's kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs the two programs a linear layer needs at level l (DESIGN.md §2.21, §4.18) on the host with a sequential CTA policy: the hoisted
// multiply-accumulate of rot_apply_grouped_level_kernel (rot_apply_grouped_rows, one ciphertext per work item) and the fused Horner
// step of ks_level_horner_kernel (the grouped program of ks_grouped_body in mode KS_ROTATE with the addend: ks_phase1,
// ks_phase2_group, ms_tau_body, ms_limb_group with ADD).  Each runs with LV = true on a top-level key (key_L rows per (digit, component),
// the special rows key_L - L further down) or with LV = false on a key of the view's own layout, so that the tests can hold the first
// to the second on restrict_key(...) bit for bit.  The Shoup companions are built here from the key and the moduli of its rows, as
// key_prepare_kernel builds them.  Built by tests/test_level_layer_emu_cpu.py once per arithmetic variant; never linked into libdpfhe.so.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "host_params.hpp"
#include "kernel_bodies.cuh"

using namespace dpfhe;
using namespace dpfhe::DPFHE_VNS;   // built once per arithmetic variant (-DDPFHE_FAST=0 / 1)

namespace {
struct HostCta {
    int nt;
    template <class F>
    void par(F f) {
        for (int t = 0; t < nt; ++t) f(t);
    }
    template <class F>
    void par_dom(F f) { par(f); }
    template <class F>
    void par_warp(F f) { par(f); }
    void mark(int) {}
    void wait_ge(const uint32_t *, uint32_t) {}
};

template <class T>
T *aligned_new(size_t n) {
    void *p = nullptr;
    if (posix_memalign(&p, 128, n * sizeof(T))) return nullptr;
    return (T *)p;
}

// the view's basis {q_0 .. q_{l-1}, p_0 .. p_{K-1}}: its parameters and tables
struct Ctx {
    HostParams hp;
    std::vector<LimbParams> lp;
    Twiddle *tw = nullptr, *itw = nullptr;
    ~Ctx() {
        free(tw);
        free(itw);
    }
};

// the key's Shoup companions: row r of every (digit, component) against key_mods[r], key_L rows each
std::vector<uint64_t> companions(const uint64_t *key, size_t words, const uint64_t *key_mods, unsigned key_L, size_t N) {
    std::vector<uint64_t> ks(words);
    for (size_t k = 0; k < words; ++k) ks[k] = (uint64_t)((((unsigned __int128)key[k]) << 64) / key_mods[(k / N) % key_L]);
    return ks;
}

// the hoisted multiply-accumulate over every limb of the view in blocks of CB ciphertexts (the last one short when the batch does not
// divide): CB = 1 is the work split of rot_apply_grouped_level_kernel, CB = 2 that of rot_apply_grouped_kernel
template <int LOGN, int NT, int CB, bool LV>
void run_rot_apply(Ctx &e, unsigned Ks, const uint64_t *ct, const uint64_t *U, const uint64_t *key, const uint64_t *key_s, uint32_t galois,
                   unsigned key_L, uint64_t *acc, size_t batch, uint64_t t_plain) {
    MsConsts K;
    GroupConsts Gc;
    build_group_consts(e.hp, Ks, t_plain, Gc, K);
    RotApplyGArgs A;
    A.ct = ct; A.U = U; A.key = key; A.key_s = key_s; A.acc = acc; A.galois = galois;
    HostCta cta{NT};
    for (size_t c0 = 0; c0 < batch; c0 += CB) {
        const uint32_t n_ct = batch - c0 < (size_t)CB ? (uint32_t)(batch - c0) : (uint32_t)CB;
        for (unsigned i = 0; i < e.hp.L; ++i)
            rot_apply_grouped_rows<LOGN, NT, CB, LV>(cta, A, Gc, K, e.lp[i], c0, n_ct, i, 0, 1 << (LOGN - 1), key_L - e.hp.L);
    }
}

// The grouped program in mode KS_ROTATE with the addend (ks_grouped_body<..., KS_ROTATE, ADD = true, RS = false, LV>) in role order for
// one ciphertext after another: every limb CTA's phase 1, the foreign digits, the special CTAs, then the division and the addition.
// a, addend, out [batch][2][l][N].
template <int LOGN, int NT, bool LV>
void run_horner(Ctx &e, unsigned Ks, const uint64_t *a, const uint64_t *addend, uint32_t galois, const uint64_t *key, const uint64_t *key_s,
                unsigned key_L, uint64_t *out, size_t batch, uint64_t t_plain) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned LK = e.hp.L, Lq = LK - Ks;
    MsConsts K;
    GroupConsts Gc;
    build_group_consts(e.hp, Ks, t_plain, Gc, K);
    const unsigned dnum = Gc.dnum;
    uint64_t *buf = aligned_new<uint64_t>(N), *scratch = aligned_new<uint64_t>((size_t)LK * N), *hyb_all = aligned_new<uint64_t>((size_t)Ks * KS_HYB_ROWS * N),
             *acc = aligned_new<uint64_t>((size_t)LK * 2 * N);
    KsArgs A;
    A.a = a; A.b = nullptr; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = Lq; A.galois = galois; A.Lk = key_L; A.hyb = hyb_all; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = 0;
    HostCta cta{NT};
    const size_t P = (size_t)Lq * N;   // the body's addend and output row stride: the view's ciphertext size
    auto hyb_of = [&](unsigned k) { return hyb_all + (size_t)k * KS_HYB_ROWS * N; };
    for (size_t ct = 0; ct < batch; ++ct) {
        for (unsigned i = 0; i < Lq; ++i)
            ks_phase1<LOGN, NT, KS_ROTATE, true, LV>(cta, buf, A, Gc.lp_up[i], ct, i, scratch + (size_t)i * N, acc + (size_t)i * 2 * N, K.qlm[i],
                                                     K.qlm_s[i], nullptr, 0, i / Ks, nullptr, key_L - LK);
        for (unsigned i = 0; i < Lq; ++i)
            for (uint32_t jj = 1; jj < dnum; ++jj)
                ks_phase2_group<LOGN, NT, false, LV>(cta, buf, A, Gc, e.lp[i], ct, i, (i / Ks + jj) % dnum, jj, scratch, N, acc + (size_t)i * 2 * N,
                                                     key_L - LK);
        for (unsigned k = 0; k < Ks; ++k) {
            const unsigned i = Lq + k;
            uint64_t *hyb = hyb_of(k);
            for (uint32_t jj = 0; jj < dnum; ++jj) ks_phase2_group<LOGN, NT, true, LV>(cta, buf, A, Gc, e.lp[i], ct, i, jj, jj, scratch, N, hyb, key_L - LK);
            for (unsigned c = 0; c < 2; ++c)
                ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)i * N, Gc.lp_up[i], hyb + ks_hyb_tau_row(0, c) * N, K);
        }
        for (unsigned i = 0; i < Lq; ++i)
            for (unsigned c = 0; c < 2; ++c)
                ms_limb_group<LOGN, NT, true, true>(cta, buf, hyb_of(0) + ks_hyb_tau_row(0, c) * N, (size_t)KS_HYB_ROWS * N, acc + ((size_t)i * 2 + c) * N,
                                                    out + ct * 2 * P + c * P + (size_t)i * N, A.tw + (size_t)i * N, e.lp[i], K, Gc, i,
                                                    addend + ct * 2 * P + c * P + (size_t)i * N);
    }
    free(buf); free(scratch); free(hyb_all); free(acc);
}
}  // namespace

#define EMU_DISPATCH(CALL)                 \
    switch (e->hp.log_n) {                 \
        case 12: CALL(12); return 0;       \
        case 13: CALL(13); return 0;       \
        case 14: CALL(14); return 0;       \
    }                                      \
    return -1;

extern "C" {

// the view's basis (l + K moduli: the ciphertext moduli, then the special primes)
void *emu_ll_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
    Ctx *e = new Ctx();
    if (!build_host_params(log_n, L, moduli, e->hp).empty()) {
        delete e;
        return nullptr;
    }
#if DPFHE_FAST
    for (unsigned l = 0; l < L; ++l)
        if (e->hp.limbs[l].lp.nqh == 0) {   // the fast bodies are only valid for moduli k * 2^32 + 1
            delete e;
            return nullptr;
        }
#endif
    const size_t N = (size_t)1 << log_n;
    e->tw = aligned_new<Twiddle>(N * L);
    e->itw = aligned_new<Twiddle>(N * L);
    for (unsigned l = 0; l < L; ++l) {
        e->lp.push_back(e->hp.limbs[l].lp);
        memcpy(e->tw + l * N, e->hp.limbs[l].tw.data(), N * sizeof(Twiddle));
        memcpy(e->itw + l * N, e->hp.limbs[l].itw.data(), N * sizeof(Twiddle));
    }
    return e;
}
void emu_ll_destroy(void *h) { delete (Ctx *)h; }

// the hoisted multiply-accumulate of one rotation: ct [batch][2][l][N], U [batch][dnum][l+K][N], key [dnum][2][key_L][N] (dnum =
// ceil(l / K), the digits the level reads) -> acc [batch][2][l+K][N].  lv = 1 reads the key through the level map (key_L > l + K), one
// ciphertext per work item as the level kernel does; lv = 0 as the view's own key (key_L = l + K), two per work item as the top-level
// kernel does on a level context.
int emu_ll_rot_apply(void *h, unsigned K, int lv, const uint64_t *ct, const uint64_t *U, const uint64_t *key, uint32_t galois, unsigned key_L,
                     const uint64_t *key_mods, uint64_t *acc, size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    const unsigned L = e->hp.L;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > L || key_L < L || (!lv && key_L != L)) return -1;
    const size_t N = (size_t)1 << e->hp.log_n, dnum = (L - K + K - 1) / K;
    const std::vector<uint64_t> ks = companions(key, dnum * 2 * key_L * N, key_mods, key_L, N);
#define APPLY(LOGN)                                                                                              \
    if (lv) run_rot_apply<LOGN, 256, 1, true>(*e, K, ct, U, key, ks.data(), galois, key_L, acc, batch, t_plain);   \
    else run_rot_apply<LOGN, 256, 2, false>(*e, K, ct, U, key, ks.data(), galois, key_L, acc, batch, t_plain)
    EMU_DISPATCH(APPLY)
#undef APPLY
}

// the fused Horner step: out = rotation of a by galois + addend, a / addend / out [batch][2][l][N]; key as emu_ll_rot_apply's
int emu_ll_horner(void *h, unsigned K, int lv, const uint64_t *a, const uint64_t *addend, uint32_t galois, const uint64_t *key, unsigned key_L,
                  const uint64_t *key_mods, uint64_t *out, size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    const unsigned L = e->hp.L;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > L || key_L < L || (!lv && key_L != L)) return -1;
    const size_t N = (size_t)1 << e->hp.log_n, dnum = (L - K + K - 1) / K;
    const std::vector<uint64_t> ks = companions(key, dnum * 2 * key_L * N, key_mods, key_L, N);
#define HORNER(LOGN)                                                                                               \
    if (lv) run_horner<LOGN, 256, true>(*e, K, a, addend, galois, key, ks.data(), key_L, out, batch, t_plain);       \
    else run_horner<LOGN, 256, false>(*e, K, a, addend, galois, key, ks.data(), key_L, out, batch, t_plain)
    EMU_DISPATCH(HORNER)
#undef HORNER
}
}
