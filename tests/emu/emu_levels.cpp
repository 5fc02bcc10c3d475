// emu_levels.cpp — host emulator of the level calls' kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs the key-switch programs of a level view (DESIGN.md §2.20, §4.17) on the host with a sequential CTA policy: the grouped program
// of ks_level_grouped_kernel (ks_phase1 in mode KS_MUL_RELIN or KS_DOT, ks_phase2_group, ms_tau_body, ms_limb_group; divided by P, or
// by P * q_{l-1} with the dropped limb's row), the one-special-prime program of ks_hybrid_level_kernel (ks_phase1, ks_phase2_digit,
// ms_limb_body) and the summed rotations' rows (rot_sum_grouped_rows).  Each runs with LV = true on a top-level key (key_L rows per
// (digit, component), the special rows key_L - L further down) or with LV = false on a key of the view's own layout, so that the tests
// can hold the first to the second on restrict_key(...) bit for bit.  The Shoup companions are built here from the key and the moduli of
// its rows, as key_prepare_kernel builds them.  Built by tests/test_levels_emu_cpu.py once per arithmetic variant; never linked into
// libdpfhe.so.
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
    bool lift_reduce = false;
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

// The grouped program (ks_grouped_body) in role order for one ciphertext after another: every limb CTA's phase 1, the foreign digits,
// the special CTAs (and with the rescale the dropped limb's CTA), then the division.  out [batch][2][l - rs][N].
template <int LOGN, int NT, bool LV>
void run_grouped(Ctx &e, unsigned Ks, bool dot, bool rs, const DotArgs &D, const uint64_t *key, const uint64_t *key_s, unsigned key_L, uint64_t *out,
                 size_t batch, uint64_t t_plain) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned LK = e.hp.L, Lq = LK - Ks, d = Lq - 1;
    MsConsts K;
    GroupConsts Gc;
    RescaleConsts R;
    if (rs) build_rescale_consts(e.hp, Ks, t_plain, Gc, K, R);
    else build_group_consts(e.hp, Ks, t_plain, Gc, K);
    const unsigned dnum = Gc.dnum;
    uint64_t *buf = aligned_new<uint64_t>(N), *scratch = aligned_new<uint64_t>((size_t)LK * N), *hyb_all = aligned_new<uint64_t>((size_t)Ks * KS_HYB_ROWS * N),
             *drop = aligned_new<uint64_t>(2 * N), *acc = aligned_new<uint64_t>((size_t)LK * 2 * N);
    KsArgs A;
    A.a = dot ? nullptr : D.a[0]; A.b = dot ? nullptr : D.b[0]; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = Lq; A.galois = 0; A.Lk = key_L; A.hyb = hyb_all; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = 0;
    HostCta cta{NT};
    const size_t P = (size_t)(Lq - (rs ? 1 : 0)) * N;
    for (size_t ct = 0; ct < batch; ++ct) {
        auto hyb_of = [&](unsigned k) { return hyb_all + (size_t)k * KS_HYB_ROWS * N; };
        for (unsigned i = 0; i < Lq; ++i) {
            if (dot)
                ks_phase1<LOGN, NT, KS_DOT, true, LV>(cta, buf, A, Gc.lp_up[i], ct, i, scratch + (size_t)i * N, acc + (size_t)i * 2 * N, K.qlm[i],
                                                      K.qlm_s[i], nullptr, 0, i / Ks, &D, key_L - LK);
            else
                ks_phase1<LOGN, NT, KS_MUL_RELIN, true, LV>(cta, buf, A, Gc.lp_up[i], ct, i, scratch + (size_t)i * N, acc + (size_t)i * 2 * N,
                                                            K.qlm[i], K.qlm_s[i], nullptr, 0, i / Ks, nullptr, key_L - LK);
        }
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
        if (rs)
            for (unsigned c = 0; c < 2; ++c)
                ms_tau_body<LOGN, NT, true>(cta, buf, acc + ((size_t)d * 2 + c) * N, acc + ((size_t)d * 2 + c) * N, A.itw + (size_t)d * N, R.lp_drop,
                                            drop + c * N, K);
        for (unsigned i = 0; i < Lq - (rs ? 1 : 0); ++i)
            for (unsigned c = 0; c < 2; ++c) {
                u64 *row = out + ct * 2 * P + c * P + (size_t)i * N;
                if (rs)
                    ms_limb_group<LOGN, NT, true, false, true>(cta, buf, hyb_of(0) + ks_hyb_tau_row(0, c) * N, (size_t)KS_HYB_ROWS * N,
                                                               acc + ((size_t)i * 2 + c) * N, row, A.tw + (size_t)i * N, e.lp[i], K, Gc, i, nullptr,
                                                               drop + c * N, &R);
                else
                    ms_limb_group<LOGN, NT, true, false>(cta, buf, hyb_of(0) + ks_hyb_tau_row(0, c) * N, (size_t)KS_HYB_ROWS * N,
                                                         acc + ((size_t)i * 2 + c) * N, row, A.tw + (size_t)i * N, e.lp[i], K, Gc, i);
            }
    }
    free(buf); free(scratch); free(hyb_all); free(drop); free(acc);
}

// the one-special-prime program (ks_hybrid_body), mode KS_MUL_RELIN (a, b) or KS_ROTATE (a, galois); out [batch][2][l][N]
template <int LOGN, int NT, bool LV>
void run_hybrid(Ctx &e, int mode, const uint64_t *a, const uint64_t *b, uint32_t galois, const uint64_t *key, const uint64_t *key_s, unsigned key_L,
                uint64_t *out, size_t batch, uint64_t t_plain) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned L = e.hp.L - 1;
    MsConsts K;
    build_ms_consts(e.hp, t_plain, K);
    uint64_t *buf = aligned_new<uint64_t>(N), *scratch = aligned_new<uint64_t>((size_t)L * N), *hyb = aligned_new<uint64_t>((size_t)KS_HYB_ROWS * N),
             *acc = aligned_new<uint64_t>((size_t)L * 2 * N);
    KsArgs A;
    A.a = a; A.b = b; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = L; A.galois = galois; A.Lk = key_L; A.hyb = hyb; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = e.lift_reduce ? 1u : 0u;
    HostCta cta{NT};
    const size_t P = (size_t)L * N;
    for (size_t ct = 0; ct < batch; ++ct) {
        for (unsigned i = 0; i < L; ++i) {
            if (mode == KS_MUL_RELIN)
                ks_phase1<LOGN, NT, KS_MUL_RELIN, true, LV>(cta, buf, A, e.lp[i], ct, i, scratch + (size_t)i * N, acc + (size_t)i * 2 * N, K.qlm[i], K.qlm_s[i],
                                                            nullptr, 0, ~0u, nullptr, key_L - e.hp.L);
            else
                ks_phase1<LOGN, NT, KS_ROTATE, true, LV>(cta, buf, A, e.lp[i], ct, i, scratch + (size_t)i * N, acc + (size_t)i * 2 * N, K.qlm[i], K.qlm_s[i],
                                                         nullptr, 0, ~0u, nullptr, key_L - e.hp.L);
        }
        for (unsigned i = 0; i < L; ++i)
            for (uint32_t jj = 1; jj < L; ++jj) {
                const uint32_t j = (i + jj) % L;
                ks_phase2_digit<LOGN, NT, true, false, LV>(cta, buf, A, e.lp[i], ct, i, j, jj, scratch + (size_t)j * N, acc + (size_t)i * 2 * N,
                                                           key_L - e.hp.L);
            }
        for (uint32_t jj = 0; jj < L; ++jj)
            ks_phase2_digit<LOGN, NT, true, true, LV>(cta, buf, A, e.lp[L], ct, L, jj, jj, scratch + (size_t)jj * N, hyb, key_L - e.hp.L);
        for (unsigned c = 0; c < 2; ++c)
            ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)L * N, e.lp[L], hyb + ks_hyb_tau_row(0, c) * N, K);
        for (unsigned i = 0; i < L; ++i)
            for (unsigned c = 0; c < 2; ++c)
                ms_limb_body<LOGN, NT, true>(cta, buf, hyb + ks_hyb_tau_row(0, c) * N, acc + ((size_t)i * 2 + c) * N, out + ct * 2 * P + c * P + (size_t)i * N,
                                             A.tw + (size_t)i * N, e.lp[i], K, i);
    }
    free(buf); free(scratch); free(hyb); free(acc);
}

// the summed rotations' accumulator rows (rot_sum_grouped_rows) over every limb of the view, one ciphertext per work item
template <int LOGN, int NT, bool LV>
void run_rot_sum(Ctx &e, unsigned Ks, const uint64_t *ct, const uint64_t *U, unsigned n_rot, const uint64_t *keys, const uint64_t *keys_s,
                 const uint32_t *galois, unsigned key_L, size_t key_words, uint64_t *acc, size_t batch, uint64_t t_plain) {
    MsConsts K;
    GroupConsts Gc;
    build_group_consts(e.hp, Ks, t_plain, Gc, K);
    RotSumGArgs A;
    memset(&A, 0, sizeof(A));
    A.ct = ct; A.U = U; A.acc = acc; A.n_rot = n_rot;
    for (unsigned m = 0; m < n_rot; ++m) {
        A.key[m] = keys + m * key_words;
        A.key_s[m] = keys_s + m * key_words;
        A.galois[m] = galois[m];
    }
    HostCta cta{NT};
    for (size_t c0 = 0; c0 < batch; ++c0)
        for (unsigned i = 0; i < e.hp.L; ++i)
            rot_sum_grouped_rows<LOGN, NT, 1, LV>(cta, A, Gc, K, e.lp[i], c0, 1, i, 0, 1 << (LOGN - 1), key_L - e.hp.L);
}

bool dot_args(DotArgs &D, const uint64_t *pool, size_t ct_words, size_t batch, unsigned n_pool, unsigned n_terms, const uint32_t *ia, const uint32_t *ib) {
    if (n_terms < 1 || n_terms > (unsigned)DOT_MAX_TERMS) return false;
    memset(&D, 0, sizeof(D));
    D.n_terms = n_terms;
    for (unsigned t = 0; t < n_terms; ++t) {
        if (ia[t] >= n_pool || ib[t] >= n_pool) return false;
        D.a[t] = pool + (size_t)ia[t] * batch * ct_words;
        D.b[t] = pool + (size_t)ib[t] * batch * ct_words;
    }
    return true;
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
void *emu_lv_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
    Ctx *e = new Ctx();
    if (!build_host_params(log_n, L, moduli, e->hp).empty()) {
        delete e;
        return nullptr;
    }
    uint64_t qmin = ~0ull, qmax = 0;
    for (unsigned l = 0; l < L; ++l) {
#if DPFHE_FAST
        if (e->hp.limbs[l].lp.nqh == 0) {   // the fast bodies are only valid for moduli k * 2^32 + 1
            delete e;
            return nullptr;
        }
#endif
        qmin = std::min<uint64_t>(qmin, moduli[l]);
        qmax = std::max<uint64_t>(qmax, moduli[l]);
    }
    e->lift_reduce = !(qmax < 2 * qmin);   // as upload_basis picks it
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
void emu_lv_destroy(void *h) { delete (Ctx *)h; }

// The grouped program with K special primes: pool [n_pool][batch][2][l][N], pair t = (pool[ia[t]], pool[ib[t]]); dot = 0: phase 1 in mode
// KS_MUL_RELIN (one pair); rs = 1: divided by P * q_{l-1}, out [batch][2][l-1][N], else [batch][2][l][N].  key: dnum digits of key_L rows
// whose moduli are key_mods; lv = 1 reads it through the level map (key_L > l + K), lv = 0 as the view's own key (key_L = l + K).
int emu_lv_grouped(void *h, unsigned K, int dot, int rs, int lv, const uint64_t *pool, unsigned n_pool, unsigned n_terms, const uint32_t *ia,
                   const uint32_t *ib, const uint64_t *key, unsigned key_L, const uint64_t *key_mods, uint64_t *out, size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    const unsigned L = e->hp.L;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > L || (rs && L - K < 2) || (!dot && n_terms != 1) || key_L < L || (!lv && key_L != L)) return -1;
    DotArgs D;
    if (!dot_args(D, pool, (size_t)2 * (L - K) << e->hp.log_n, batch, n_pool, n_terms, ia, ib)) return -1;
    const size_t N = (size_t)1 << e->hp.log_n, dnum = (L - K + K - 1) / K;
    const std::vector<uint64_t> ks = companions(key, dnum * 2 * key_L * N, key_mods, key_L, N);
#define GRP(LOGN)                                                                                                          \
    if (lv) run_grouped<LOGN, 256, true>(*e, K, dot != 0, rs != 0, D, key, ks.data(), key_L, out, batch, t_plain);           \
    else run_grouped<LOGN, 256, false>(*e, K, dot != 0, rs != 0, D, key, ks.data(), key_L, out, batch, t_plain)
    EMU_DISPATCH(GRP)
#undef GRP
}

// the one-special-prime program: mode 0 = ct x ct (a, b [batch][2][l][N]), 1 = rotation of a by galois; key [l][2][key_L][N]
int emu_lv_hybrid(void *h, int rotate, int lv, const uint64_t *a, const uint64_t *b, uint32_t galois, const uint64_t *key, unsigned key_L,
                  const uint64_t *key_mods, uint64_t *out, size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    const unsigned L = e->hp.L;
    if (L < 2 || key_L < L || (!lv && key_L != L)) return -1;
    const size_t N = (size_t)1 << e->hp.log_n;
    const std::vector<uint64_t> ks = companions(key, (size_t)(L - 1) * 2 * key_L * N, key_mods, key_L, N);
    const int mode = rotate ? KS_ROTATE : KS_MUL_RELIN;
#define HYB(LOGN)                                                                                                   \
    if (lv) run_hybrid<LOGN, 256, true>(*e, mode, a, b, galois, key, ks.data(), key_L, out, batch, t_plain);          \
    else run_hybrid<LOGN, 256, false>(*e, mode, a, b, galois, key, ks.data(), key_L, out, batch, t_plain)
    EMU_DISPATCH(HYB)
#undef HYB
}

// the summed rotations' rows: ct [batch][2][l][N], U [batch][dnum][l+K][N], keys [n_rot][dnum][2][key_L][N] (dnum = ceil(l / K), the
// digits the level reads) -> acc [batch][2][l+K][N]
int emu_lv_rot_sum(void *h, unsigned K, int lv, const uint64_t *ct, const uint64_t *U, unsigned n_rot, const uint64_t *keys, const uint32_t *galois,
                   unsigned key_L, const uint64_t *key_mods, uint64_t *acc, size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    const unsigned L = e->hp.L;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > L || n_rot < 1 || n_rot > (unsigned)ROT_SUM_MAX || key_L < L || (!lv && key_L != L)) return -1;
    const size_t N = (size_t)1 << e->hp.log_n, dnum = (L - K + K - 1) / K, key_words = dnum * 2 * key_L * N;
    const std::vector<uint64_t> ks = companions(keys, n_rot * key_words, key_mods, key_L, N);
#define ROT(LOGN)                                                                                                            \
    if (lv) run_rot_sum<LOGN, 256, true>(*e, K, ct, U, n_rot, keys, ks.data(), galois, key_L, key_words, acc, batch, t_plain);  \
    else run_rot_sum<LOGN, 256, false>(*e, K, ct, U, n_rot, keys, ks.data(), galois, key_L, key_words, acc, batch, t_plain)
    EMU_DISPATCH(ROT)
#undef ROT
}
}
