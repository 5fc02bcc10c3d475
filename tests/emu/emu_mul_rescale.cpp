// emu_mul_rescale.cpp — host emulator of multiply-and-rescale (TEST INFRASTRUCTURE ONLY).
//
// Runs the bodies of ks_rescale_grouped_kernel (deeppowers_b200/csrc/kernel_bodies.cuh: ks_phase1 in mode KS_MUL_RELIN or KS_DOT, the
// grouped phase 2, ms_tau_body for the special rows and for the dropped limb's row, ms_limb_group<..., DROP> for the kept limbs) in
// the kernel's role order with a sequential CTA policy, with the constants of host_params.cpp:build_rescale_consts.  A second entry
// runs the division alone on a crafted accumulator, so that the tests can place every y of the divided set where they want it.
// Built by tests/test_mul_rescale_cpu.py once per arithmetic variant; never linked into libdpfhe.so.
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

struct Ctx {
    HostParams hp;
    std::vector<LimbParams> lp;
    Twiddle *tw = nullptr, *itw = nullptr;
    ~Ctx() {
        free(tw);
        free(itw);
    }
};

// the division of one polynomial's accumulator acc [L][N] (the rows of every limb, below 16q) into out [Lq-1][N]: the special CTAs'
// and the dropped CTA's inverse transforms, then the kept limbs' ms_limb_group over K + 1 rows.  acc is used as the work rows.
template <int LOGN, int NT>
void divide_one(Ctx &e, HostCta &cta, uint64_t *buf, unsigned Ks, const MsConsts &K, const GroupConsts &G, const RescaleConsts &R, uint64_t *acc,
                uint64_t *tau, uint64_t *drop, uint64_t *out) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned Lq = e.hp.L - Ks, d = Lq - 1;
    for (unsigned k = 0; k < Ks; ++k) {
        const unsigned i = Lq + k;
        ms_tau_body<LOGN, NT, true>(cta, buf, acc + (size_t)i * N, acc + (size_t)i * N, e.itw + (size_t)i * N, G.lp_up[i], tau + (size_t)k * N, K);
    }
    ms_tau_body<LOGN, NT, true>(cta, buf, acc + (size_t)d * N, acc + (size_t)d * N, e.itw + (size_t)d * N, R.lp_drop, drop, K);
    for (unsigned i = 0; i < d; ++i)
        ms_limb_group<LOGN, NT, true, false, true>(cta, buf, tau, N, acc + (size_t)i * N, out + (size_t)i * N, e.tw + (size_t)i * N, e.lp[i], K, G, i,
                                                   nullptr, drop, &R);
}

// the kernel's program: groups ciphertexts in flight per round (digit slots and accumulators double-buffered by round parity)
template <int LOGN, int NT>
void run_mul_rescale(Ctx &e, unsigned Ks, bool dot, const DotArgs &D, const uint64_t *key, uint64_t *out, size_t batch, uint64_t t_plain,
                     unsigned groups) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned LK = e.hp.L, Lq = LK - Ks, GS = LK, d = Lq - 1;
    MsConsts K;
    GroupConsts Gc;
    RescaleConsts R;
    build_rescale_consts(e.hp, Ks, t_plain, Gc, K, R);
    const unsigned dnum = Gc.dnum;
    uint64_t *buf = aligned_new<uint64_t>(N);
    uint64_t *scratch = aligned_new<uint64_t>((size_t)groups * GS * 2 * N);
    uint64_t *hyb_all = aligned_new<uint64_t>((size_t)groups * Ks * KS_HYB_ROWS * N);
    uint64_t *drop_all = aligned_new<uint64_t>((size_t)groups * 4 * N);
    uint64_t *acc = aligned_new<uint64_t>((size_t)groups * GS * 2 * 2 * N);   // [slot][parity][2][N]
    const size_t key_words = (size_t)2 * dnum * LK * N;
    uint64_t *key_s = aligned_new<uint64_t>(key_words);   // Shoup companions, as key_prepare_kernel builds them
    for (size_t k = 0; k < key_words; ++k) key_s[k] = (uint64_t)((((unsigned __int128)key[k]) << 64) / e.lp[(k / N) % LK].q);
    KsArgs A;
    A.a = dot ? nullptr : D.a[0]; A.b = dot ? nullptr : D.b[0]; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = Lq; A.galois = 0; A.Lk = LK; A.hyb = hyb_all; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = 0;
    auto acc_of = [&](unsigned slot, unsigned parity) { return acc + ((size_t)slot * 2 + parity) * 2 * N; };
    HostCta cta{NT};
    const size_t P = (size_t)d * N;
    for (size_t r = 0; r * groups < batch; ++r) {
        const unsigned par = (unsigned)(r & 1);
        for (unsigned g = 0; g < groups; ++g) {
            const size_t ct = r * groups + g;
            if (ct >= batch) break;
            const unsigned base = g * GS;
            auto hyb_of = [&](unsigned k) { return hyb_all + ((size_t)g * Ks + k) * KS_HYB_ROWS * N; };
            auto drop_of = [&](unsigned c) { return drop_all + (((size_t)g * 2 + par) * 2 + c) * N; };
            const uint64_t *t_rows = scratch + ((size_t)base * 2 + par) * N;
            for (unsigned i = 0; i < Lq; ++i) {
                uint64_t *slot = scratch + ((size_t)(base + i) * 2 + par) * N;
                if (dot)
                    ks_phase1<LOGN, NT, KS_DOT, true>(cta, buf, A, Gc.lp_up[i], ct, i, slot, acc_of(base + i, par), K.qlm[i], K.qlm_s[i], nullptr, 0,
                                                      i / Ks, &D);
                else
                    ks_phase1<LOGN, NT, KS_MUL_RELIN, true>(cta, buf, A, Gc.lp_up[i], ct, i, slot, acc_of(base + i, par), K.qlm[i], K.qlm_s[i],
                                                            nullptr, 0, i / Ks);
            }
            for (unsigned i = 0; i < Lq; ++i)
                for (uint32_t jj = 1; jj < dnum; ++jj)
                    ks_phase2_group<LOGN, NT, false>(cta, buf, A, Gc, e.lp[i], ct, i, (i / Ks + jj) % dnum, jj, t_rows, 2 * N, acc_of(base + i, par));
            for (unsigned k = 0; k < Ks; ++k) {
                const unsigned i = Lq + k;
                uint64_t *hyb = hyb_of(k);
                for (uint32_t jj = 0; jj < dnum; ++jj)
                    ks_phase2_group<LOGN, NT, true>(cta, buf, A, Gc, e.lp[i], ct, i, (g + jj) % dnum, jj, t_rows, 2 * N, hyb);
                for (unsigned c = 0; c < 2; ++c)
                    ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)i * N, Gc.lp_up[i], hyb + ks_hyb_tau_row(par, c) * N, K);
            }
            for (unsigned c = 0; c < 2; ++c)   // the dropped limb's CTA
                ms_tau_body<LOGN, NT, true>(cta, buf, acc_of(base + d, par) + c * N, acc_of(base + d, par) + c * N, A.itw + (size_t)d * N, R.lp_drop,
                                            drop_of(c), K);
            for (unsigned i = 0; i < d; ++i)
                for (unsigned c = 0; c < 2; ++c)
                    ms_limb_group<LOGN, NT, true, false, true>(cta, buf, hyb_of(0) + ks_hyb_tau_row(par, c) * N, (size_t)KS_HYB_ROWS * N,
                                                               acc_of(base + i, par) + c * N, out + ct * 2 * P + c * P + (size_t)i * N,
                                                               A.tw + (size_t)i * N, e.lp[i], K, Gc, i, nullptr, drop_of(c), &R);
        }
    }
    free(buf); free(scratch); free(hyb_all); free(drop_all); free(acc); free(key_s);
}

template <int LOGN, int NT>
void run_divide(Ctx &e, unsigned Ks, const uint64_t *acc_in, uint64_t t_plain, uint64_t *out, size_t n_polys) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned L = e.hp.L, Lq = L - Ks;
    MsConsts K;
    GroupConsts Gc;
    RescaleConsts R;
    build_rescale_consts(e.hp, Ks, t_plain, Gc, K, R);
    uint64_t *buf = aligned_new<uint64_t>(N), *acc = aligned_new<uint64_t>((size_t)L * N), *tau = aligned_new<uint64_t>((size_t)Ks * N),
             *drop = aligned_new<uint64_t>(N);
    HostCta cta{NT};
    for (size_t n = 0; n < n_polys; ++n) {
        memcpy(acc, acc_in + n * L * N, (size_t)L * N * 8);
        divide_one<LOGN, NT>(e, cta, buf, Ks, K, Gc, R, acc, tau, drop, out + n * (Lq - 1) * N);
    }
    free(buf); free(acc); free(tau); free(drop);
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

bool shape_ok(const Ctx &e, unsigned K) { return K >= 1 && K <= (unsigned)KS_MAX_SPECIAL && 2 * K <= e.hp.L && e.hp.L - K >= 2; }
}  // namespace

extern "C" {

void *emu_mr_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
    Ctx *e = new Ctx();
    if (!build_host_params(log_n, L, moduli, e->hp).empty()) {
        delete e;
        return nullptr;
    }
#if DPFHE_FAST
    for (unsigned l = 0; l < L; ++l)   // the fast bodies are only valid for moduli k * 2^32 + 1
        if (e->hp.limbs[l].lp.nqh == 0) {
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
void emu_mr_destroy(void *h) { delete (Ctx *)h; }

// out [batch][2][L-K-1][N] through the kernel bodies; pool [n_pool][batch][2][L-K][N], pair t = (pool[ia[t]], pool[ib[t]]); key
// [dnum][2][L][N].  dot = 0 runs phase 1 in mode KS_MUL_RELIN (one pair), dot = 1 in mode KS_DOT.
int emu_mr_mul_rescale(void *h, unsigned K, int dot, const uint64_t *pool, unsigned n_pool, unsigned n_terms, const uint32_t *ia,
                       const uint32_t *ib, const uint64_t *key, uint64_t *out, size_t batch, uint64_t t_plain, unsigned groups) {
    Ctx *e = (Ctx *)h;
    if (!shape_ok(*e, K) || groups < 1 || (!dot && n_terms != 1)) return -1;
    DotArgs D;
    if (!dot_args(D, pool, (size_t)2 * (e->hp.L - K) << e->hp.log_n, batch, n_pool, n_terms, ia, ib)) return -1;
    switch (e->hp.log_n) {
        case 12: run_mul_rescale<12, 256>(*e, K, dot != 0, D, key, out, batch, t_plain, groups); return 0;
        case 13: run_mul_rescale<13, 256>(*e, K, dot != 0, D, key, out, batch, t_plain, groups); return 0;
        case 14: run_mul_rescale<14, 256>(*e, K, dot != 0, D, key, out, batch, t_plain, groups); return 0;
    }
    return -1;
}

// the division alone: acc [n_polys][L][N] (every row below 16q) -> out [n_polys][L-K-1][N]
int emu_mr_divide(void *h, unsigned K, const uint64_t *acc, uint64_t t_plain, uint64_t *out, size_t n_polys) {
    Ctx *e = (Ctx *)h;
    if (!shape_ok(*e, K)) return -1;
    switch (e->hp.log_n) {
        case 12: run_divide<12, 256>(*e, K, acc, t_plain, out, n_polys); return 0;
        case 13: run_divide<13, 256>(*e, K, acc, t_plain, out, n_polys); return 0;
        case 14: run_divide<14, 256>(*e, K, acc, t_plain, out, n_polys); return 0;
    }
    return -1;
}
}
