// emu_ct_dot.cpp — host emulator of the encrypted inner product (TEST INFRASTRUCTURE ONLY).
//
// Runs ks_phase1 in mode KS_DOT and the unchanged grouped bodies (deeppowers_b200/csrc/kernel_bodies.cuh) in the role order of
// ct_dot_grouped_kernel with a sequential CTA policy, as emu.cpp's run_ks_grouped does for the other modes.  Built by
// tests/test_ct_dot_cpu.py once per arithmetic variant with DPFHE_DOT_TRACK, which records the largest intermediates of the summed
// tensor product; never linked into libdpfhe.so.
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

// groups: ciphertexts in flight per round (the digit slots and accumulators are double-buffered by round parity, as on the device)
template <int LOGN, int NT>
void run_ct_dot(Ctx &e, unsigned Ks, const DotArgs &D, const uint64_t *key, uint64_t *out, size_t batch, uint64_t t_plain, unsigned groups) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned LK = e.hp.L, Lq = LK - Ks, GS = LK;
    MsConsts K;
    GroupConsts Gc;
    build_group_consts(e.hp, Ks, t_plain, Gc, K);
    const unsigned dnum = Gc.dnum;
    uint64_t *buf = aligned_new<uint64_t>(N);
    uint64_t *scratch = aligned_new<uint64_t>((size_t)groups * GS * 2 * N);
    uint64_t *hyb_all = aligned_new<uint64_t>((size_t)groups * Ks * KS_HYB_ROWS * N);
    uint64_t *acc = aligned_new<uint64_t>((size_t)groups * GS * 2 * 2 * N);   // [slot][parity][2][N]
    const size_t key_words = (size_t)2 * dnum * LK * N;
    uint64_t *key_s = aligned_new<uint64_t>(key_words);   // Shoup companions, as key_prepare_kernel builds them
    for (size_t k = 0; k < key_words; ++k) key_s[k] = (uint64_t)((((unsigned __int128)key[k]) << 64) / e.lp[(k / N) % LK].q);
    KsArgs A;
    A.a = nullptr; A.b = nullptr; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = Lq; A.galois = 0; A.Lk = LK; A.hyb = hyb_all; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = 0;
    auto acc_of = [&](unsigned slot, unsigned parity) { return acc + ((size_t)slot * 2 + parity) * 2 * N; };
    HostCta cta{NT};
    for (size_t r = 0; r * groups < batch; ++r) {
        const unsigned par = (unsigned)(r & 1);
        for (unsigned g = 0; g < groups; ++g) {
            const size_t ct = r * groups + g;
            if (ct >= batch) break;
            const unsigned base = g * GS;
            auto hyb_of = [&](unsigned k) { return hyb_all + ((size_t)g * Ks + k) * KS_HYB_ROWS * N; };
            const uint64_t *t_rows = scratch + ((size_t)base * 2 + par) * N;
            for (unsigned i = 0; i < Lq; ++i)
                ks_phase1<LOGN, NT, KS_DOT, true>(cta, buf, A, Gc.lp_up[i], ct, i, scratch + ((size_t)(base + i) * 2 + par) * N, acc_of(base + i, par),
                                                  K.qlm[i], K.qlm_s[i], nullptr, 0, i / Ks, &D);
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
            const size_t P = (size_t)Lq * N;
            for (unsigned i = 0; i < Lq; ++i)
                for (unsigned c = 0; c < 2; ++c)
                    ms_limb_group<LOGN, NT>(cta, buf, hyb_of(0) + ks_hyb_tau_row(par, c) * N, (size_t)KS_HYB_ROWS * N, acc_of(base + i, par) + c * N,
                                            out + ct * 2 * P + c * P + (size_t)i * N, A.tw + (size_t)i * N, e.lp[i], K, Gc, i);
        }
    }
    free(buf); free(scratch); free(hyb_all); free(acc); free(key_s);
}

// pair t = (pool[ia[t]], pool[ib[t]]), pool [n_pool][batch][2][Lq][N]
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

extern "C" {

void *emu_dot_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
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
void emu_dot_destroy(void *h) { delete (Ctx *)h; }

// out [batch][2][L-K][N] through the kernel bodies; key [dnum][2][L][N]
int emu_dot_ct_dot(void *h, unsigned K, const uint64_t *pool, unsigned n_pool, unsigned n_terms, const uint32_t *ia, const uint32_t *ib,
                   const uint64_t *key, uint64_t *out, size_t batch, uint64_t t_plain, unsigned groups) {
    Ctx *e = (Ctx *)h;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > e->hp.L || groups < 1) return -1;
    DotArgs D;
    if (!dot_args(D, pool, (size_t)2 * (e->hp.L - K) << e->hp.log_n, batch, n_pool, n_terms, ia, ib)) return -1;
    switch (e->hp.log_n) {
        case 12: run_ct_dot<12, 256>(*e, K, D, key, out, batch, t_plain, groups); return 0;
        case 13: run_ct_dot<13, 256>(*e, K, D, key, out, batch, t_plain, groups); return 0;
        case 14: run_ct_dot<14, 256>(*e, K, D, key, out, batch, t_plain, groups); return 0;
    }
    return -1;
}

// the summed tensor product alone, as the kernel body leaves it (congruent mod q_l, below 15 q_l): sums [3][Lq][N] of ciphertext 0
// of a pool [n_pool][1][2][Lq][N]
int emu_dot_sums(void *h, unsigned Lq, const uint64_t *pool, unsigned n_pool, unsigned n_terms, const uint32_t *ia, const uint32_t *ib, uint64_t *sums) {
    Ctx *e = (Ctx *)h;
    if (Lq < 1 || Lq > e->hp.L) return -1;
    const size_t N = (size_t)1 << e->hp.log_n, P = (size_t)Lq * N;
    DotArgs D;
    if (!dot_args(D, pool, 2 * P, 1, n_pool, n_terms, ia, ib)) return -1;
    for (unsigned l = 0; l < Lq; ++l)
        for (size_t c = 0; c < N / 2; ++c) {
            U64x2 d[3];
            dot_coeff_pair(D, l * N + 2 * c, P, e->lp[l], d[0], d[1], d[2]);
            for (int k = 0; k < 3; ++k) {
                sums[k * P + l * N + 2 * c] = d[k].x;
                sums[k * P + l * N + 2 * c + 1] = d[k].y;
            }
        }
    return 0;
}

// largest intermediates since the last call: out[0] = the largest 128-bit running sum over 2^(2b) (b = bit length of the modulus;
// barrett_lazy_long wants it below 16), out[1] = the largest reduced value over q (it promises below 15); then reset
void emu_dot_track(double *out) {
    DotTrack &t = dot_track();
    out[0] = t.sum_over_q2;
    out[1] = t.red_over_q;
    t = DotTrack();
}
}
