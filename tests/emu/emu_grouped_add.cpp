// emu_grouped_add.cpp — host emulator of the grouped rotation with the fused Horner addition (TEST INFRASTRUCTURE ONLY).
//
// Runs the role programs of ks_grouped_kernel<LOGN, 256, 3, KS_ROTATE, ADD> (deeppowers_b200/csrc/kernel_bodies.cuh: ks_phase1,
// ks_phase2_group, ms_tau_body, ms_limb_group<..., ADD>) with a sequential CTA policy, in dependency order, groups of Lq + K slots
// as the kernel has them.  Built by tests/test_grouped_add_cpu.py once per arithmetic variant; never linked into libdpfhe.so.
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

// ADD = false is the plain grouped rotation (the reference the fused form is compared with in the same build)
template <int LOGN, int NT, bool ADD>
void run_rotate_grouped(Ctx &e, unsigned Ks, const uint64_t *ct, const uint64_t *addend, const uint64_t *key, uint64_t *out, size_t batch,
                        uint32_t galois, uint64_t t_plain, unsigned G) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned LK = e.hp.L, Lq = LK - Ks, GS = LK;
    unsigned groups = G / GS;
    if (groups == 0) groups = 1;
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
    A.a = ct; A.b = ct; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = Lq; A.galois = galois; A.Lk = LK; A.hyb = hyb_all; A.only = nullptr;
    A.acc = acc; A.acc_par = 2; A.lift_reduce = 0;
    auto acc_of = [&](unsigned slot, unsigned parity) { return acc + ((size_t)slot * 2 + parity) * 2 * N; };
    HostCta cta{NT};
    for (size_t r = 0; r * groups < batch; ++r) {
        const unsigned par = (unsigned)(r & 1);
        for (unsigned g = 0; g < groups; ++g) {
            const size_t c_idx = r * groups + g;
            if (c_idx >= batch) break;
            const unsigned base = g * GS;
            auto hyb_of = [&](unsigned k) { return hyb_all + ((size_t)g * Ks + k) * KS_HYB_ROWS * N; };
            const uint64_t *t_rows = scratch + ((size_t)base * 2 + par) * N;
            for (unsigned i = 0; i < Lq; ++i)
                ks_phase1<LOGN, NT, KS_ROTATE, true>(cta, buf, A, Gc.lp_up[i], c_idx, i, scratch + ((size_t)(base + i) * 2 + par) * N, acc_of(base + i, par),
                                                     K.qlm[i], K.qlm_s[i], nullptr, 0, i / Ks);
            for (unsigned i = 0; i < Lq; ++i)
                for (uint32_t jj = 1; jj < dnum; ++jj)
                    ks_phase2_group<LOGN, NT, false>(cta, buf, A, Gc, e.lp[i], c_idx, i, (i / Ks + jj) % dnum, jj, t_rows, 2 * N, acc_of(base + i, par));
            for (unsigned k = 0; k < Ks; ++k) {
                const unsigned i = Lq + k;
                uint64_t *hyb = hyb_of(k);
                for (uint32_t jj = 0; jj < dnum; ++jj)
                    ks_phase2_group<LOGN, NT, true>(cta, buf, A, Gc, e.lp[i], c_idx, i, (g + jj) % dnum, jj, t_rows, 2 * N, hyb);
                for (unsigned c = 0; c < 2; ++c)
                    ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)i * N, Gc.lp_up[i], hyb + ks_hyb_tau_row(par, c) * N, K);
            }
            const size_t P = (size_t)Lq * N;
            for (unsigned i = 0; i < Lq; ++i)
                for (unsigned c = 0; c < 2; ++c) {
                    const size_t row_off = c_idx * 2 * P + c * P + (size_t)i * N;
                    ms_limb_group<LOGN, NT, true, ADD>(cta, buf, hyb_of(0) + ks_hyb_tau_row(par, c) * N, (size_t)KS_HYB_ROWS * N, acc_of(base + i, par) + c * N,
                                                       out + row_off, A.tw + (size_t)i * N, e.lp[i], K, Gc, i, ADD ? addend + row_off : nullptr);
                }
        }
    }
    free(buf);
    free(scratch);
    free(hyb_all);
    free(acc);
    free(key_s);
}

template <bool ADD>
int dispatch(Ctx &e, unsigned K, const uint64_t *ct, const uint64_t *addend, const uint64_t *key, uint64_t *out, size_t batch, uint32_t galois,
             uint64_t t_plain, unsigned G) {
    switch (e.hp.log_n) {   // 256 threads at every N, as the device kernel (N = 16384 takes the half-limb path)
        case 12: run_rotate_grouped<12, 256, ADD>(e, K, ct, addend, key, out, batch, galois, t_plain, G); return 0;
        case 13: run_rotate_grouped<13, 256, ADD>(e, K, ct, addend, key, out, batch, galois, t_plain, G); return 0;
        case 14: run_rotate_grouped<14, 256, ADD>(e, K, ct, addend, key, out, batch, galois, t_plain, G); return 0;
    }
    return -1;
}
}  // namespace

extern "C" {

void *emu_ga_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
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
void emu_ga_destroy(void *h) { delete (Ctx *)h; }

// out = rotate_grouped(ct) + addend (addend canonical, [batch][2][L-K][N]); addend == NULL: the plain grouped rotation.
// G: resident slots (groups of L), as the persistent grid
int emu_ga_rotate(void *h, unsigned K, const uint64_t *ct, const uint64_t *addend, const uint64_t *key, uint64_t *out, size_t batch,
                  uint32_t galois, uint64_t t_plain, unsigned G) {
    Ctx *e = (Ctx *)h;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > e->hp.L) return -1;
    return addend ? dispatch<true>(*e, K, ct, addend, key, out, batch, galois, t_plain, G)
                  : dispatch<false>(*e, K, ct, nullptr, key, out, batch, galois, t_plain, G);
}
}
