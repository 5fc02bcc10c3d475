// emu_fused_blk.cpp — host emulator of the fused key switch at N <= 8192 (TEST INFRASTRUCTURE ONLY).
//
// Runs the bodies of ks_fused_kernel<LOGN, 256, 2, MODE> at N = 4096 and 8192 (deeppowers_b200/csrc/kernel_bodies.cuh:
// ks_blk_phase1_local, ks_blk_phase1_outer, ks_blk_phase2) with a sequential CTA policy.  Each CTA of a limb's pair has its own
// transform buffer and accumulator half-rows; the pair barriers of the kernel become phase order: every CTA's local phase 1,
// then every CTA's outer stage (reading the partner's buffer), then the foreign digits.  Built by tests/test_fused_blk_cpu.py
// once per arithmetic variant; never linked into libdpfhe.so.
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

template <int LOGN, int MODE>
void run(Ctx &e, const uint64_t *a, const uint64_t *b, const uint64_t *key, uint64_t *out, size_t batch, uint32_t galois, bool lift_reduce) {
    constexpr int NT = 256, PAIR = ks_blk_pair<LOGN>();
    const size_t N = (size_t)1 << LOGN, BLK = (size_t)1 << KS_BLK_LOGN;
    const unsigned L = e.hp.L;
    // per CTA (limb i, half h): transform buffer and accumulator half-rows, as the kernel's shared memory
    uint64_t *bufs = aligned_new<uint64_t>((size_t)L * PAIR * BLK);
    U64x2 *accs = aligned_new<U64x2>((size_t)L * PAIR * 2 * KS_BLK_HC);
    uint64_t *scratch = aligned_new<uint64_t>((size_t)L * N);   // one digit slot per limb
    const size_t key_words = (size_t)2 * L * L * N;
    uint64_t *key_s = aligned_new<uint64_t>(key_words);   // Shoup companions, as key_prepare_kernel builds them
    for (size_t k = 0; k < key_words; ++k) key_s[k] = (uint64_t)((((unsigned __int128)key[k]) << 64) / e.lp[(k / N) % L].q);
    KsArgs A;
    A.a = a; A.b = b; A.key = key; A.key_s = key_s; A.out = out; A.scratch = scratch;
    A.tw = e.tw; A.itw = e.itw; A.L = L; A.galois = galois; A.Lk = L; A.hyb = nullptr; A.only = nullptr;
    A.acc = nullptr; A.acc_par = 1; A.lift_reduce = lift_reduce ? 1u : 0u;
    auto buf_of = [&](unsigned i, int h) { return bufs + ((size_t)i * PAIR + h) * BLK; };
    auto acc_of = [&](unsigned i, int h) { return accs + ((size_t)i * PAIR + h) * 2 * KS_BLK_HC; };
    HostCta cta{NT};
    for (size_t ct = 0; ct < batch; ++ct) {
        for (unsigned i = 0; i < L; ++i)
            for (int h = 0; h < PAIR; ++h) ks_blk_phase1_local<LOGN, NT, MODE>(cta, buf_of(i, h), acc_of(i, h), A, e.lp[i], ct, i, h);
        if (L == 1) continue;
        for (unsigned i = 0; i < L; ++i)
            for (int h = 0; h < PAIR; ++h)
                ks_blk_phase1_outer<LOGN, NT>(cta, buf_of(i, h), buf_of(i, h ^ (PAIR - 1)), A, e.lp[i], i, h, scratch + (size_t)i * N);
        for (unsigned i = 0; i < L; ++i)
            for (int h = 0; h < PAIR; ++h)
                for (uint32_t jj = 1; jj < L; ++jj) {
                    const uint32_t j = (i + jj) % L;
                    ks_blk_phase2<LOGN, NT>(cta, buf_of(i, h), acc_of(i, h), A, e.lp[i], ct, i, j, jj, h, scratch + (size_t)j * N);
                }
    }
    free(bufs);
    free(accs);
    free(scratch);
    free(key_s);
}

template <int LOGN>
int dispatch_mode(Ctx &e, int mode, const uint64_t *a, const uint64_t *b, const uint64_t *key, uint64_t *out, size_t batch, uint32_t galois,
                  bool lift_reduce) {
    switch (mode) {
        case KS_MUL_RELIN: run<LOGN, KS_MUL_RELIN>(e, a, b, key, out, batch, galois, lift_reduce); return 0;
        case KS_PLAIN: run<LOGN, KS_PLAIN>(e, a, b, key, out, batch, galois, lift_reduce); return 0;
        case KS_ROTATE: run<LOGN, KS_ROTATE>(e, a, b, key, out, batch, galois, lift_reduce); return 0;
    }
    return -1;
}
}  // namespace

extern "C" {

void *emu_fb_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
    if (log_n != 12 && log_n != 13) return nullptr;
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
void emu_fb_destroy(void *h) { delete (Ctx *)h; }

// mode: KS_MUL_RELIN (a, b ciphertexts), KS_PLAIN (a = digits [batch][L][N]), KS_ROTATE (a ciphertexts, galois); key [L][2][L][N].
// lift_reduce: reduce each digit into the limb it is lifted to (the library does so unless every modulus is below twice every other)
int emu_fb_ks(void *h, int mode, const uint64_t *a, const uint64_t *b, const uint64_t *key, uint64_t *out, size_t batch, uint32_t galois,
              int lift_reduce) {
    Ctx *e = (Ctx *)h;
    if (e->hp.log_n == 12) return dispatch_mode<12>(*e, mode, a, b, key, out, batch, galois, lift_reduce != 0);
    return dispatch_mode<13>(*e, mode, a, b, key, out, batch, galois, lift_reduce != 0);
}
}
