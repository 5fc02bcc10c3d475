// emu_keys.cpp — host emulator of the key generation and encryption kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs keys_limb_body (N <= 8192) and keys_half_body (N = 16384, both CTAs of the pair) of deeppowers_b200/csrc/keys.cuh and
// decrypt_chunk with a sequential CTA policy, one (item, limb) at a time as the grid of keys.cu does, with the launch constants
// from the product's build_key_args.  Built by tests/test_keys_emu_cpu.py; never linked into libdpfhe.so.
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "host_params.hpp"
#include "keys.cuh"

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
};

struct Ctx {
    HostParams hp;
    std::vector<Twiddle> tw;   // [L][N] device layout
};

template <int LOGN, int MODE>
void run(const Ctx &c, const KeyArgs &A, size_t n_items) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<uint64_t> buf(N);
    std::vector<signed char> small(N);
    HostCta cta{256};
    for (size_t w = 0; w < n_items * L; ++w) {
        const unsigned l = (unsigned)(w % L);
        const LimbParams p = c.hp.limbs[l].lp;
        const Twiddle *tw = c.tw.data() + l * N;
        if (LOGN == NTT_PAIR_LOGN) {   // keys_ntt_pair_kernel: the two CTAs of the pair, each with half a limb
            for (int h = 0; h < 2; ++h) keys_half_body<256, MODE>(cta, buf.data(), small.data(), A, tw, p, l, L, w / L, h);
        } else {
            keys_limb_body<LOGN, 256, MODE>(cta, buf.data(), small.data(), A, tw, p, l, L, w / L);
        }
    }
}

template <int LOGN>
int run_mode(const Ctx &c, int mode, const KeyArgs &A, size_t n_items) {
    switch (mode) {
        case KM_SECRET: run<LOGN, KM_SECRET>(c, A, n_items); return 0;
        case KM_ENC: run<LOGN, KM_ENC>(c, A, n_items); return 0;
        case KM_RELIN: run<LOGN, KM_RELIN>(c, A, n_items); return 0;
        case KM_GALOIS: run<LOGN, KM_GALOIS>(c, A, n_items); return 0;
    }
    return -1;
}
}  // namespace

extern "C" {

void *emu_keys_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
    Ctx *c = new Ctx();
    if (!build_host_params(log_n, L, moduli, c->hp).empty()) {
        delete c;
        return nullptr;
    }
    const size_t N = (size_t)1 << log_n;
    c->tw.resize(L * N);
    for (unsigned l = 0; l < L; ++l)
        for (size_t k = 0; k < N; ++k) c->tw[l * N + k] = c->hp.limbs[l].tw[k];
    return c;
}
void emu_keys_destroy(void *h) { delete (Ctx *)h; }

// mode as keys.cu (0 secret, 1 encryption, 2 relinearisation key, 3 Galois keys); n_items: 1, ciphertexts, or n_elts * digits
int emu_keys_run(void *h, int mode, const uint8_t *seed, unsigned K, uint64_t t_plain, uint64_t item0, const uint64_t *galois,
                 unsigned n_elts, const uint64_t *s, const uint64_t *pt, uint64_t *out, size_t n_items) {
    const Ctx &c = *(const Ctx *)h;
    if (n_elts > (unsigned)KEYS_MAX_ELTS) return -2;
    KeyArgs A = build_key_args(c.hp, seed, K, t_plain);
    for (unsigned e = 0; e < n_elts; ++e) A.galois[e] = galois[e];
    A.item0 = item0;
    A.s = s;
    A.pt = pt;
    A.out = out;
    switch (c.hp.log_n) {
        case 12: return run_mode<12>(c, mode, A, n_items);
        case 13: return run_mode<13>(c, mode, A, n_items);
        case 14: return run_mode<14>(c, mode, A, n_items);
    }
    return -1;
}

// pt [n][L][N] = c0 + c1 s (+ c2 s^2) by decrypt_chunk, chunk by chunk
int emu_keys_decrypt(void *h, const uint64_t *ct, const uint64_t *s, unsigned n_comp, uint64_t *pt, size_t n) {
    const Ctx &c = *(const Ctx *)h;
    const size_t NC = ((size_t)1 << c.hp.log_n) / 2, pc = NC * c.hp.L;
    auto C = reinterpret_cast<const U64x2 *>(ct), S = reinterpret_cast<const U64x2 *>(s);
    auto O = reinterpret_cast<U64x2 *>(pt);
    for (size_t ch = 0; ch < n * pc; ++ch) {
        const size_t k = ch / pc, in_poly = ch % pc;
        O[ch] = decrypt_chunk(C + k * n_comp * pc + in_poly, S + in_poly, pc, n_comp, c.hp.limbs[in_poly / NC].lp);
    }
    return 0;
}
}
