// emu_public_keys.cpp — host emulator of the public-key kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs the public-key mode of keys_limb_body (N <= 8192) and keys_half_body (N = 16384, both CTAs of the pair) and the
// public-key encryption body pub_enc_body of deeppowers_b200/csrc/keys.cuh with a sequential CTA policy, one (item, limb) at a
// time as the grid of keys.cu does, with the launch constants from the product's build_key_args.  Built by
// tests/test_public_key_emu_cpu.py; never linked into libdpfhe.so.
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

// n_items items of one mode, every (item, limb) in grid order; at N = 16384 both CTAs of the pair
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
        for (int h = 0; h < (LOGN == NTT_PAIR_LOGN ? 2 : 1); ++h) {
            if constexpr (MODE == KM_ENC_PUBLIC) pub_enc_body<LOGN, 256>(cta, buf.data(), small.data(), A, tw, p, l, L, w / L, h);
            else if constexpr (LOGN == NTT_PAIR_LOGN) keys_half_body<256, MODE>(cta, buf.data(), small.data(), A, tw, p, l, L, w / L, h);
            else keys_limb_body<LOGN, 256, MODE>(cta, buf.data(), small.data(), A, tw, p, l, L, w / L);
        }
    }
}

template <int MODE>
int run_n(const Ctx &c, const KeyArgs &A, size_t n_items) {
    switch (c.hp.log_n) {
        case 12: run<12, MODE>(c, A, n_items); return 0;
        case 13: run<13, MODE>(c, A, n_items); return 0;
        case 14: run<14, MODE>(c, A, n_items); return 0;
    }
    return -1;
}
}  // namespace

extern "C" {

void *emu_pk_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
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
void emu_pk_destroy(void *h) { delete (Ctx *)h; }

// the public key [2][L][N] (KM_PUBLIC_KEY) under the secret s
int emu_pk_public_keygen(void *h, const uint8_t *seed, uint64_t t_plain, const uint64_t *s, uint64_t *pk) {
    const Ctx &c = *(const Ctx *)h;
    KeyArgs A = build_key_args(c.hp, seed, 0, t_plain);
    A.s = s;
    A.out = pk;
    return run_n<KM_PUBLIC_KEY>(c, A, 1);
}

// n public-key encryptions (KM_ENC_PUBLIC) of pt [n][L][N] under pk [2][L][N] -> ct [n][2][L][N]
int emu_pk_encrypt_public(void *h, const uint8_t *seed, uint64_t t_plain, uint64_t item0, const uint64_t *pk, const uint64_t *pt,
                          uint64_t *ct, size_t n) {
    const Ctx &c = *(const Ctx *)h;
    KeyArgs A = build_key_args(c.hp, seed, 0, t_plain);
    A.item0 = item0;
    A.s = pk;
    A.pt = pt;
    A.out = ct;
    return run_n<KM_ENC_PUBLIC>(c, A, n);
}
}
