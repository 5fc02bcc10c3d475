// emu_seeded.cpp — host emulator of the seeded key-generation / encryption bodies and of the expansion body (TEST INFRASTRUCTURE ONLY).
//
// Runs keys_limb_body / keys_half_body of deeppowers_b200/csrc/keys.cuh in the seeded modes (KM_ENC_SEEDED, KM_RELIN_SEEDED,
// KM_GALOIS_SEEDED) with a sequential CTA policy, one (item, limb) at a time as keys_seeded_ntt(_pair)_kernel does, and expand_block
// block by block as expand_seeded_kernel does, with the launch constants from the product's build_key_args.  Built by
// tests/test_seeded_emu_cpu.py in both arithmetic variants; never linked into libdpfhe.so.
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "host_params.hpp"
#include "keys.cuh"

using namespace dpfhe;
using namespace dpfhe::DPFHE_VNS;

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
    std::vector<Twiddle> tw;
};

template <int LOGN, int MODE>
void run(const Ctx &c, const SeededKeyArgs &A, size_t n_items) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<uint64_t> buf(N);
    std::vector<signed char> small(N);
    HostCta cta{256};
    for (size_t w = 0; w < n_items * L; ++w) {
        const unsigned l = (unsigned)(w % L);
        const Twiddle *tw = c.tw.data() + l * N;
        if (LOGN == NTT_PAIR_LOGN) {
            for (int h = 0; h < 2; ++h) keys_half_body<256, MODE>(cta, buf.data(), small.data(), A, tw, c.hp.limbs[l].lp, l, L, w / L, h);
        } else {
            keys_limb_body<LOGN, 256, MODE>(cta, buf.data(), small.data(), A, tw, c.hp.limbs[l].lp, l, L, w / L);
        }
    }
}

template <int LOGN>
int run_mode(const Ctx &c, int mode, const SeededKeyArgs &A, size_t n_items) {
    switch (mode) {
        case KM_ENC_SEEDED: run<LOGN, KM_ENC_SEEDED>(c, A, n_items); return 0;
        case KM_RELIN_SEEDED: run<LOGN, KM_RELIN_SEEDED>(c, A, n_items); return 0;
        case KM_GALOIS_SEEDED: run<LOGN, KM_GALOIS_SEEDED>(c, A, n_items); return 0;
    }
    return -1;
}

template <int LOGN>
void expand(const Ctx &c, bool keys, const SeededKeyArgs &A, const uint64_t *src, uint64_t *dst, size_t n_rows) {
    const size_t n_blocks = n_rows * c.hp.L << (LOGN - 2);
    auto S = reinterpret_cast<const U64x2 *>(src);
    auto D = reinterpret_cast<U64x2 *>(dst);
    for (size_t w = 0; w < n_blocks; ++w) {
        const LimbParams &p = c.hp.limbs[(w >> (LOGN - 2)) % c.hp.L].lp;
        if (keys) expand_block<LOGN, true>(S, D, A, p, c.hp.L, w);
        else expand_block<LOGN, false>(S, D, A, p, c.hp.L, w);
    }
}

SeededKeyArgs args(const Ctx &c, const uint8_t *seed, const uint8_t *a_seed, unsigned K, uint64_t t_plain, uint64_t item0,
                   const uint64_t *galois, unsigned n_elts) {
    SeededKeyArgs A;
    static_cast<KeyArgs &>(A) = build_key_args(c.hp, seed, K, t_plain);
    for (int i = 0; i < 8; ++i)
        A.a_seed[i] = (uint32_t)a_seed[4 * i] | (uint32_t)a_seed[4 * i + 1] << 8 | (uint32_t)a_seed[4 * i + 2] << 16 | (uint32_t)a_seed[4 * i + 3] << 24;
    for (unsigned e = 0; e < n_elts; ++e) A.galois[e] = galois[e];
    A.item0 = item0;
    return A;
}
}  // namespace

extern "C" {

void *emu_seeded_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
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
void emu_seeded_destroy(void *h) { delete (Ctx *)h; }

// mode as keys.cu (6 seeded encryption, 7 seeded relinearisation key, 8 seeded Galois keys); n_items: ciphertexts or n_elts * digits
int emu_seeded_run(void *h, int mode, const uint8_t *seed, const uint8_t *a_seed, unsigned K, uint64_t t_plain, uint64_t item0,
                   const uint64_t *galois, unsigned n_elts, const uint64_t *s, const uint64_t *pt, uint64_t *out, size_t n_items) {
    const Ctx &c = *(const Ctx *)h;
    if (n_elts > (unsigned)KEYS_MAX_ELTS) return -2;
    SeededKeyArgs A = args(c, seed, a_seed, K, t_plain, item0, galois, n_elts);
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

// seeded rows [n_rows][L][N] -> [n_rows][2][L][N]; keys: n_rows = n_elts * digits with items galois[e], else ciphertexts item0 + k
int emu_seeded_expand(void *h, int keys, const uint8_t *a_seed, unsigned K, uint64_t item0, const uint64_t *galois, unsigned n_elts,
                      const uint64_t *src, uint64_t *dst, size_t n_rows) {
    const Ctx &c = *(const Ctx *)h;
    if (n_elts > (unsigned)KEYS_MAX_ELTS) return -2;
    const SeededKeyArgs A = args(c, a_seed, a_seed, K, 0, item0, galois, n_elts);
    switch (c.hp.log_n) {
        case 12: expand<12>(c, keys != 0, A, src, dst, n_rows); return 0;
        case 13: expand<13>(c, keys != 0, A, src, dst, n_rows); return 0;
        case 14: expand<14>(c, keys != 0, A, src, dst, n_rows); return 0;
    }
    return -1;
}
}
