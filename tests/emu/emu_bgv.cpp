// emu_bgv.cpp — host emulator of the BGV slot-encoding kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs bgv_enc_body, the lifting load stage of the forward transform, ntt_inv_body and bgv_dec_body of
// deeppowers_b200/csrc/kernel_bodies.cuh with a sequential CTA policy, in the order the kernels of abi.cu run them, and the
// product's table builders of host_params.cpp.  Built by tests/test_bgv_encoding_cpu.py; never linked into libdpfhe.so.
#include <cstdint>
#include <cstdlib>
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
};

struct Ctx {
    HostParams hp;
    std::vector<Twiddle> tw, itw;   // [L][N] device layout
};

Ctx *make(unsigned log_n, unsigned L, const uint64_t *moduli) {
    Ctx *c = new Ctx();
    if (!build_host_params(log_n, L, moduli, c->hp).empty()) {
        delete c;
        return nullptr;
    }
    const size_t N = (size_t)1 << log_n;
    c->tw.resize(L * N);
    c->itw.resize(L * N);
    for (unsigned l = 0; l < L; ++l)
        for (size_t k = 0; k < N; ++k) {
            c->tw[l * N + k] = c->hp.limbs[l].tw[k];
            c->itw[l * N + k] = c->hp.limbs[l].itw[k];
        }
    return c;
}

// the tables as the context uploads them: tab holds [4][N] twiddle rows and [2][N/2] positions
bool tables(const Ctx &c, uint64_t t, std::vector<uint32_t> &tab, BgvTables &T) {
    if (!build_bgv_tables(c.hp, t, tab, T)) return false;
    const size_t N = (size_t)1 << c.hp.log_n;
    T.tw = tab.data();
    T.pos = tab.data() + 4 * N;
    return true;
}

template <int LOGN>
void encode(Ctx &c, const int64_t *slots, uint64_t *pt, size_t n_vec, const BgvTables &T) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<uint32_t> a(N), x(N);
    std::vector<uint64_t> buf(N);
    HostCta enc{512}, ntt{256};
    for (size_t v = 0; v < n_vec; ++v) {
        bgv_enc_body<LOGN, 512>(enc, a.data(), slots + v * N, x.data(), T);
        for (unsigned l = 0; l < L; ++l) {
            const LimbParams p = c.hp.limbs[l].lp;
            auto src = [&](int ch) {
                U64x2 r;
                r.x = bgv_lift(x[2 * ch], T.m.t, p);
                r.y = bgv_lift(x[2 * ch + 1], T.m.t, p);
                return r;
            };
            uint64_t *out = pt + (v * L + l) * N;
            if (LOGN == NTT_PAIR_LOGN) {   // bgv_enc_ntt_pair_kernel: two half buffers
                for (int h = 0; h < 2; ++h) {
                    ntt_fwd_half_load_src<256>(ntt, buf.data(), src, c.tw.data() + l * N, p, h);
                    ntt_fwd_half_finish<256>(ntt, buf.data(), out, c.tw.data() + l * N, p, h);
                }
            } else {
                ntt_fwd_src_body<LOGN, 256>(ntt, buf.data(), src, out, c.tw.data() + l * N, p);
            }
        }
    }
}

template <int LOGN>
void decode(Ctx &c, const uint64_t *pt, uint64_t *slots, size_t n_vec, const BgvTables &T, uint64_t t) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<uint32_t> a(N);
    std::vector<uint64_t> work(pt, pt + n_vec * L * N), buf(N);
    std::vector<LimbParams> lp(L);
    for (unsigned l = 0; l < L; ++l) lp[l] = c.hp.limbs[l].lp;
    BgvConsts K;
    build_bgv_consts(c.hp, t, K);
    HostCta dec{512}, ntt{256};
    for (size_t w = 0; w < n_vec * L; ++w) ntt_inv_body<LOGN, 256>(ntt, buf.data(), work.data() + w * N, c.itw.data() + (w % L) * N, lp[w % L]);
    for (size_t v = 0; v < n_vec; ++v) bgv_dec_body<LOGN, 512>(dec, a.data(), work.data() + v * L * N, slots + v * N, T, lp.data(), K, L);
}
}  // namespace

extern "C" {

void *emu_bgv_create(unsigned log_n, unsigned L, const uint64_t *moduli) { return make(log_n, L, moduli); }
void emu_bgv_destroy(void *h) { delete (Ctx *)h; }
// the product's zeta for t, or 0 when it rejects t
uint64_t emu_bgv_zeta(void *h, uint64_t t) {
    const Ctx *c = (const Ctx *)h;
    return bgv_plain_modulus_valid(c->hp.log_n, t) ? bgv_zeta(c->hp.log_n, t) : 0;
}
int emu_bgv_encode(void *h, const int64_t *slots, uint64_t *pt, size_t n_vec, uint64_t t) {
    Ctx &c = *(Ctx *)h;
    std::vector<uint32_t> tab;
    BgvTables T;
    if (!tables(c, t, tab, T)) return -2;
    switch (c.hp.log_n) {
        case 12: encode<12>(c, slots, pt, n_vec, T); return 0;
        case 13: encode<13>(c, slots, pt, n_vec, T); return 0;
        case 14: encode<14>(c, slots, pt, n_vec, T); return 0;
    }
    return -1;
}
int emu_bgv_decode(void *h, const uint64_t *pt, uint64_t *slots, size_t n_vec, uint64_t t) {
    Ctx &c = *(Ctx *)h;
    std::vector<uint32_t> tab;
    BgvTables T;
    if (!tables(c, t, tab, T)) return -2;
    switch (c.hp.log_n) {
        case 12: decode<12>(c, pt, slots, n_vec, T, t); return 0;
        case 13: decode<13>(c, pt, slots, n_vec, T, t); return 0;
        case 14: decode<14>(c, pt, slots, n_vec, T, t); return 0;
    }
    return -1;
}
}
