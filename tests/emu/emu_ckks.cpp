// emu_ckks.cpp — host emulator of the CKKS slot-encoding kernel bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs ckks_enc_fft_body, the reducing load stage of the forward transform, ntt_inv_body and ckks_dec_fft_body of
// deeppowers_b200/csrc/kernel_bodies.cuh with a sequential CTA policy, in the order the kernels of abi.cu run them, and the
// product's table builders of host_params.cpp.  Built by tests/test_ckks_encoding_cpu.py with -ffp-contract=off; never linked
// into libdpfhe.so.
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
    std::vector<Cplx> ctw;
    std::vector<uint32_t> tj;
    std::vector<uint64_t> pow2;
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
    build_ckks_tables(c->hp, c->ctw, c->tj, c->pow2);
    return c;
}

template <int LOGN>
void encode(Ctx &c, const double *slots, uint64_t *pt, size_t n_vec, double scale) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<Cplx> a(N / 2);
    std::vector<double> x(N);
    std::vector<uint64_t> buf(N);
    HostCta fft{512}, ntt{256};
    const double sc = scale * (2.0 / (double)N);
    for (size_t v = 0; v < n_vec; ++v) {
        ckks_enc_fft_body<LOGN, 512>(fft, a.data(), reinterpret_cast<const Cplx *>(slots) + v * (N / 2), x.data(), c.ctw.data(), c.tj.data(), sc);
        for (unsigned l = 0; l < L; ++l) {
            const LimbParams p = c.hp.limbs[l].lp;
            const uint64_t *p2 = c.pow2.data() + (size_t)l * CKKS_POW2_E;
            auto src = [&](int ch) {
                U64x2 r;
                r.x = ckks_reduce(x[2 * ch], p, p2);
                r.y = ckks_reduce(x[2 * ch + 1], p, p2);
                return r;
            };
            uint64_t *out = pt + (v * L + l) * N;
            if (LOGN == NTT_PAIR_LOGN) {   // ckks_enc_ntt_pair_kernel: two half buffers
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
void decode(Ctx &c, const uint64_t *pt, double *slots, size_t n_vec, double scale) {
    constexpr size_t N = (size_t)1 << LOGN;
    const unsigned L = c.hp.L;
    std::vector<Cplx> a(N / 2);
    std::vector<uint64_t> work(pt, pt + n_vec * L * N), buf(N);
    std::vector<LimbParams> lp(L);
    for (unsigned l = 0; l < L; ++l) lp[l] = c.hp.limbs[l].lp;
    CkksConsts K;
    build_ckks_consts(c.hp, scale, K);
    HostCta fft{512}, ntt{256};
    for (size_t w = 0; w < n_vec * L; ++w) ntt_inv_body<LOGN, 256>(ntt, buf.data(), work.data() + w * N, c.itw.data() + (w % L) * N, lp[w % L]);
    for (size_t v = 0; v < n_vec; ++v)
        ckks_dec_fft_body<LOGN, 512>(fft, a.data(), work.data() + v * L * N, reinterpret_cast<Cplx *>(slots) + v * (N / 2), c.ctw.data(),
                                     c.tj.data(), lp.data(), K, L);
}
}  // namespace

extern "C" {

void *emu_ckks_create(unsigned log_n, unsigned L, const uint64_t *moduli) { return make(log_n, L, moduli); }
void emu_ckks_destroy(void *h) { delete (Ctx *)h; }
// the product's twiddle table: N pairs (cos, sin)(pi k / N)
void emu_ckks_twiddles(void *h, double *out) {
    const Ctx *c = (const Ctx *)h;
    for (size_t k = 0; k < c->ctw.size(); ++k) {
        out[2 * k] = c->ctw[k].re;
        out[2 * k + 1] = c->ctw[k].im;
    }
}
int emu_ckks_encode(void *h, const double *slots, uint64_t *pt, size_t n_vec, double scale) {
    Ctx &c = *(Ctx *)h;
    switch (c.hp.log_n) {
        case 12: encode<12>(c, slots, pt, n_vec, scale); return 0;
        case 13: encode<13>(c, slots, pt, n_vec, scale); return 0;
        case 14: encode<14>(c, slots, pt, n_vec, scale); return 0;
    }
    return -1;
}
int emu_ckks_decode(void *h, const uint64_t *pt, double *slots, size_t n_vec, double scale) {
    Ctx &c = *(Ctx *)h;
    switch (c.hp.log_n) {
        case 12: decode<12>(c, pt, slots, n_vec, scale); return 0;
        case 13: decode<13>(c, pt, slots, n_vec, scale); return 0;
        case 14: decode<14>(c, pt, slots, n_vec, scale); return 0;
    }
    return -1;
}
}
