// emu_ckks_comb.cpp — host emulator of the CKKS combination fused into the final rescale (TEST INFRASTRUCTURE ONLY).
//
// Runs ckks_comb_tau_body and ckks_comb_limb_body of deeppowers_b200/csrc/eval.cuh CTA by CTA, as the grids of eval.cu do (same
// thread counts), with the coefficient pairs from the product's build_ckks_comb_coeffs and the rescale constants from
// build_ms_consts(t = 0).  Also exports the product's host rounding and exact reduction of the coefficients.  Built by
// tests/test_ckks_comb_emu_cpu.py once per arithmetic variant; never linked into libdpfhe.so.
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "eval.cuh"
#include "host_params.hpp"

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

template <int LOGN, int NT>
void run(const HostParams &hp, const CkksCombArgs<CKKS_COMB_MAX_TERMS> &A, uint64_t *tau, uint64_t *out, size_t n_polys) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned Lc = A.Lc, Lo = Lc - 1;
    std::vector<uint64_t> buf(N);
    HostCta cta{NT};
    for (size_t w = 0; w < n_polys; ++w)
        ckks_comb_tau_body<LOGN, NT>(cta, buf.data(), A, w, hp.limbs[Lc - 1].itw.data(), hp.limbs[Lc - 1].lp, tau + w * N);
    for (size_t w = 0; w < n_polys * Lo; ++w) {
        const size_t poly = w / Lo;
        const unsigned i = (unsigned)(w % Lo);
        ckks_comb_limb_body<LOGN, NT>(cta, buf.data(), A, poly, i, tau + poly * N, out + (poly * Lo + i) * N, hp.limbs[i].tw.data(), hp.limbs[i].lp);
    }
}
}  // namespace

extern "C" {

// out [batch][2][Lc-1][N] = mod_switch_down_{t=0}(sum_i coeffs[i] in[i]|_Lc + constant on c0) over moduli q_0 .. q_{Lc-1};
// in[i] is [batch][2][levels[i]][N].  0 on success
int emu_ckks_comb(unsigned log_n, unsigned Lc, const uint64_t *moduli, unsigned n_terms, const uint64_t *const *in, const unsigned *levels,
                  const double *coeffs, double constant, uint64_t *out, size_t batch) {
    HostParams hp;
    if (!build_host_params(log_n, Lc, moduli, hp).empty() || Lc < 2 || n_terms < 1 || n_terms > (unsigned)CKKS_COMB_MAX_TERMS) return -1;
    for (unsigned i = 0; i < n_terms; ++i)
        if (levels[i] < Lc) return -1;
    std::vector<LimbParams> lps(Lc);
    for (unsigned l = 0; l < Lc; ++l) lps[l] = hp.limbs[l].lp;
    auto *A = new CkksCombArgs<CKKS_COMB_MAX_TERMS>();
    build_ckks_comb_coeffs(lps.data(), Lc, coeffs, n_terms, constant, *A);
    for (unsigned i = 0; i < n_terms; ++i) {
        A->in[i] = reinterpret_cast<const U64x2 *>(in[i]);
        A->Lk[i] = levels[i];
    }
    A->log_half = log_n - 1;
    build_ms_consts(hp, 0, A->K);
    const size_t n_polys = 2 * batch;
    std::vector<uint64_t> tau(n_polys << log_n);
    int rc = 0;
    switch (log_n) {
        case 12: run<12, 256>(hp, *A, tau.data(), out, n_polys); break;
        case 13: run<13, 256>(hp, *A, tau.data(), out, n_polys); break;
        case 14: run<14, 512>(hp, *A, tau.data(), out, n_polys); break;
        default: rc = -1;
    }
    delete A;
    return rc;
}

// the product's exact reduction of an integer-valued double, and its rounding of a combination coefficient
uint64_t emu_double_mod(double x, uint64_t q) { return double_mod(x, q); }
double emu_ckks_comb_coeff(double a, double m, double s) { return ckks_comb_coeff(a, m, s); }
}
