// emu_lincomb.cpp — host emulator of the scalar linear-combination body (TEST INFRASTRUCTURE ONLY).
//
// Runs lincomb_chunk of deeppowers_b200/csrc/eval.cuh chunk by chunk, as the grid of eval.cu does, with the coefficient pairs from the
// product's build_lincomb_coeffs.  Built by tests/test_polyeval_cpu.py once per arithmetic variant; never linked into libdpfhe.so.
#include <cstdint>
#include <vector>

#include "eval.cuh"
#include "host_params.hpp"

using namespace dpfhe;
using namespace dpfhe::DPFHE_VNS;

extern "C" {

// out [batch][2][L][N] = sum_i coeffs[i] in[i] + constant (+ pt) on c0; out may be one of the inputs.  0 on success
int emu_lincomb(unsigned log_n, unsigned L, const uint64_t *moduli, unsigned n_terms, const uint64_t *const *in, const int64_t *coeffs,
                int64_t constant, const uint64_t *pt, uint64_t *out, size_t batch) {
    HostParams hp;
    if (!build_host_params(log_n, L, moduli, hp).empty() || n_terms < 1 || n_terms > (unsigned)LINCOMB_MAX_TERMS) return -1;
    std::vector<LimbParams> lps(L);
    for (unsigned l = 0; l < L; ++l) lps[l] = hp.limbs[l].lp;
    auto *A = new LincombArgs<LINCOMB_MAX_TERMS>();
    build_lincomb_coeffs(lps.data(), L, coeffs, n_terms, constant, *A);
    for (unsigned i = 0; i < n_terms; ++i) A->in[i] = reinterpret_cast<const U64x2 *>(in[i]);
    A->out = reinterpret_cast<U64x2 *>(out);
    A->pt = reinterpret_cast<const U64x2 *>(pt);
    A->log_half = log_n - 1;
    A->n_chunks = batch * 2 * L * ((size_t)1 << (log_n - 1));
    for (size_t c = 0; c < A->n_chunks; ++c) A->out[c] = lincomb_chunk(*A, c, lps[(c >> A->log_half) % L]);
    delete A;
    return 0;
}
}
