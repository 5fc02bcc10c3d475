// emu_rotate_sum.cpp — host emulator of the summed rotations (TEST INFRASTRUCTURE ONLY).
//
// Runs the bodies of dpfhe_rotate_sum_grouped's four kernels (deeppowers_b200/csrc/kernel_bodies.cuh) in kernel order with a
// sequential CTA policy: hoistg_phase1/2 in the role order of ks_hoistg_kernel, rot_sum_grouped_rows over the work items of
// rot_sum_grouped_kernel (one ciphertext x one limb), then the md_tau / md_limb bodies.  Built by tests/test_rotate_sum_cpu.py once
// per arithmetic variant; never linked into libdpfhe.so.
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

// NT_MD: the threads of the mod-down kernels (512 at N = 16384, as launch_mod_down_special)
template <int LOGN, int NT, int NT_MD>
void run_rotate_sum(Ctx &e, unsigned Ks, const uint64_t *ct, unsigned n_rot, const uint64_t *galois, const uint64_t *keys, uint64_t *out, size_t batch,
                    uint64_t t_plain) {
    const size_t N = (size_t)1 << LOGN;
    const unsigned L = e.hp.L, Lq = L - Ks;
    MsConsts K;
    GroupConsts G;
    build_group_consts(e.hp, Ks, t_plain, G, K);
    const unsigned dnum = G.dnum;
    const size_t P = (size_t)L * N, key_words = (size_t)2 * dnum * L * N;
    uint64_t *buf = aligned_new<uint64_t>(N), *scratch = aligned_new<uint64_t>((size_t)L * 2 * N);
    uint64_t *U = aligned_new<uint64_t>(batch * dnum * L * N), *acc = aligned_new<uint64_t>(batch * 2 * P), *tau = aligned_new<uint64_t>((size_t)Ks * N);
    uint64_t *key_s = aligned_new<uint64_t>(n_rot * key_words);   // Shoup companions, as key_prepare_kernel builds them
    for (size_t k = 0; k < n_rot * key_words; ++k) key_s[k] = (uint64_t)((((unsigned __int128)keys[k]) << 64) / e.lp[(k / N) % L].q);
    HoistGArgs H;
    H.ct = ct; H.U = U; H.scratch = scratch; H.tw = e.tw; H.itw = e.itw;
    HostCta cta{NT}, cta_md{NT_MD};
    for (size_t c = 0; c < batch; ++c) {
        const unsigned par = (unsigned)(c & 1);
        const uint64_t *t_rows = scratch + (size_t)par * N;
        for (unsigned i = 0; i < Lq; ++i) hoistg_phase1<LOGN, NT>(cta, buf, H, G, c, i, scratch + ((size_t)i * 2 + par) * N);
        for (unsigned i = 0; i < L; ++i)
            for (unsigned g = 0; g < dnum; ++g)
                if (i >= Lq || i / Ks != g) hoistg_phase2<LOGN, NT>(cta, buf, H, G, e.lp[i], c, i, g, t_rows, 2 * N);
    }
    RotSumGArgs A;
    memset(&A, 0, sizeof(A));
    A.ct = ct; A.U = U; A.acc = acc; A.n_rot = n_rot;
    for (unsigned m = 0; m < n_rot; ++m) {
        A.key[m] = keys + m * key_words;
        A.key_s[m] = key_s + m * key_words;
        A.galois[m] = (uint32_t)galois[m];
    }
    for (size_t c = 0; c < batch; ++c)
        for (unsigned i = 0; i < L; ++i) rot_sum_grouped_rows<LOGN, NT, 1>(cta, A, G, K, e.lp[i], c, 1, i);
    for (size_t w = 0; w < 2 * batch; ++w) {   // the division by P, one polynomial at a time
        for (unsigned k = 0; k < Ks; ++k)
            ms_tau_body<LOGN, NT_MD>(cta_md, buf, acc + (w * L + Lq + k) * N, nullptr, e.itw + (size_t)(Lq + k) * N, G.lp_up[Lq + k], tau + (size_t)k * N, K);
        for (unsigned i = 0; i < Lq; ++i)
            ms_limb_group<LOGN, NT_MD, false>(cta_md, buf, tau, N, acc + (w * L + i) * N, out + (w * Lq + i) * N, e.tw + (size_t)i * N, e.lp[i], K, G, i);
    }
    free(buf); free(scratch); free(U); free(acc); free(tau); free(key_s);
}
}  // namespace

extern "C" {

void *emu_rs_create(unsigned log_n, unsigned L, const uint64_t *moduli) {
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
void emu_rs_destroy(void *h) { delete (Ctx *)h; }

// the trim schedule of rot_sum_grouped_rows (LazyBound) over n additions: trim[k] = 1 where the row takes csub(8q) after addition k;
// returns SB, the bound of one Shoup product in multiples of q
int emu_rs_schedule(unsigned n, int *trim) {
    LazyBound b;
    for (unsigned k = 0; k < n; ++k) trim[k] = b.add() ? 1 : 0;
    return SB;
}

// the summed multiply-accumulate alone on given lifts U [batch][dnum][L][N]: acc [batch][2][L][N] (the lazy bound's threshold test)
int emu_rs_mac(void *h, unsigned K, const uint64_t *ct, const uint64_t *U, unsigned n_rot, const uint64_t *galois, const uint64_t *keys,
               uint64_t *acc, size_t batch) {
    Ctx *e = (Ctx *)h;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > e->hp.L || n_rot < 1 || n_rot > (unsigned)ROT_SUM_MAX) return -1;
    MsConsts Kc;
    GroupConsts G;
    build_group_consts(e->hp, K, 0, G, Kc);
    const unsigned L = e->hp.L;
    const size_t N = (size_t)1 << e->hp.log_n, key_words = (size_t)2 * G.dnum * L * N;
    std::vector<uint64_t> key_s(n_rot * key_words);
    for (size_t k = 0; k < key_s.size(); ++k) key_s[k] = (uint64_t)((((unsigned __int128)keys[k]) << 64) / e->lp[(k / N) % L].q);
    RotSumGArgs A;
    memset(&A, 0, sizeof(A));
    A.ct = ct; A.U = U; A.acc = acc; A.n_rot = n_rot;
    for (unsigned m = 0; m < n_rot; ++m) {
        A.key[m] = keys + m * key_words;
        A.key_s[m] = key_s.data() + m * key_words;
        A.galois[m] = (uint32_t)galois[m];
    }
    HostCta cta{256};
    for (size_t c = 0; c < batch; ++c)
        for (unsigned i = 0; i < L; ++i) {
            switch (e->hp.log_n) {
                case 12: rot_sum_grouped_rows<12, 256, 1>(cta, A, G, Kc, e->lp[i], c, 1, i); break;
                case 13: rot_sum_grouped_rows<13, 256, 1>(cta, A, G, Kc, e->lp[i], c, 1, i); break;
                case 14: rot_sum_grouped_rows<14, 256, 1>(cta, A, G, Kc, e->lp[i], c, 1, i); break;
                default: return -1;
            }
        }
    return 0;
}

// out [batch][2][L-K][N] = ct + sum_m rot_m(ct) through the kernel bodies; keys [n_rot][dnum][2][L][N]
int emu_rs_rotate_sum(void *h, unsigned K, const uint64_t *ct, unsigned n_rot, const uint64_t *galois, const uint64_t *keys, uint64_t *out,
                      size_t batch, uint64_t t_plain) {
    Ctx *e = (Ctx *)h;
    if (K < 1 || K > (unsigned)KS_MAX_SPECIAL || 2 * K > e->hp.L || n_rot < 1 || n_rot > (unsigned)ROT_SUM_MAX) return -1;
    switch (e->hp.log_n) {
        case 12: run_rotate_sum<12, 256, 256>(*e, K, ct, n_rot, galois, keys, out, batch, t_plain); return 0;
        case 13: run_rotate_sum<13, 256, 256>(*e, K, ct, n_rot, galois, keys, out, batch, t_plain); return 0;
        case 14: run_rotate_sum<14, 256, 512>(*e, K, ct, n_rot, galois, keys, out, batch, t_plain); return 0;
    }
    return -1;
}
}
