// devarith.cu — the product's scalar arithmetic and register-level transform pieces, run element-wise on the device and
// on the host (TEST INFRASTRUCTURE ONLY).
//
// modarith.cuh and ntt_core.cuh are __host__ __device__, but much of their device code is different code from the host's
// (inline PTX carry and borrow chains, __umul64hi, __umulhi, __funnelshift_r).  This harness calls the product's own
// functions from one dispatcher, `apply`, compiled for both sides of the same translation unit, so that the device output
// can be compared with the host output word for word (tests/test_gpu_devarith.py) and the host output with exact integers
// and with the emulator (tests/test_devarith_cpu.py).  Nothing here re-implements the arithmetic.  It is built once per
// arithmetic variant (-DDPFHE_FAST=0 / 1) into tests/_devarith/ by tests/devarith/harness.py and is never linked into
// libdpfhe.so.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <vector>

#include "host_params.hpp"
#include "kernel_bodies.cuh"

using namespace dpfhe;
using namespace dpfhe::DPFHE_VNS;

namespace {

// X(name, input words, output words).  The fwd16 entries are the entry bounds the product instantiates:
// fwd_bound_after(BIN, K + 0/4/8) for BIN in {1, 3, 4} and K = LOGN - 12 in {0, 1, 2} (ntt_core.cuh, fwd_passes_blk).
#define DEVARITH_OPS(X)                                                                                                \
    X(umulhi64, 2, 1) X(mulhi_approx, 2, 1) X(csub, 2, 1) X(mad_lo64, 3, 1) X(sub_mul_q, 2, 1)                         \
    X(shoup_exact, 3, 1) X(shoup_lazy, 3, 1) X(mul128, 2, 2) X(sub128, 4, 2) X(barrett_lazy, 2, 1)                     \
    X(barrett_lazy_long, 2, 1) X(mulmod_lazy, 2, 1) X(mulmod, 2, 1) X(word_reduce, 1, 1) X(canon, 1, 1)                \
    X(canon4, 1, 1) X(canon_near60, 1, 1) X(canon_store, 1, 1) X(pti_fold, 4, 1) X(bgv_lift, 2, 1)                     \
    X(ct_bfly, 4, 2) X(gs_bfly, 4, 2) X(inv16, 46, 16) X(inv_final_product, 3, 1)                                      \
    X(fwd16_1, 46, 16) X(fwd16_3, 46, 16) X(fwd16_4, 46, 16) X(fwd16_5, 46, 16) X(fwd16_7, 46, 16)                     \
    X(fwd16_8, 46, 16) X(fwd16_9, 46, 16) X(fwd16_11, 46, 16) X(fwd16_12, 46, 16) X(fwd16_16, 46, 16)                  \
    X(mulhi32, 2, 1) X(shoup32, 3, 1) X(add32, 2, 1) X(sub32, 2, 1) X(reduce64_32, 1, 1)

enum Op {
#define X(name, nin, nout) OP_##name,
    DEVARITH_OPS(X)
#undef X
    OP_COUNT
};
const char *const OP_NAMES[] = {
#define X(name, nin, nout) #name,
    DEVARITH_OPS(X)
#undef X
};
constexpr int OP_NIN[] = {
#define X(name, nin, nout) nin,
    DEVARITH_OPS(X)
#undef X
};
constexpr int OP_NOUT[] = {
#define X(name, nin, nout) nout,
    DEVARITH_OPS(X)
#undef X
};
constexpr int FIRST_U32_OP = OP_mulhi32;   // ops from here on run modulo a plaintext modulus t (Mod32), the others modulo a limb

struct Params {
    LimbParams lp;
    Mod32 m;
};

// 16 values, then 15 twiddles w and their Shoup companions: stage u, sub-group j uses entry 2^u - 1 + j
template <int BIN>
DPFHE_HD void run_fwd16(const u64 *in, u64 *out, const LimbParams &p) {
    u64 x[16];
    for (int k = 0; k < 16; ++k) x[k] = in[k];
    fwd16<BIN>(x, p, [&](int u, int j) { return Twiddle{in[16 + (1 << u) - 1 + j], in[31 + (1 << u) - 1 + j]}; });
    for (int k = 0; k < 16; ++k) out[k] = x[k];
}

DPFHE_HD void apply(int op, const Params &P, const u64 *in, u64 *out) {
    const LimbParams &p = P.lp;
    switch (op) {
        case OP_umulhi64: out[0] = umulhi64(in[0], in[1]); break;
        case OP_mulhi_approx: out[0] = mulhi_approx(in[0], in[1]); break;
        case OP_csub: out[0] = csub(in[0], in[1]); break;
        case OP_mad_lo64: out[0] = mad_lo64(in[0], in[1], in[2]); break;
        case OP_sub_mul_q: out[0] = sub_mul_q(in[0], in[1], p); break;
        case OP_shoup_exact: out[0] = shoup_exact(in[0], in[1], in[2], p); break;
        case OP_shoup_lazy: out[0] = shoup_lazy(in[0], in[1], in[2], p); break;
        case OP_mul128: mul128(in[0], in[1], out[0], out[1]); break;
        case OP_sub128: {
            u64 hi = in[0], lo = in[1];
            sub128(hi, lo, in[2], in[3]);
            out[0] = hi;
            out[1] = lo;
            break;
        }
        case OP_barrett_lazy: out[0] = barrett_lazy(in[0], in[1], p); break;
        case OP_barrett_lazy_long: out[0] = barrett_lazy_long(in[0], in[1], p); break;
        case OP_mulmod_lazy: out[0] = mulmod_lazy(in[0], in[1], p); break;
        case OP_mulmod: out[0] = mulmod(in[0], in[1], p); break;
        case OP_word_reduce: out[0] = word_reduce(in[0], p); break;
        case OP_canon: out[0] = canon(in[0], p); break;
        case OP_canon4: out[0] = canon4(in[0], p); break;
        case OP_canon_near60: out[0] = canon_near60(in[0], p); break;
        case OP_canon_store: out[0] = canon_store(in[0], p); break;
        case OP_pti_fold: out[0] = pti_fold(in[0], in[1], in[2], in[3], p); break;
        case OP_bgv_lift: out[0] = bgv_lift((u32)in[0], (u32)in[1], p); break;
        case OP_ct_bfly:
        case OP_gs_bfly: {
            u64 x = in[0], y = in[1];
            const Twiddle w{in[2], in[3]};
            if (op == OP_ct_bfly) ct_bfly(x, y, w, p);
            else gs_bfly(x, y, w, p);
            out[0] = x;
            out[1] = y;
            break;
        }
        case OP_inv16: {
            u64 x[16];
            for (int k = 0; k < 16; ++k) x[k] = in[k];
            inv16(x, p, [&](int u, int j) { return Twiddle{in[16 + (1 << u) - 1 + j], in[31 + (1 << u) - 1 + j]}; });
            for (int k = 0; k < 16; ++k) out[k] = x[k];
            break;
        }
        case OP_inv_final_product: out[0] = inv_final_product(in[0], in[1], in[2], p); break;
        case OP_fwd16_1: run_fwd16<1>(in, out, p); break;
        case OP_fwd16_3: run_fwd16<3>(in, out, p); break;
        case OP_fwd16_4: run_fwd16<4>(in, out, p); break;
        case OP_fwd16_5: run_fwd16<5>(in, out, p); break;
        case OP_fwd16_7: run_fwd16<7>(in, out, p); break;
        case OP_fwd16_8: run_fwd16<8>(in, out, p); break;
        case OP_fwd16_9: run_fwd16<9>(in, out, p); break;
        case OP_fwd16_11: run_fwd16<11>(in, out, p); break;
        case OP_fwd16_12: run_fwd16<12>(in, out, p); break;
        case OP_fwd16_16: run_fwd16<16>(in, out, p); break;
        case OP_mulhi32: out[0] = mulhi32((u32)in[0], (u32)in[1]); break;
        case OP_shoup32: out[0] = shoup32((u32)in[0], (u32)in[1], (u32)in[2], P.m.t); break;
        case OP_add32: out[0] = add32((u32)in[0], (u32)in[1], P.m.t); break;
        case OP_sub32: out[0] = sub32((u32)in[0], (u32)in[1], P.m.t); break;
        case OP_reduce64_32: out[0] = reduce64_32(in[0], P.m); break;
    }
}

// one case per index; the indices do not depend on the data
__global__ void apply_kernel(int op, int nin, int nout, Params P, const u64 *__restrict__ in, u64 *__restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        apply(op, P, in + i * nin, out + i * nout);
}

struct Harness {
    HostParams hp;
    std::vector<Mod32> m32;
};

bool params_of(const Harness *h, int op, unsigned idx, Params &P) {
    if (op < 0 || op >= OP_COUNT) return false;
    memset(&P, 0, sizeof(P));
    if (op >= FIRST_U32_OP) {
        if (idx >= h->m32.size()) return false;
        P.m = h->m32[idx];
    } else {
        if (idx >= h->hp.L) return false;
        P.lp = h->hp.limbs[idx].lp;
    }
    return true;
}

}  // namespace

extern "C" {

int devarith_fast() { return DPFHE_FAST; }
int devarith_op_count() { return OP_COUNT; }
const char *devarith_op_name(int op) { return op >= 0 && op < OP_COUNT ? OP_NAMES[op] : nullptr; }
int devarith_op_nin(int op) { return op >= 0 && op < OP_COUNT ? OP_NIN[op] : -1; }
int devarith_op_nout(int op) { return op >= 0 && op < OP_COUNT ? OP_NOUT[op] : -1; }

// L moduli (limb parameters derived by the product's host code for N = 4096) and n_t plaintext moduli (their Mod32).  Returns
// null when the product rejects a modulus, and in the fast build when a modulus is not k * 2^32 + 1 (as emu_create).
void *devarith_create(unsigned L, const uint64_t *moduli, unsigned n_t, const uint64_t *ts) {
    Harness *h = new Harness();
    if (L == 0 || !build_host_params(12, L, moduli, h->hp).empty()) {
        delete h;
        return nullptr;
    }
#if DPFHE_FAST
    for (unsigned l = 0; l < L; ++l)
        if (h->hp.limbs[l].lp.nqh == 0) {
            delete h;
            return nullptr;
        }
#endif
    for (unsigned k = 0; k < n_t; ++k) h->m32.push_back(make_mod32(ts[k]));
    return h;
}
void devarith_destroy(void *h) { delete (Harness *)h; }

// the limb constants as the product derives them, 14 words (types.hpp: LimbParams)
int devarith_limb_params(void *h, unsigned l, uint64_t *out) {
    const Harness *H = (const Harness *)h;
    if (l >= H->hp.L) return -1;
    static_assert(sizeof(LimbParams) == 14 * 8, "LimbParams layout");
    memcpy(out, &H->hp.limbs[l].lp, sizeof(LimbParams));
    return 0;
}
// Mod32 of plaintext modulus k: t, r32, r32_s, one_s
int devarith_mod32(void *h, unsigned k, uint32_t *out) {
    const Harness *H = (const Harness *)h;
    if (k >= H->m32.size()) return -1;
    const Mod32 &m = H->m32[k];
    out[0] = m.t;
    out[1] = m.r32;
    out[2] = m.r32_s;
    out[3] = m.one_s;
    return 0;
}

// the host build of `apply` over n cases
int devarith_run_host(void *h, int op, unsigned idx, const uint64_t *in, uint64_t *out, size_t n) {
    Params P;
    if (!params_of((const Harness *)h, op, idx, P)) return -1;
    for (size_t i = 0; i < n; ++i) apply(op, P, in + i * OP_NIN[op], out + i * OP_NOUT[op]);
    return 0;
}

// the device build of `apply` over n cases on the current device: allocate, copy, launch, synchronise, free.  Returns the
// CUDA error code (0 on success), or -1 for an unknown op or index.
int devarith_run_device(void *h, int op, unsigned idx, const uint64_t *in, uint64_t *out, size_t n) {
    Params P;
    if (!params_of((const Harness *)h, op, idx, P)) return -1;
    if (n == 0) return 0;
    const size_t in_bytes = n * OP_NIN[op] * sizeof(u64), out_bytes = n * OP_NOUT[op] * sizeof(u64);
    u64 *d_in = nullptr, *d_out = nullptr;
    cudaError_t err = cudaMalloc(&d_in, in_bytes);
    if (err == cudaSuccess) err = cudaMalloc(&d_out, out_bytes);
    if (err == cudaSuccess) err = cudaMemcpy(d_in, in, in_bytes, cudaMemcpyHostToDevice);
    if (err == cudaSuccess) err = cudaMemset(d_out, 0xFF, out_bytes);
    if (err == cudaSuccess) {
        const unsigned threads = 256;
        const size_t want = (n + threads - 1) / threads;
        apply_kernel<<<(unsigned)(want < 4096 ? want : 4096), threads>>>(op, OP_NIN[op], OP_NOUT[op], P, d_in, d_out, n);
        err = cudaGetLastError();
    }
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    if (err == cudaSuccess) err = cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost);
    cudaFree(d_in);
    cudaFree(d_out);
    return (int)err;
}

}  // extern "C"
