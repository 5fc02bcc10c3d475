// kernels.cu — sm_90a kernels and their launchers (DESIGN.md §4).
//
// No tensor cores (pure 64-bit modular integer work), no Triton, no CPU fallback.
//   ntt_kernel            one CTA per limb transform, limb resident in swizzled shared memory
//   ks_fused_kernel       persistent cooperative kernel: tensor / permute -> INTT -> publish digit
//                         -> (L-1) x [lift + NTT + multiply-accumulate with the switch key] -> out
//   pointwise kernels     128-bit vectorised grid-stride loops
#include <cooperative_groups.h>
#include <cuda.h>   // CUtensorMap (types only: the driver entry point is fetched at run time, libcuda is not linked)
#include <cuda_runtime.h>

#include <atomic>

#include "kernel_bodies.cuh"
#include "launch_util.hpp"

// The file is large (every kernel x three ring degrees x three modes); the build compiles it in two parts per variant, in parallel:
// -DDPFHE_PART=1 everything but the special-prime key-switch family, 2 its one-special-prime kernel, 3 the grouped kernels; no flag = all.
#ifndef DPFHE_PART
#define DPFHE_PART 0
#endif
#define DPFHE_PART_MAIN (DPFHE_PART == 0 || DPFHE_PART == 1)
#define DPFHE_PART_HYBRID (DPFHE_PART == 0 || DPFHE_PART == 2)
#define DPFHE_PART_GROUPED (DPFHE_PART == 0 || DPFHE_PART == 3)

// compiled twice: -DDPFHE_FAST=0 -> namespace dpfhe::gen, -DDPFHE_FAST=1 -> namespace dpfhe::fast (types.hpp)
namespace dpfhe {
namespace DPFHE_VNS {

// The protocol of the persistent kernels (DESIGN.md §4.4, §4.7): tickets, mailboxes and flags carry 32-bit round numbers.
__device__ __forceinline__ u32 ld_acquire_u32(const u32 *p) {
    u32 v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(u32 *p, u32 v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ u64 ld_acquire_u64(const u64 *p) {
    u64 v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u64(u64 *p, u64 v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// the calling thread waits until *flag has reached round `tag`; the signed difference keeps the comparison right across wrap-around
__device__ __forceinline__ void spin_until(const u32 *flag, u32 tag) {
    while ((int)(ld_acquire_u32(flag) - tag) < 0) {
    }
}
// thread k < count waits for flags[k], then the CTA meets at a barrier
__device__ __forceinline__ void wait_flags(const u32 *flags, u32 count, u32 tag) {
    if (threadIdx.x < count) spin_until(flags + threadIdx.x, tag);
    __syncthreads();
}
// makes the CTA's global stores visible, then thread 0 release-stores round `tag` to *flag
__device__ __forceinline__ void publish_flag(u32 *flag, u32 tag) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) st_release_u32(flag, tag);
}
// the ciphertext of round `tag`, returned to every thread: the group's leader draws it from the global ticket counter and, if
// `post`, posts it tagged with the round in the mailbox box(); the other members spin until that tag appears there.  Only thread 0
// evaluates box(), so the mailbox address is not held in a register through the rest of the round.
template <class Box>
__device__ __forceinline__ u32 draw_ticket(u32 *ticket, Box box, u32 tag, bool leader, bool post) {
    __shared__ u32 s_ct;
    if (threadIdx.x == 0) {
        u64 *const mb = box();
        if (leader) {
            const u32 t = atomicAdd(ticket, 1u);
            if (post) st_release_u64(mb, ((u64)tag << 32) | t);
            s_ct = t;
        } else {
            u64 m;
            do m = ld_acquire_u64(mb);
            while ((u32)(m >> 32) != tag);
            s_ct = (u32)m;
        }
    }
    __syncthreads();
    return s_ct;
}

// barrier scopes of the CTA policy (ntt_core.cuh): CTA, 256-thread domain, warp.
// PROF: thread 0 accumulates clock64() deltas per phase id into prof[blockIdx][id] (diagnostics only).
template <int NT, bool PROF = false>
struct DevCta {
    unsigned long long *prof = nullptr;
    long long last = 0;
    unsigned long long t_start = 0, c_start = 0;
    __device__ __forceinline__ void prof_begin(unsigned long long *all) {
        if (PROF) {
            prof = all + (size_t)blockIdx.x * 16;
            last = clock64();
            c_start = (unsigned long long)last;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));
        }
    }
    __device__ __forceinline__ void prof_end() {
        if (PROF && threadIdx.x == 0) {   // CTA lifetime in nanoseconds (globaltimer) and in SM cycles
            unsigned long long t_end;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
            prof[14] += t_end - t_start;
            prof[15] += (unsigned long long)clock64() - c_start;
        }
    }
    __device__ __forceinline__ void mark(int id) {
        if (PROF && threadIdx.x == 0) {
            const long long now = clock64();
            prof[id] += (unsigned long long)(now - last);
            last = now;
        }
    }
    template <class F>
    __device__ __forceinline__ void par(F f) {
        f((int)threadIdx.x);
        __syncthreads();
    }
    // blocks the CTA until the monotone counter *flag has reached `target` (wrap-safe comparison)
    __device__ __forceinline__ void wait_ge(const u32 *flag, u32 target) { wait_flags(flag, 1, target); }
    template <class F>
    __device__ __forceinline__ void par_dom(F f) {
        f((int)threadIdx.x);
        if (NT <= 256) __syncthreads();
        else asm volatile("bar.sync %0, 256;" ::"r"(1 + ((int)threadIdx.x >> 8)) : "memory");
    }
    template <class F>
    __device__ __forceinline__ void par_warp(F f) {
        f((int)threadIdx.x);
        __syncwarp();
    }
};

#if DPFHE_PART_MAIN
// ------------------------------------------------------------------ standalone transforms
// The per-limb constants travel in the kernel parameter block (constant bank), so q, 2q, 8q ...
// are read through uniform registers / constant operands instead of occupying vector registers.
template <int LOGN, int NT, int MINB, bool INVERSE>
__global__ void __launch_bounds__(NT, MINB) ntt_kernel(u64 *data, const Twiddle *__restrict__ tables,
                                                        const __grid_constant__ LimbTable lt, u32 L, size_t n_limbs) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    for (size_t w = blockIdx.x; w < n_limbs; w += gridDim.x) {
        const u32 l = (u32)(w % L);
        const LimbParams &p = lt.lp[l];
        if (INVERSE) ntt_inv_body<LOGN, NT>(cta, buf, data + w * N, tables + (size_t)l * N, p);
        else ntt_fwd_body<LOGN, NT>(cta, buf, data + w * N, tables + (size_t)l * N, p);
    }
}

// Inverse transform whose input copy is done by the TMA unit: the swizzled shared-memory layout of ntt_core.cuh IS the layout a
// 2-D tensor map with CU_TENSOR_MAP_SWIZZLE_128B produces (rows of 128 bytes = 16 coefficients, 16-byte chunk index XOR row & 7),
// so one elected thread issues cp.async.bulk.tensor for the whole limb (boxes of 256 rows = 32 KiB) and everybody waits on the
// mbarrier, instead of 256 threads looping over LDG.128 + STS.128.  One limb per CTA (grid = n_limbs): the barrier is used once.
__device__ __forceinline__ u32 smem_addr(const void *p) { return (u32)__cvta_generic_to_shared(p); }

template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ntt_inv_tma_kernel(const __grid_constant__ CUtensorMap tm, u64 *data, const Twiddle *__restrict__ itw,
                                                                const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ __align__(8) unsigned long long bar;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    constexpr int ROWS = (int)(N * 8 / 128), BOX_ROWS = ROWS < 256 ? ROWS : 256, BOXES = ROWS / BOX_ROWS;
    DevCta<NT> cta;
    const size_t w = blockIdx.x;
    const u32 l = (u32)(w % L);
    const u32 bar_a = smem_addr(&bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"((u32)(N * 8)) : "memory");
#pragma unroll
        for (int b = 0; b < BOXES; ++b) {
            const int row = (int)(w * ROWS) + b * BOX_ROWS;
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                         ::"r"(smem_addr(smem_raw + (size_t)b * BOX_ROWS * 128)), "l"(reinterpret_cast<unsigned long long>(&tm)), "r"(0), "r"(row), "r"(bar_a)
                         : "memory");
        }
    }
    {   // every thread waits for the bytes to land (phase 0 of the barrier)
        u32 done = 0;
        while (!done) {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done)
                         : "r"(bar_a)
                         : "memory");
        }
    }
    ntt_inv_resident<LOGN, NT>(cta, buf, data + w * N, itw + (size_t)l * N, lt.lp[l]);
}

// N = 16384: one limb per CLUSTER of two CTAs (64 KiB of shared memory each, so three CTAs still share an SM); see
// kernel_bodies.cuh "transforms by a PAIR of CTAs".  The inverse reads the partner's half through distributed shared memory.
template <int NT, int MINB, bool INVERSE>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(NT, MINB)
    ntt_pair_kernel(u64 *data, const Twiddle *__restrict__ tables, const __grid_constant__ LimbTable lt, u32 L, size_t n_limbs) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << NTT_PAIR_LOGN;
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int h = (int)cluster.block_rank();
    const u64 *peer = cluster.map_shared_rank(buf, h ^ 1);
    DevCta<NT> cta;
    for (size_t w = blockIdx.x / 2; w < n_limbs; w += gridDim.x / 2) {
        const u32 l = (u32)(w % L);
        const LimbParams &p = lt.lp[l];
        const Twiddle *tw = tables + (size_t)l * N;
        if (!INVERSE) {
            ntt_fwd_half_load<NT>(cta, buf, data + w * N, tw, p, h);
            cluster.sync();   // both CTAs have read the whole limb: the in-place stores may begin
            ntt_fwd_half_finish<NT>(cta, buf, data + w * N, tw, p, h);
        } else {
            ntt_inv_half_passes<NT>(cta, buf, data + w * N, tw, p, h);
            cluster.sync();   // the partner's half is complete in its shared memory
            ntt_inv_half_outer<NT>(cta, buf, peer, data + w * N, tw, p, h);
            cluster.sync();   // the partner has finished reading this CTA's shared memory
        }
    }
}

// ------------------------------------------------------------------ modulus switching (two launches)
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ms_tau_kernel(const u64 *in, u64 *tau, const Twiddle *__restrict__ itw,
                                                           const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                           u32 L, size_t n_polys) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const LimbParams &p = lt.lp[L - 1];
    for (size_t w = blockIdx.x; w < n_polys; w += gridDim.x)
        ms_tau_body<LOGN, NT>(cta, buf, in + (w * L + (L - 1)) * N, nullptr, itw + (size_t)(L - 1) * N, p, tau + w * N, K);
}

template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ms_limb_kernel(const u64 *in, const u64 *tau, u64 *out, const Twiddle *__restrict__ tw,
                                                            const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                            u32 L, size_t n_items) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const u32 Lo = L - 1;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const size_t poly = w / Lo;
        const u32 i = (u32)(w % Lo);
        ms_limb_body<LOGN, NT>(cta, buf, tau + poly * N, in + (poly * L + i) * N, out + (poly * Lo + i) * N, tw + (size_t)i * N, lt.lp[i], K, i);
    }
}

// division by the product of the last K limbs (DESIGN.md §2.11): tau' of every special limb, then one item per kept limb
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) md_tau_kernel(const u64 *in, u64 *tau, const Twiddle *__restrict__ itw, const __grid_constant__ MsConsts K,
                                                           const __grid_constant__ GroupConsts G, size_t n_items) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const u32 L = G.Lq + G.K;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const size_t poly = w / G.K;
        const u32 s = G.Lq + (u32)(w % G.K);
        ms_tau_body<LOGN, NT>(cta, buf, in + (poly * L + s) * N, nullptr, itw + (size_t)s * N, G.lp_up[s], tau + w * N, K);
    }
}

template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) md_limb_kernel(const u64 *in, const u64 *tau, u64 *out, const Twiddle *__restrict__ tw,
                                                            const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                            const __grid_constant__ GroupConsts G, size_t n_items) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const u32 Lq = G.Lq, L = Lq + G.K;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const size_t poly = w / Lq;
        const u32 i = (u32)(w % Lq);
        ms_limb_group<LOGN, NT, false>(cta, buf, tau + poly * G.K * N, N, in + (poly * L + i) * N, out + (poly * Lq + i) * N, tw + (size_t)i * N,
                                       lt.lp[i], K, G, i);
    }
}

// ------------------------------------------------------------------ CKKS slot encoding (DESIGN.md §2.12, §4.8)
// One CTA per vector: its N/2 complex values (64 KiB at N = 8192, 128 KiB at N = 16384) stay in shared memory for all stages.
template <int LOGN, int NT>
__global__ void __launch_bounds__(NT, 1) ckks_enc_fft_kernel(const Cplx *slots, double *coeffs, const Cplx *__restrict__ tw,
                                                              const u32 *__restrict__ tj, double sc) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t v = blockIdx.x;
    ckks_enc_fft_body<LOGN, NT>(cta, reinterpret_cast<Cplx *>(smem_raw), slots + v * (N / 2), coeffs + v * N, tw, tj, sc);
}

// forward transform of one limb of one encoded vector, the coefficients reduced into the limb by the load stage
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ckks_enc_ntt_kernel(const double *coeffs, u64 *pt, const Twiddle *__restrict__ tw,
                                                                 const u64 *__restrict__ pow2, const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t w = blockIdx.x;
    const u32 l = (u32)(w % L);
    const LimbParams &p = lt.lp[l];
    const double *x = coeffs + (w / L) * N;
    const u64 *p2 = pow2 + (size_t)l * CKKS_POW2_E;
    auto src = [&](int c) {
        U64x2 r;
        r.x = ckks_reduce(x[2 * c], p, p2);
        r.y = ckks_reduce(x[2 * c + 1], p, p2);
        return r;
    };
    ntt_fwd_src_body<LOGN, NT>(cta, buf, src, pt + w * N, tw + (size_t)l * N, p);
}

// N = 16384: two CTAs per limb, each keeping half of the outer radix-4 step (as ntt_pair_kernel's forward half; the input is
// not overwritten, so the two CTAs need no cluster barrier)
template <int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ckks_enc_ntt_pair_kernel(const double *coeffs, u64 *pt, const Twiddle *__restrict__ tw,
                                                                      const u64 *__restrict__ pow2, const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << NTT_PAIR_LOGN;
    DevCta<NT> cta;
    const size_t w = blockIdx.x / 2;
    const int h = (int)(blockIdx.x & 1);
    const u32 l = (u32)(w % L);
    const LimbParams &p = lt.lp[l];
    const double *x = coeffs + (w / L) * N;
    const u64 *p2 = pow2 + (size_t)l * CKKS_POW2_E;
    auto src = [&](int c) {
        U64x2 r;
        r.x = ckks_reduce(x[2 * c], p, p2);
        r.y = ckks_reduce(x[2 * c + 1], p, p2);
        return r;
    };
    ntt_fwd_half_load_src<NT>(cta, buf, src, tw + (size_t)l * N, p, h);
    ntt_fwd_half_finish<NT>(cta, buf, pt + w * N, tw + (size_t)l * N, p, h);
}

// decode: Garner, centring, Horner, scaling and the forward special FFT of one vector; work [n_vec][L][N] holds the inverse
// transforms (overwritten by the mixed-radix digits)
template <int LOGN, int NT>
__global__ void __launch_bounds__(NT, 1) ckks_dec_kernel(u64 *work, Cplx *slots, const Cplx *__restrict__ tw, const u32 *__restrict__ tj,
                                                          const __grid_constant__ LimbTable lt, const __grid_constant__ CkksConsts K, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t v = blockIdx.x;
    ckks_dec_fft_body<LOGN, NT>(cta, reinterpret_cast<Cplx *>(smem_raw), work + v * L * N, slots + v * (N / 2), tw, tj, lt.lp, K, L);
}

// ------------------------------------------------------------------ BGV slot encoding (DESIGN.md §2.13, §4.9)
// One CTA per vector: its N words mod t (16 / 32 / 64 KiB at N = 4096 / 8192 / 16384) stay in shared memory for all stages.
template <int LOGN, int NT>
__global__ void __launch_bounds__(NT, 1) bgv_enc_kernel(const int64_t *slots, u32 *coeffs, const __grid_constant__ BgvTables T) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t v = blockIdx.x;
    bgv_enc_body<LOGN, NT>(cta, reinterpret_cast<u32 *>(smem_raw), slots + v * N, coeffs + v * N, T);
}

// forward transform of one limb of one encoded vector, the coefficients lifted (centred) into the limb by the load stage
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) bgv_enc_ntt_kernel(const u32 *coeffs, u64 *pt, const Twiddle *__restrict__ tw, u32 t,
                                                                const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t w = blockIdx.x;
    const u32 l = (u32)(w % L);
    const LimbParams &p = lt.lp[l];
    const uint2 *x = reinterpret_cast<const uint2 *>(coeffs + (w / L) * N);
    auto src = [&](int c) {
        const uint2 v = x[c];
        U64x2 r;
        r.x = bgv_lift(v.x, t, p);
        r.y = bgv_lift(v.y, t, p);
        return r;
    };
    ntt_fwd_src_body<LOGN, NT>(cta, buf, src, pt + w * N, tw + (size_t)l * N, p);
}

// N = 16384: two CTAs per limb, as ckks_enc_ntt_pair_kernel
template <int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) bgv_enc_ntt_pair_kernel(const u32 *coeffs, u64 *pt, const Twiddle *__restrict__ tw, u32 t,
                                                                     const __grid_constant__ LimbTable lt, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    constexpr size_t N = (size_t)1 << NTT_PAIR_LOGN;
    DevCta<NT> cta;
    const size_t w = blockIdx.x / 2;
    const int h = (int)(blockIdx.x & 1);
    const u32 l = (u32)(w % L);
    const LimbParams &p = lt.lp[l];
    const uint2 *x = reinterpret_cast<const uint2 *>(coeffs + (w / L) * N);
    auto src = [&](int c) {
        const uint2 v = x[c];
        U64x2 r;
        r.x = bgv_lift(v.x, t, p);
        r.y = bgv_lift(v.y, t, p);
        return r;
    };
    ntt_fwd_half_load_src<NT>(cta, buf, src, tw + (size_t)l * N, p, h);
    ntt_fwd_half_finish<NT>(cta, buf, pt + w * N, tw + (size_t)l * N, p, h);
}

// decode: Garner, centring, reduction mod t, the forward transform mod t and the slot gather of one vector; work [n_vec][L][N]
// holds the inverse transforms (overwritten by the mixed-radix digits)
template <int LOGN, int NT>
__global__ void __launch_bounds__(NT, 1) bgv_dec_kernel(u64 *work, u64 *slots, const __grid_constant__ BgvTables T, const __grid_constant__ LimbTable lt,
                                                         const __grid_constant__ BgvConsts K, u32 L) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    DevCta<NT> cta;
    const size_t v = blockIdx.x;
    bgv_dec_body<LOGN, NT>(cta, reinterpret_cast<u32 *>(smem_raw), work + v * L * N, slots + v * N, T, lt.lp, K, L);
}

#endif
// ------------------------------------------------------------------ fused key-switch family
// TMA-unit bulk prefetch of a contiguous region into L2 (SASS: UBLKPF.L2); bytes must be a multiple of 16
__device__ __forceinline__ void bulk_prefetch_l2(const void *p, u32 bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

#if DPFHE_PART_MAIN
// grid = G CTAs, G a multiple of the group size, all co-resident (cooperative launch).  A group processes one ciphertext at a
// time; its leader draws the next ciphertext index from a global ticket counter and posts it in the group's mailbox (dynamic
// balancing: groups that run ahead take more work); the members exchange their INTT'd digits through `scratch`
// (double-buffered by round parity, L2 resident) under release/acquire flags.
// FILTER (hoisted-rotation fallback): only the ciphertexts flagged in A.only are processed; the digit slots then
// alternate over the rounds that actually run.
//   N <= 8192 (ks_fused_blk): one 4096-point block per CTA, accumulators in shared memory; a group is L pairs (N = 8192, each
//             pair a cluster of two CTAs) or L CTAs (N = 4096); pair `slot` owns limb i = slot % L and digit slot `slot`.
//   N = 16384 (else branch of ks_fused_kernel): one limb per CTA in two halves, accumulators in L2-resident scratch rows; a group is L CTAs.

// Tickets are drawn in order, so ciphertext ct + pf_dist will be started by some group a few microseconds from now: thread 0
// pulls this CTA's share of its inputs (`bytes` at offset `off` of every input polynomial of ciphertext nc = ct + pf_dist) from HBM
// into L2 with the TMA unit's bulk prefetch, so the tensor phase that consumes them is L2- rather than HBM-latency bound.  The
// callers test that condition themselves, so that only thread 0 evaluates the offset.
template <int LOGN, int MODE>
__device__ __forceinline__ void prefetch_inputs(const KsArgs &A, size_t nc, size_t off, u32 bytes) {
    constexpr size_t N = (size_t)1 << LOGN;
    const size_t P = (size_t)A.L * N;
    if (MODE == KS_PLAIN) {
        bulk_prefetch_l2(A.a + nc * P + off, bytes);
    } else {
        bulk_prefetch_l2(A.a + nc * 2 * P + off, bytes);
        bulk_prefetch_l2(A.a + nc * 2 * P + P + off, bytes);
        if (MODE == KS_MUL_RELIN) {
            bulk_prefetch_l2(A.b + nc * 2 * P + off, bytes);
            bulk_prefetch_l2(A.b + nc * 2 * P + P + off, bytes);
        }
    }
}

template <int LOGN, int NT, int MODE, bool PROF, bool FILTER>
__device__ __forceinline__ void ks_fused_blk(const KsArgs &A, const LimbTable &lt, size_t batch, u32 *flags, u32 epoch, u32 *ticket, u64 *mail,
                                             unsigned long long *prof, u32 pf_dist) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    constexpr u32 PAIR = (u32)ks_blk_pair<LOGN>();
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    U64x2 *acc = reinterpret_cast<U64x2 *>(smem_raw + ((size_t)8 << KS_BLK_LOGN));
    DevCta<NT, PROF> cta;
    cta.prof_begin(prof);
    namespace cg = cooperative_groups;
    const u32 L = A.L, h = blockIdx.x % PAIR, slot = blockIdx.x / PAIR, i = slot % L, group = slot / L;
    const u64 *peer = buf;
    if constexpr (PAIR == 2) peer = cg::this_cluster().map_shared_rank(buf, (int)h ^ 1);
    auto pair_sync = [&]() {
        if constexpr (PAIR == 2) cg::this_cluster().sync();
        else __syncthreads();
    };
    const LimbParams &p = lt.lp[i];
    u32 executed = 0;
    for (u32 round = 0;; ++round) {
        if (FILTER) __syncthreads();
        // FILTER: static assignment computed by every thread (see the N = 16384 branch below).  The round tag epoch + round + 1 is
        // written out at each use in both fused loops: held in a register through the round, it spills at N = 16384.
        const size_t ct = FILTER ? (size_t)round * (gridDim.x / (L * PAIR)) + group
                                 : (size_t)draw_ticket(ticket, [&] { return mail + group; }, epoch + round + 1, i == 0 && h == 0,
                                                       L * PAIR > 1);
        if (ct >= batch) break;   // every member of the group reads the same ticket, so they leave together
        if (FILTER && A.only[ct] == 0u) continue;
        if (pf_dist && threadIdx.x == 0 && ct + pf_dist < batch)
            prefetch_inputs<LOGN, MODE>(A, ct + pf_dist, (size_t)i * N + ((size_t)h << KS_BLK_LOGN), 8u << KS_BLK_LOGN);
        const u32 parity = (FILTER ? executed++ : round) & 1u;
        ks_blk_phase1_local<LOGN, NT, MODE>(cta, buf, acc, A, p, ct, i, (int)h);
        // the partner's block has been through the inverse passes, and the partner has read this round's mailbox (with L = 1 this
        // barrier is what keeps a leader from posting the next ticket before its partner has read the current one)
        pair_sync();
        if (L > 1) {
            ks_blk_phase1_outer<LOGN, NT>(cta, buf, peer, A, p, i, (int)h, A.scratch + ((size_t)slot * 2 + parity) * N);
            __threadfence();
            pair_sync();   // both halves of t_i are stored, and the partner has finished reading this CTA's buffer
            if (h == 0 && threadIdx.x == 0) st_release_u32(flags + slot, epoch + round + 1);
            for (u32 jj = 1; jj < L; ++jj) {
                const u32 j = (i + jj) % L, sib = slot - i + j;
                wait_flags(flags + sib, 1, epoch + round + 1);
                cta.mark(3);   // waiting for the sibling's digit
                ks_blk_phase2<LOGN, NT>(cta, buf, acc, A, p, ct, i, j, jj, (int)h, A.scratch + ((size_t)sib * 2 + parity) * N);
            }
        }
    }
    cta.prof_end();
}

template <int LOGN, int NT, int MINB, int MODE, bool PROF, bool FILTER = false>
__global__ void __launch_bounds__(NT, MINB) ks_fused_kernel(KsArgs A, const __grid_constant__ LimbTable lt, size_t batch, u32 *flags, u32 epoch,
                                                            u32 *ticket, u64 *mail, unsigned long long *prof, u32 pf_dist, u32 *consumed) {
    if constexpr (LOGN <= 13) {
        ks_fused_blk<LOGN, NT, MODE, PROF, FILTER>(A, lt, batch, flags, epoch, ticket, mail, prof, pf_dist);
    } else {
        // the L CTAs of slots [g*L, (g+1)*L) form group g: CTA `slot` owns output limb i = slot % L; the leader is i == 0
        extern __shared__ __align__(1024) unsigned char smem_raw[];
        constexpr size_t N = (size_t)1 << LOGN;
        u64 *buf = reinterpret_cast<u64 *>(smem_raw);
        DevCta<NT, PROF> cta;
        cta.prof_begin(prof);
        const u32 L = A.L, slot = blockIdx.x, i = slot % L, group = slot / L;
        const LimbParams &p = lt.lp[i];
        u32 executed = 0;
        // Single-buffered digit slots (consumed != nullptr): slot s holds ONE digit; its owner may overwrite it only after the L-1
        // siblings that read the previous digit have signalled.  The counters are monotone across launches: the value found at
        // kernel start is the base (no reader of an earlier launch is still running).  One slot per CTA instead of two keeps
        // half of the digit slots out of the kernel's cross-phase working set in the L2.
        __shared__ u32 s_base;
        if (consumed && threadIdx.x == 0) s_base = ld_acquire_u32(consumed + slot);
        __syncthreads();
        const u32 consumed_base = consumed ? s_base : 0u;
        u32 published = 0;   // digits this CTA has published in this launch
        for (u32 round = 0;; ++round) {
            if (FILTER) __syncthreads();
            // FILTER: static assignment computed by every thread.  Skipped rounds involve no exchange between the members of
            // a group, so a leader handing out tickets could run ahead and overwrite a mailbox tag (or the posted ticket in
            // shared memory) before it was read.
            const size_t ct = FILTER ? (size_t)round * (gridDim.x / L) + group
                                     : (size_t)draw_ticket(ticket, [&] { return mail + group; }, epoch + round + 1, i == 0, L > 1);
            if (ct >= batch) break;   // every member of the group reads the same ticket, so they leave together
            if (FILTER && A.only[ct] == 0u) continue;
            if (pf_dist && threadIdx.x == 0 && ct + pf_dist < batch) prefetch_inputs<LOGN, MODE>(A, ct + pf_dist, (size_t)i * N, (u32)(N * 8));
            const u32 parity = consumed ? 0u : (FILTER ? executed++ : round) & 1u;
            const size_t slot_stride = consumed ? 1 : 2;      // digit slots per CTA
            u64 *acc_rows = A.acc + (size_t)slot * 2 * N;   // this CTA's two lazy accumulator rows (L2 resident, reused every round)
            ks_phase1<LOGN, NT, MODE>(cta, buf, A, p, ct, i, A.scratch + ((size_t)slot * slot_stride + parity) * N, acc_rows, 0, 0,
                                      consumed && L > 1 ? consumed + slot : nullptr, consumed_base + published * (L - 1));
            ++published;
            if (L > 1) {
                publish_flag(flags + slot, epoch + round + 1);
                for (u32 jj = 1; jj < L; ++jj) {
                    const u32 j = (i + jj) % L, sib = slot - i + j;
                    wait_flags(flags + sib, 1, epoch + round + 1);
                    cta.mark(3);   // waiting for the sibling's digit
                    ks_phase2_digit<LOGN, NT>(cta, buf, A, p, ct, i, j, jj, A.scratch + ((size_t)sib * slot_stride + parity) * N, acc_rows);
                    // every thread is past its last read of the sibling's digit (the body ends with a CTA barrier): hand the slot back
                    if (consumed && threadIdx.x == 0) {
                        __threadfence();
                        atomicAdd(consumed + sib, 1u);
                    }
                }
            }
        }
        cta.prof_end();
    }
}

// Hoisted rotations, step 1 (DESIGN.md §4.4d): the same group / ticket / flag machinery as ks_fused_kernel, but the digits
// are the unpermuted c1 limbs and phase 2 stores the lifted transforms U[ct][j][i] instead of multiplying them with a key.
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ks_hoist_kernel(HoistArgs A, const __grid_constant__ LimbTable lt, size_t batch, u32 *flags, u32 epoch,
                                                            u32 *ticket, u64 *mail) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    DevCta<NT> cta;
    const u32 L = A.L, slot = blockIdx.x, i = slot % L, group = slot / L;
    const LimbParams &p = lt.lp[i];
    for (u32 round = 0;; ++round) {
        const u32 tag = epoch + round + 1;
        const size_t ct = draw_ticket(ticket, [&] { return mail + group; }, tag, i == 0, true);
        if (ct >= batch) break;
        const u32 parity = round & 1u;
        hoist_phase1<LOGN, NT>(cta, buf, A, p, ct, i, A.scratch + ((size_t)slot * 2 + parity) * N);
        publish_flag(flags + slot, tag);
        for (u32 jj = 1; jj < L; ++jj) {
            const u32 j = (i + jj) % L, sib = slot - i + j;
            wait_flags(flags + sib, 1, tag);
            hoist_phase2<LOGN, NT>(cta, buf, A, p, ct, i, j, A.scratch + ((size_t)sib * 2 + parity) * N);
        }
    }
}

// step 2: one rotation applied to blocks of ROT_CB ciphertexts x one limb; no transforms, only gathers and multiply-accumulates
template <int LOGN, int NT, int MINB, int ROT_CB, bool PF>
__global__ void __launch_bounds__(NT, MINB) rot_apply_kernel(RotApplyArgs A, const __grid_constant__ LimbTable lt, size_t batch, u32 nseg) {
    DevCta<NT> cta;
    constexpr int NC = 1 << (LOGN - 1);
    const size_t n_blocks = (batch + ROT_CB - 1) / ROT_CB, n_items = n_blocks * A.L * nseg;
    const int seg_chunks = NC / (int)nseg;   // nseg is a power of two <= NC / NT
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const u32 seg = (u32)(w % nseg), i = (u32)((w / nseg) % A.L);
        const size_t ct0 = (w / nseg / A.L) * ROT_CB;
        const u32 n_ct = (u32)(batch - ct0 < (size_t)ROT_CB ? batch - ct0 : (size_t)ROT_CB);
        rot_apply_rows<LOGN, NT, ROT_CB, PF>(cta, A, lt.lp[i], ct0, n_ct, i, (int)seg * seg_chunks, ((int)seg + 1) * seg_chunks);
    }
}

// coefficient-form indicator of the positions that sigma_g negates: X^k -> X^(kg mod 2N), negative when kg mod 2N >= N
template <int LOGN>
__global__ void __launch_bounds__(256) negmask_kernel(u64 *mask, u32 g, u32 L) {
    constexpr u32 N = 1u << LOGN;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < N; k += gridDim.x * blockDim.x) {
        const u32 e = (k * g) & (2 * N - 1);
        const u64 v = e >= N ? 1ull : 0ull;
        for (u32 l = 0; l < L; ++l) mask[(size_t)l * N + (e & (N - 1))] = v;
    }
}

// kprime[c][i][n] = M[i][n] * sum_{j != i} (q_j mod q_i) * key[j][c][i][n]  mod q_i, canonical
template <int LOGN>
__global__ void __launch_bounds__(256) kprime_kernel(const u64 *__restrict__ key, const u64 *__restrict__ M, const u64 *__restrict__ delta,
                                                     u64 *__restrict__ out, const LimbParams *__restrict__ lps, u32 L) {
    constexpr size_t N = (size_t)1 << LOGN;
    const size_t P = (size_t)L * N, total = 2 * P;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const u32 c = (u32)(e / P), i = (u32)((e % P) / N);
        const size_t n = e % N;
        const LimbParams p = lps[i];
        u64 s = 0;
        for (u32 j = 0; j < L; ++j) {
            if (j == i) continue;
            s = csub(s + mulmod(key[((size_t)j * 2 + c) * P + (size_t)i * N + n], delta[j * L + i], p), p.q);
        }
        out[e] = mulmod(s, M[(size_t)i * N + n], p);
    }
}

#endif
#if DPFHE_PART_HYBRID
// Hybrid (special-prime) variant, DESIGN.md §2.10.  A group is L + 1 CTAs: CTA i < L owns ciphertext limb i,
// CTA L owns the special limb.  Per ciphertext:
//   limb CTA    tensor/permute, p*own terms + first key term, INTT, publish digit        (as above)
//               L-1 x [lift + NTT + MAC]                                                  (as above, nothing final)
//               2 x [centred lift of tau' + NTT], out = (acc - s*u) / p                   (ms_limb_body)
//   special CTA L x [lift + NTT_p + MAC into its scratch rows]; 2 x INTT_p (* t^-1) -> tau', publish
// Both roles run six transforms per ciphertext at L = 4.  The special CTA can only finish after every digit arrived,
// so a limb CTA postpones the division step of ciphertext r until it has done the digit and multiply-accumulate
// work of ciphertext r + 1 (software pipeline of depth one): tau' rows, like the digits and the mailbox, are
// double-buffered by round parity, and the output rows keep the lazy accumulators in between (DESIGN.md §4.6).
// LV (DESIGN.md §4.17): a level view reading the top-level key through ks_key_row, its stride A.Lk the top-level L; the body is
// shared by the two kernels below.
template <int LOGN, int NT, int MODE, bool LV>
__device__ __forceinline__ void ks_hybrid_body(const KsArgs &A, const LimbTable &lt, const MsConsts &K, size_t batch, u32 *flags, u32 epoch,
                                               u32 *ticket, u64 *mail) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    DevCta<NT> cta;
    const u32 L = A.L, GS = L + 1, slot = blockIdx.x, i = slot % GS, group = slot / GS, base = slot - i;
    const u32 key_shift = LV ? A.Lk - GS : 0u;   // Lq - l
    const bool special = i == L;
    const LimbParams &p = lt.lp[i];
    u64 *hyb = A.hyb + (size_t)group * KS_HYB_ROWS * N;
    // the postponed division of one ciphertext (limb CTAs): needs tau' of that round
    auto acc_of = [&](u32 parity) { return A.acc + ((size_t)slot * 2 + parity) * 2 * N; };   // accumulator rows, double-buffered by round parity
    auto divide = [&](size_t ct, u32 tag, u32 parity) {
        wait_flags(flags + (base + L), 1, tag);
        const size_t P = (size_t)L * N;
        for (u32 c = 0; c < 2; ++c) {
            u64 *row = A.out + ct * 2 * P + c * P + (size_t)i * N;   // lazy accumulator -> final value in the output row
            ms_limb_body<LOGN, NT, true>(cta, buf, hyb + ks_hyb_tau_row(parity, c) * N, acc_of(parity) + c * N, row, A.tw + (size_t)i * N, p, K, i);
        }
    };
    bool pending = false;
    size_t prev_ct = 0;
    u32 prev_tag = 0, prev_parity = 0;
    for (u32 round = 0;; ++round) {
        const u32 tag = epoch + round + 1, parity = round & 1u;
        const size_t ct = draw_ticket(ticket, [&] { return mail + (size_t)group * 2 + parity; }, tag, i == 0, true);
        if (ct >= batch) break;
        if (!special) {
            if constexpr (LV)
                ks_phase1<LOGN, NT, MODE, true, true>(cta, buf, A, p, ct, i, A.scratch + ((size_t)slot * 2 + parity) * N, acc_of(parity), K.qlm[i],
                                                      K.qlm_s[i], nullptr, 0, ~0u, nullptr, key_shift);
            else
                ks_phase1<LOGN, NT, MODE, true>(cta, buf, A, p, ct, i, A.scratch + ((size_t)slot * 2 + parity) * N, acc_of(parity), K.qlm[i], K.qlm_s[i]);
            publish_flag(flags + slot, tag);
            for (u32 jj = 1; jj < L; ++jj) {
                const u32 j = (i + jj) % L;
                wait_flags(flags + (base + j), 1, tag);
                ks_phase2_digit<LOGN, NT, true, false, LV>(cta, buf, A, p, ct, i, j, jj, A.scratch + ((size_t)(base + j) * 2 + parity) * N, acc_of(parity),
                                                           key_shift);
            }
            if (pending) divide(prev_ct, prev_tag, prev_parity);
            pending = true;
            prev_ct = ct;
            prev_tag = tag;
            prev_parity = parity;
        } else {
            for (u32 jj = 0; jj < L; ++jj) {
                const u32 j = (group + jj) % L;   // groups start at different digits: spreads the key-column reads
                wait_flags(flags + (base + j), 1, tag);
                ks_phase2_digit<LOGN, NT, true, true, LV>(cta, buf, A, p, ct, i, j, jj, A.scratch + ((size_t)(base + j) * 2 + parity) * N, hyb, key_shift);
            }
            for (u32 c = 0; c < 2; ++c)
                ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)i * N, p, hyb + ks_hyb_tau_row(parity, c) * N, K);
            publish_flag(flags + slot, tag);
        }
    }
    if (pending) divide(prev_ct, prev_tag, prev_parity);   // the group's last ciphertext
}

template <int LOGN, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) ks_hybrid_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                             size_t batch, u32 *flags, u32 epoch, u32 *ticket, u64 *mail) {
    ks_hybrid_body<LOGN, NT, MODE, false>(A, lt, K, batch, flags, epoch, ticket, mail);
}

// one special prime at level l (DESIGN.md §2.20, §4.17): ks_hybrid_kernel's program on the level's view, reading the top-level key
template <int LOGN, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) ks_hybrid_level_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                   size_t batch, u32 *flags, u32 epoch, u32 *ticket, u64 *mail) {
    ks_hybrid_body<LOGN, NT, MODE, true>(A, lt, K, batch, flags, epoch, ticket, mail);
}

#endif
#if DPFHE_PART_GROUPED
// Grouped hybrid variant (dnum < L), DESIGN.md §2.11.  A group is Lq + K CTAs: CTA i < Lq owns ciphertext limb i, CTA Lq + k
// special prime k.  The roles are those of ks_hybrid_kernel with digits of K limbs:
//   limb CTA    tensor/permute, P*own terms + the key term of its own digit, INTT (scaled by Qhat^-1), publish
//               (dnum-1) x [basis conversion of a foreign digit + NTT + MAC]
//               2 x [basis conversion of the K tau' rows + NTT], out = (acc - s*u) / P     (one round late, as above)
//   special CTA dnum x [basis conversion + NTT + MAC into its scratch rows]; 2 x INTT (* (t Phat)^-1) -> tau', publish
// With Lq = 4, K = 2 every CTA runs four transforms per ciphertext (24 in all, against 30 for one special prime).
// ADD (KS_ROTATE only): the division step adds addend [batch][2][Lq][N] (canonical) to the result before its one store, so that a
// Horner step of a linear layer, out = rot(acc) + inner_g, is one launch (DESIGN.md §4.4b′).  out must not alias a or addend.
// KS_DOT (DESIGN.md §2.18, §4.15): the limb CTAs build their digit from the summed tensor products of dot's pairs; everything after
// phase 1 is the same program.  The body is shared by the kernels below, which differ in their parameter block only.
// RS (multiply-and-rescale, DESIGN.md §2.19, §4.16; modes KS_MUL_RELIN and KS_DOT): the division is by P' = P * qbar, qbar = q_{Lq-1}.
// The dropped limb's CTA runs phases 1 and 2 as before, then turns its accumulator rows into y_qbar as a special CTA does (inverse
// transform, (t P)^-1 folded into N^-1) and publishes them on its group's flag in R; it divides nothing and stores no output.  The
// other limb CTAs divide one round late over K + 1 rows and write [batch][2][Lq-1][N].
// LV (DESIGN.md §4.17): a level view reading the top-level key through ks_key_row, its stride A.Lk the top-level L.
template <int LOGN, int NT, int MODE, bool ADD, bool RS = false, bool LV = false>
__device__ __forceinline__ void ks_grouped_body(const KsArgs &A, const LimbTable &lt, const MsConsts &K, const GroupConsts &G, size_t batch, u32 *flags,
                                                u32 epoch, u32 *ticket, u64 *mail, const u64 *addend, const DotArgs *dot,
                                                const RescaleConsts *R = nullptr) {
    static_assert(!ADD || MODE == KS_ROTATE, "the fused addition is a Horner step of rotations");
    static_assert(!RS || (!ADD && (MODE == KS_MUL_RELIN || MODE == KS_DOT)), "multiply-and-rescale follows a product");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    DevCta<NT> cta;
    const u32 Lq = G.Lq, Ks = G.K, dnum = G.dnum, GS = Lq + Ks, slot = blockIdx.x, i = slot % GS, group = slot / GS, base = slot - i;
    const u32 key_shift = LV ? A.Lk - GS : 0u;   // Lq - l of the top level
    const bool special = i >= Lq;
    const LimbParams &p = lt.lp[i];
    // rows of special prime k of this group: accumulators (0, 1) and tau' (double-buffered by round parity)
    auto hyb_of = [&](u32 k) { return A.hyb + ((size_t)group * Ks + k) * KS_HYB_ROWS * N; };
    auto acc_of = [&](u32 parity) { return A.acc + ((size_t)slot * 2 + parity) * 2 * N; };
    // y_qbar row c of round parity `parity` (RS)
    auto drop_of = [&](u32 parity, u32 c) { return R->tau + (((size_t)group * 2 + parity) * 2 + c) * N; };
    auto divide = [&](size_t ct, u32 tag, u32 parity) {
        if constexpr (RS) if (threadIdx.x == 0) spin_until(R->tau_flag + group, tag);   // the barrier of the next wait covers it
        wait_flags(flags + (base + Lq), Ks, tag);
        if constexpr (RS) {
            const size_t P = (size_t)(Lq - 1) * N;
            for (u32 c = 0; c < 2; ++c)
                ms_limb_group<LOGN, NT, true, false, true>(cta, buf, hyb_of(0) + ks_hyb_tau_row(parity, c) * N, (size_t)KS_HYB_ROWS * N, acc_of(parity) + c * N,
                                                           A.out + ct * 2 * P + c * P + (size_t)i * N, A.tw + (size_t)i * N, p, K, G, i, nullptr,
                                                           drop_of(parity, c), R);
            return;
        }
        const size_t P = (size_t)Lq * N;
        for (u32 c = 0; c < 2; ++c) {
            u64 *row = A.out + ct * 2 * P + c * P + (size_t)i * N;
            const u64 *add_row = nullptr;
            if constexpr (ADD) add_row = addend + ct * 2 * P + c * P + (size_t)i * N;
            ms_limb_group<LOGN, NT, true, ADD>(cta, buf, hyb_of(0) + ks_hyb_tau_row(parity, c) * N, (size_t)KS_HYB_ROWS * N, acc_of(parity) + c * N, row,
                                               A.tw + (size_t)i * N, p, K, G, i, add_row);
        }
    };
    bool pending = false;
    size_t prev_ct = 0;
    u32 prev_tag = 0, prev_parity = 0;
    for (u32 round = 0;; ++round) {
        const u32 tag = epoch + round + 1, parity = round & 1u;
        const size_t ct = draw_ticket(ticket, [&] { return mail + (size_t)group * 2 + parity; }, tag, i == 0, true);
        if (ct >= batch) break;
        const u64 *t_rows = A.scratch + ((size_t)base * 2 + parity) * N;   // row of limb j: + j * 2N
        if (!special) {
            const u32 g_own = i / Ks;
            ks_phase1<LOGN, NT, MODE, true, LV>(cta, buf, A, G.lp_up[i], ct, i, A.scratch + ((size_t)slot * 2 + parity) * N, acc_of(parity), K.qlm[i],
                                                K.qlm_s[i], nullptr, 0, g_own, dot, key_shift);
            publish_flag(flags + slot, tag);
            for (u32 jj = 1; jj < dnum; ++jj) {
                const u32 g = (g_own + jj) % dnum, lo = g * Ks, cnt = lo + Ks < Lq ? Ks : Lq - lo;
                wait_flags(flags + (base + lo), cnt, tag);
                ks_phase2_group<LOGN, NT, false, LV>(cta, buf, A, G, p, ct, i, g, jj, t_rows, 2 * N, acc_of(parity), key_shift);
            }
            if constexpr (RS) if (i == Lq - 1) {
                // the dropped limb.  Its y_qbar rows of this parity were last read by the divide() of round - 2, which every other
                // limb CTA runs before its digit of this round: the foreign digits were awaited above, the digit mates (limbs lo ..
                // Lq-2 of its own digit, never awaited by phase 2) are awaited here.  Its digit slot is protected by the mailbox:
                // limb 0 posts this round only after its divide(round - 2), which waited for every special CTA of round - 2.
                const u32 lo = g_own * Ks;
                wait_flags(flags + (base + lo), i - lo, tag);
                for (u32 c = 0; c < 2; ++c)
                    ms_tau_body<LOGN, NT, true>(cta, buf, acc_of(parity) + c * N, acc_of(parity) + c * N, A.itw + (size_t)i * N, R->lp_drop,
                                                drop_of(parity, c), K);
                publish_flag(R->tau_flag + group, tag);
                continue;
            }
            if (pending) divide(prev_ct, prev_tag, prev_parity);
            pending = true;
            prev_ct = ct;
            prev_tag = tag;
            prev_parity = parity;
        } else {
            u64 *hyb = hyb_of(i - Lq);
            for (u32 jj = 0; jj < dnum; ++jj) {
                const u32 g = (group + jj) % dnum, lo = g * Ks, cnt = lo + Ks < Lq ? Ks : Lq - lo;
                wait_flags(flags + (base + lo), cnt, tag);
                ks_phase2_group<LOGN, NT, true, LV>(cta, buf, A, G, p, ct, i, g, jj, t_rows, 2 * N, hyb, key_shift);
            }
            for (u32 c = 0; c < 2; ++c)
                ms_tau_body<LOGN, NT, true>(cta, buf, hyb + c * N, hyb + c * N, A.itw + (size_t)i * N, G.lp_up[i], hyb + ks_hyb_tau_row(parity, c) * N, K);
            publish_flag(flags + slot, tag);
        }
    }
    if (pending) divide(prev_ct, prev_tag, prev_parity);   // the group's last ciphertext
}

template <int LOGN, int NT, int MINB, int MODE, bool ADD = false>
__global__ void __launch_bounds__(NT, MINB) ks_grouped_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                              const __grid_constant__ GroupConsts G, size_t batch, u32 *flags, u32 epoch,
                                                              u32 *ticket, u64 *mail, const u64 *addend) {
    ks_grouped_body<LOGN, NT, MODE, ADD>(A, lt, K, G, batch, flags, epoch, ticket, mail, addend, nullptr);
}

// multiply-and-rescale (DESIGN.md §2.19): the program in mode MODE (KS_MUL_RELIN or KS_DOT, D unused by the former) with the division
// by P * q_{Lq-1}; R carries the dropped limb's constants and rows
template <int LOGN, int NT, int MINB, int MODE>
__global__ void __launch_bounds__(NT, MINB) ks_rescale_grouped_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                      const __grid_constant__ GroupConsts G, const __grid_constant__ DotArgs D,
                                                                      const __grid_constant__ RescaleConsts R, size_t batch, u32 *flags, u32 epoch,
                                                                      u32 *ticket, u64 *mail) {
    ks_grouped_body<LOGN, NT, MODE, false, true>(A, lt, K, G, batch, flags, epoch, ticket, mail, nullptr, MODE == KS_DOT ? &D : nullptr, &R);
}

// every grouped call at level l (DESIGN.md §2.20, §4.17): the program in mode MODE (KS_MUL_RELIN, KS_ROTATE, KS_DOT) with the division
// by P (RS = false) or by P * q_{l-1} (RS = true, ks_rescale_grouped_kernel's), on the level's view, reading the top-level key.  One
// parameter block, that of ks_rescale_grouped_kernel, for all of them; D and R are unused where the mode has none.
template <int LOGN, int NT, int MINB, int MODE, bool RS>
__global__ void __launch_bounds__(NT, MINB) ks_level_grouped_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                    const __grid_constant__ GroupConsts G, const __grid_constant__ DotArgs D,
                                                                    const __grid_constant__ RescaleConsts R, size_t batch, u32 *flags, u32 epoch,
                                                                    u32 *ticket, u64 *mail) {
    ks_grouped_body<LOGN, NT, MODE, false, RS, true>(A, lt, K, G, batch, flags, epoch, ticket, mail, nullptr, MODE == KS_DOT ? &D : nullptr,
                                                     RS ? &R : nullptr);
}

// the fused Horner step of a linear layer at level l (DESIGN.md §2.21, §4.18): ks_grouped_kernel's rotation with the addend
// [batch][2][l][N] (ADD), on the level's view, reading the top-level key.  ks_level_grouped_kernel's parameter block plus the addend.
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ks_level_horner_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                   const __grid_constant__ GroupConsts G, const __grid_constant__ DotArgs D,
                                                                   const __grid_constant__ RescaleConsts R, size_t batch, u32 *flags, u32 epoch,
                                                                   u32 *ticket, u64 *mail, const u64 *addend) {
    ks_grouped_body<LOGN, NT, KS_ROTATE, true, false, true>(A, lt, K, G, batch, flags, epoch, ticket, mail, addend, nullptr, nullptr);
}

// the encrypted inner product: ks_grouped_kernel's program in mode KS_DOT, with the operand tables of the call in D
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ct_dot_grouped_kernel(KsArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                  const __grid_constant__ GroupConsts G, const __grid_constant__ DotArgs D,
                                                                  size_t batch, u32 *flags, u32 epoch, u32 *ticket, u64 *mail) {
    ks_grouped_body<LOGN, NT, KS_DOT, false>(A, lt, K, G, batch, flags, epoch, ticket, mail, nullptr, &D);
}

// Hoisted rotations with grouped hybrid keys, step 1 (DESIGN.md §2.11b): groups of L CTAs (every limb of the context) build
// U[ct][g][i]; ticket / mailbox / flag machinery as in ks_hoist_kernel, the digits converted as in ks_grouped_kernel.
// A limb CTA waits only for the digits of foreign groups and a special CTA publishes no digit, so the rounds of a group are
// not held together by the digit flags alone: every CTA also publishes done[slot] = tag at the end of a round, and enters round
// r only when the whole group has finished round r - 2 — the round whose digit slots and mailbox (both double-buffered by
// round parity) round r overwrites.
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) ks_hoistg_kernel(HoistGArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ GroupConsts G,
                                                             size_t batch, u32 *flags, u32 *done, u32 epoch, u32 *ticket, u64 *mail) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr size_t N = (size_t)1 << LOGN;
    u64 *buf = reinterpret_cast<u64 *>(smem_raw);
    DevCta<NT> cta;
    const u32 Lq = G.Lq, Ks = G.K, dnum = G.dnum, GS = Lq + Ks, slot = blockIdx.x, i = slot % GS, group = slot / GS, base = slot - i;
    const LimbParams &p = lt.lp[i];
    for (u32 round = 0;; ++round) {
        const u32 tag = epoch + round + 1, parity = round & 1u;
        if (round >= 2) wait_flags(done + base, GS, tag - 2);
        const size_t ct = draw_ticket(ticket, [&] { return mail + (size_t)group * 2 + parity; }, tag, i == 0, true);
        if (ct >= batch) break;
        const u64 *t_rows = A.scratch + ((size_t)base * 2 + parity) * N;
        u32 g_own = dnum;   // a special limb belongs to no digit
        if (i < Lq) {
            g_own = i / Ks;
            hoistg_phase1<LOGN, NT>(cta, buf, A, G, ct, i, A.scratch + ((size_t)slot * 2 + parity) * N);
            publish_flag(flags + slot, tag);
        }
        for (u32 jj = 0; jj < dnum; ++jj) {
            const u32 g = (group + i + jj) % dnum;
            if (g == g_own) continue;
            const u32 lo = g * Ks, cnt = lo + Ks < Lq ? Ks : Lq - lo;
            wait_flags(flags + (base + lo), cnt, tag);
            hoistg_phase2<LOGN, NT>(cta, buf, A, G, p, ct, i, g, t_rows, 2 * N);
        }
        __syncthreads();   // every thread is past its last read of the group's digit slots
        if (threadIdx.x == 0) st_release_u32(done + slot, tag);
    }
}

// step 2: one rotation applied to blocks of ROT_CB ciphertexts x one limb of the context (gathers + multiply-accumulates)
template <int LOGN, int NT, int MINB, int ROT_CB>
__global__ void __launch_bounds__(NT, MINB) rot_apply_grouped_kernel(RotApplyGArgs A, const __grid_constant__ LimbTable lt, const __grid_constant__ MsConsts K,
                                                                     const __grid_constant__ GroupConsts G, size_t batch, u32 nseg) {
    DevCta<NT> cta;
    constexpr int NC = 1 << (LOGN - 1);
    const u32 L = G.Lq + G.K;
    const size_t n_blocks = (batch + ROT_CB - 1) / ROT_CB, n_items = n_blocks * L * nseg;
    const int seg_chunks = NC / (int)nseg;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const u32 seg = (u32)(w % nseg), i = (u32)((w / nseg) % L);
        const size_t ct0 = (w / nseg / L) * ROT_CB;
        const u32 n_ct = (u32)(batch - ct0 < (size_t)ROT_CB ? batch - ct0 : (size_t)ROT_CB);
        rot_apply_grouped_rows<LOGN, NT, ROT_CB>(cta, A, G, K, lt.lp[i], ct0, n_ct, i, (int)seg * seg_chunks, ((int)seg + 1) * seg_chunks);
    }
}

// the same at level l (DESIGN.md §2.21, §4.18): the key is a top-level key, key_shift = Lq - l rows longer per (digit, component)
template <int LOGN, int NT, int MINB, int ROT_CB>
__global__ void __launch_bounds__(NT, MINB) rot_apply_grouped_level_kernel(RotApplyGArgs A, const __grid_constant__ LimbTable lt,
                                                                           const __grid_constant__ MsConsts K, const __grid_constant__ GroupConsts G,
                                                                           size_t batch, u32 nseg, u32 key_shift) {
    DevCta<NT> cta;
    constexpr int NC = 1 << (LOGN - 1);
    const u32 L = G.Lq + G.K;
    const size_t n_blocks = (batch + ROT_CB - 1) / ROT_CB, n_items = n_blocks * L * nseg;
    const int seg_chunks = NC / (int)nseg;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const u32 seg = (u32)(w % nseg), i = (u32)((w / nseg) % L);
        const size_t ct0 = (w / nseg / L) * ROT_CB;
        const u32 n_ct = (u32)(batch - ct0 < (size_t)ROT_CB ? batch - ct0 : (size_t)ROT_CB);
        rot_apply_grouped_rows<LOGN, NT, ROT_CB, true>(cta, A, G, K, lt.lp[i], ct0, n_ct, i, (int)seg * seg_chunks, ((int)seg + 1) * seg_chunks,
                                                       key_shift);
    }
}

// summed rotations (DESIGN.md §2.17): the accumulators of every rotation of a stage, summed, for blocks of ROT_CB ciphertexts x one
// limb x one segment of the row; the work split of rot_apply_grouped_kernel
template <int LOGN, int NT, int MINB, int ROT_CB>
__global__ void __launch_bounds__(NT, MINB) rot_sum_grouped_kernel(const __grid_constant__ RotSumGArgs A, const __grid_constant__ LimbTable lt,
                                                                   const __grid_constant__ MsConsts K, const __grid_constant__ GroupConsts G,
                                                                   size_t batch, u32 nseg) {
    DevCta<NT> cta;
    constexpr int NC = 1 << (LOGN - 1);
    const u32 L = G.Lq + G.K;
    const size_t n_blocks = (batch + ROT_CB - 1) / ROT_CB, n_items = n_blocks * L * nseg;
    const int seg_chunks = NC / (int)nseg;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const u32 seg = (u32)(w % nseg), i = (u32)((w / nseg) % L);
        const size_t ct0 = (w / nseg / L) * ROT_CB;
        const u32 n_ct = (u32)(batch - ct0 < (size_t)ROT_CB ? batch - ct0 : (size_t)ROT_CB);
        rot_sum_grouped_rows<LOGN, NT, ROT_CB>(cta, A, G, K, lt.lp[i], ct0, n_ct, i, (int)seg * seg_chunks, ((int)seg + 1) * seg_chunks);
    }
}

// the same at level l (DESIGN.md §2.20, §4.17): the keys are top-level keys, key_shift = Lq - l rows longer per (digit, component)
template <int LOGN, int NT, int MINB, int ROT_CB>
__global__ void __launch_bounds__(NT, MINB) rot_sum_grouped_level_kernel(const __grid_constant__ RotSumGArgs A, const __grid_constant__ LimbTable lt,
                                                                         const __grid_constant__ MsConsts K, const __grid_constant__ GroupConsts G,
                                                                         size_t batch, u32 nseg, u32 key_shift) {
    DevCta<NT> cta;
    constexpr int NC = 1 << (LOGN - 1);
    const u32 L = G.Lq + G.K;
    const size_t n_blocks = (batch + ROT_CB - 1) / ROT_CB, n_items = n_blocks * L * nseg;
    const int seg_chunks = NC / (int)nseg;
    for (size_t w = blockIdx.x; w < n_items; w += gridDim.x) {
        const u32 seg = (u32)(w % nseg), i = (u32)((w / nseg) % L);
        const size_t ct0 = (w / nseg / L) * ROT_CB;
        const u32 n_ct = (u32)(batch - ct0 < (size_t)ROT_CB ? batch - ct0 : (size_t)ROT_CB);
        rot_sum_grouped_rows<LOGN, NT, ROT_CB, true>(cta, A, G, K, lt.lp[i], ct0, n_ct, i, (int)seg * seg_chunks, ((int)seg + 1) * seg_chunks,
                                                     key_shift);
    }
}

#endif
#if DPFHE_PART_MAIN
// ------------------------------------------------------------------ plaintext inner products (BSGS inner loop)
template <int LOGN, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) pt_inner_kernel(PtInnerArgs A, const __grid_constant__ LimbTable lt, u32 g0, u32 gcnt) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    constexpr u32 TILES_PER_LIMB = (1u << LOGN) / PTI_COEFFS;
    DevCta<NT> cta;
    const u32 limb = blockIdx.x / TILES_PER_LIMB, tile = blockIdx.x % TILES_PER_LIMB;
    pt_inner_tile<LOGN, NT>(cta, reinterpret_cast<u64 *>(smem_raw), A, lt.lp[limb], limb, tile, g0, gcnt);
}

// ------------------------------------------------------------------ element-wise kernels
// all operate on 16-byte chunks; chunk index -> limb = (chunk / (N/2)) % L
template <int LOGN>
__global__ void __launch_bounds__(256) pointwise_mul_kernel(const U64x2 *__restrict__ a, const U64x2 *__restrict__ b,
                                                            U64x2 *__restrict__ out, const LimbParams *__restrict__ lps,
                                                            u32 L, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const LimbParams p = lps[(c / NC) % L];
        st_stream(out + c, mul_chunk(ld_stream(a + c), ld_stream(b + c), p));
    }
}

// out = a + b mod q (canonical operands); out may alias either input
template <int LOGN>
__global__ void __launch_bounds__(256) poly_add_kernel(const U64x2 *__restrict__ a, const U64x2 *__restrict__ b, U64x2 *__restrict__ out,
                                                       const LimbParams *__restrict__ lps, u32 L, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const u64 q = lps[(c / NC) % L].q;
        const U64x2 x = ld_stream(a + c), y = ld_stream(b + c);
        U64x2 r;
        r.x = csub(x.x + y.x, q);
        r.y = csub(x.y + y.y, q);
        st_stream(out + c, r);
    }
}

// ct [batch][2][L][N] x pt [L][N]
template <int LOGN>
__global__ void __launch_bounds__(256) ct_mul_plain_kernel(const U64x2 *__restrict__ ct, const U64x2 *__restrict__ pt,
                                                           U64x2 *__restrict__ out, const LimbParams *__restrict__ lps,
                                                           u32 L, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    const size_t pc = NC * L;   // chunks per polynomial
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const size_t in_poly = c % pc;
        const LimbParams p = lps[in_poly / NC];
        st_stream(out + c, mul_chunk(ld_stream(ct + c), ld_keep(pt + in_poly), p));
    }
}

// acc += ct o pt  (fused multiply-accumulate used by diagonal-method linear layers); acc may be lazy-free: all canonical
template <int LOGN>
__global__ void __launch_bounds__(256) ct_mul_plain_acc_kernel(const U64x2 *__restrict__ ct, const U64x2 *__restrict__ pt,
                                                               U64x2 *__restrict__ acc, const LimbParams *__restrict__ lps,
                                                               u32 L, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    const size_t pc = NC * L;
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const size_t in_poly = c % pc;
        const LimbParams p = lps[in_poly / NC];
        const U64x2 x = ld_stream(ct + c), m = ld_keep(pt + in_poly), a = ld_stream(acc + c);
        U64x2 r;
        r.x = csub(a.x + canon4(mulmod_lazy(x.x, m.x, p), p), p.q);
        r.y = csub(a.y + canon4(mulmod_lazy(x.y, m.y, p), p), p.q);
        st_stream(acc + c, r);
    }
}

// a,b [batch][2][L][N] -> d [batch][3][L][N]; one thread per chunk of one polynomial position
template <int LOGN>
__global__ void __launch_bounds__(256) ct_tensor_kernel(const U64x2 *__restrict__ a, const U64x2 *__restrict__ b,
                                                        U64x2 *__restrict__ d, const LimbParams *__restrict__ lps,
                                                        u32 L, size_t batch) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    const size_t pc = NC * L, total = batch * pc;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const size_t ct = t / pc, in_poly = t % pc;
        const LimbParams p = lps[in_poly / NC];
        const U64x2 a0 = ld_stream(a + ct * 2 * pc + in_poly), a1 = ld_stream(a + ct * 2 * pc + pc + in_poly);
        const U64x2 b0 = ld_stream(b + ct * 2 * pc + in_poly), b1 = ld_stream(b + ct * 2 * pc + pc + in_poly);
        U64x2 d0, d1, d2;
        tensor_coeff(a0.x, a1.x, b0.x, b1.x, p, d0.x, d1.x, d2.x);
        tensor_coeff(a0.y, a1.y, b0.y, b1.y, p, d0.y, d1.y, d2.y);
        d0.x = canon4(d0.x, p); d0.y = canon4(d0.y, p);
        d1.x = canon4(d1.x, p); d1.y = canon4(d1.y, p);
        d2.x = canon4(d2.x, p); d2.y = canon4(d2.y, p);
        st_stream(d + ct * 3 * pc + in_poly, d0);
        st_stream(d + ct * 3 * pc + pc + in_poly, d1);
        st_stream(d + ct * 3 * pc + 2 * pc + in_poly, d2);
    }
}

// synthetic residues (DESIGN.md §5): x[k] = mulhi64(splitmix64(seed + k), q_limb)
template <int LOGN>
__global__ void __launch_bounds__(256) fill_uniform_kernel(U64x2 *__restrict__ out, const LimbParams *__restrict__ lps, u32 L,
                                                           u64 seed, u64 first_elem, size_t n_chunks) {
    constexpr size_t NC = (size_t)1 << (LOGN - 1);
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (size_t)gridDim.x * blockDim.x) {
        const u64 q = lps[(c / NC) % L].q;
        U64x2 v;
        v.x = __umul64hi(splitmix64(seed + first_elem + 2 * c), q);
        v.y = __umul64hi(splitmix64(seed + first_elem + 2 * c + 1), q);
        st_stream(out + c, v);
    }
}

#endif
// Shoup companions of a switch key: ks[e] = floor(key[e] * 2^64 / q_limb(e)); layout [L][2][L][N]
template <int LOGN>
__global__ void __launch_bounds__(256) key_prepare_kernel(const u64 *__restrict__ key, u64 *__restrict__ key_s,
                                                          const LimbParams *__restrict__ lps, u32 L, size_t n) {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const u64 q = lps[(e >> LOGN) % L].q;
        key_s[e] = (u64)((((unsigned __int128)key[e]) << 64) / q);
    }
}

// ------------------------------------------------------------------ launchers
template <int LOGN>
struct Geometry {
    static constexpr int NT = LOGN == 12 ? 256 : 512;
    static constexpr size_t LIMB_BYTES = (size_t)8 << LOGN;
    static constexpr size_t KS_SMEM = (size_t)8 << (LOGN <= 13 ? LOGN : 13);   // persistent key-switch kernels: a limb, half a limb at N = 16384
};

#if DPFHE_PART_MAIN
template <int LOGN, int NT, int MINB, bool INV>
static cudaError_t launch_ntt_t(const LaunchCtx &lc, u64 *data, size_t n_limbs, cudaStream_t st) {
    auto kern = ntt_kernel<LOGN, NT, MINB, INV>;
    const size_t smem = Geometry<LOGN>::LIMB_BYTES;
    static ConfiguredMask configured;
    cudaError_t e = set_smem_once(configured, lc.device, smem, kern);
    if (e != cudaSuccess) return e;
    // one CTA per limb transform; the grid-stride loop only matters beyond 2^31-1 limbs
    const size_t grid = n_limbs < 0x7fffffffull ? n_limbs : 0x7fffffffull;
    kern<<<(unsigned)grid, NT, smem, st>>>(data, INV ? lc.itw : lc.tw, lc.lt, lc.L, n_limbs);
    return cudaGetLastError();
}

// tensor map of the caller's array seen as rows of 128 bytes; the encode function comes from the driver through the runtime
// (cudaGetDriverEntryPoint), so libdpfhe.so does not link libcuda
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static std::atomic<EncodeTiledFn> cached{nullptr};
    EncodeTiledFn f = cached.load();
    if (f) return f;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p)
        return nullptr;
    cached.store(reinterpret_cast<EncodeTiledFn>(p));
    return reinterpret_cast<EncodeTiledFn>(p);
}

// returns cudaErrorNotSupported when the TMA path does not apply (no driver entry point, too many rows for 32-bit coordinates):
// the caller then runs the ordinary kernel
template <int LOGN, int NT, int MINB>
static cudaError_t launch_ntt_inv_tma(const LaunchCtx &lc, u64 *data, size_t n_limbs, cudaStream_t st) {
    constexpr size_t ROWS = ((size_t)1 << LOGN) * 8 / 128;
    const size_t rows = n_limbs * ROWS;
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc || rows >= 0x7fffffffull || n_limbs >= 0x7fffffffull) return cudaErrorNotSupported;
    CUtensorMap tm;
    const cuuint64_t dims[2] = {16, (cuuint64_t)rows}, strides[1] = {128};
    const cuuint32_t box[2] = {16, (cuuint32_t)(ROWS < 256 ? ROWS : 256)}, estr[2] = {1, 1};
    if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, data, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return cudaErrorNotSupported;
    auto kern = ntt_inv_tma_kernel<LOGN, NT, MINB>;
    const size_t smem = Geometry<LOGN>::LIMB_BYTES;
    static ConfiguredMask configured;
    cudaError_t e = set_smem_once(configured, lc.device, smem, kern);
    if (e != cudaSuccess) return e;
    kern<<<(unsigned)n_limbs, NT, smem, st>>>(tm, data, lc.itw, lc.lt, lc.L);
    return cudaGetLastError();
}

template <int LOGN, int NT, int MINB>
static cudaError_t launch_ntt_dir(const LaunchCtx &lc, u64 *data, size_t n_limbs, bool inverse, cudaStream_t st) {
    if constexpr (LOGN <= 13 && NT == 256) {
        if (inverse && lc.ntt_tma) {
            cudaError_t e = launch_ntt_inv_tma<LOGN, NT, MINB>(lc, data, n_limbs, st);
            if (e != cudaErrorNotSupported) return e;
        }
    }
    return inverse ? launch_ntt_t<LOGN, NT, MINB, true>(lc, data, n_limbs, st) : launch_ntt_t<LOGN, NT, MINB, false>(lc, data, n_limbs, st);
}

template <bool INV>
static cudaError_t launch_ntt_pair_t(const LaunchCtx &lc, u64 *data, size_t n_limbs, cudaStream_t st) {
    constexpr int NT = 256, MINB = 3;
    auto kern = ntt_pair_kernel<NT, MINB, INV>;
    const size_t smem = Geometry<13>::LIMB_BYTES;   // half a limb
    static ConfiguredMask configured;
    cudaError_t e = set_smem_once(configured, lc.device, smem, kern);
    if (e != cudaSuccess) return e;
    const size_t pairs = n_limbs < 0x3fffffffull ? n_limbs : 0x3fffffffull;
    kern<<<(unsigned)(2 * pairs), NT, smem, st>>>(data, INV ? lc.itw : lc.tw, lc.lt, lc.L, n_limbs);
    return cudaGetLastError();
}

cudaError_t launch_ntt(const LaunchCtx &lc, u64 *data, size_t n_polys, bool inverse, cudaStream_t st) {
    const size_t n_limbs = n_polys * lc.L;
    if (n_limbs == 0) return cudaSuccess;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        if constexpr (LOGN == 12) {
            return launch_ntt_dir<12, 256, 2>(lc, data, n_limbs, inverse, st);
        } else if constexpr (LOGN == 13) {
            switch (lc.ntt_cfg) {   // tuning variants (DPFHE_NTT_CFG), default 0
                case 1: return launch_ntt_dir<13, 512, 1>(lc, data, n_limbs, inverse, st);   //  9.9 M NTT/s
                case 2: return launch_ntt_dir<13, 512, 2>(lc, data, n_limbs, inverse, st);   // 12.6 M (64 regs, spills)
                case 3: return launch_ntt_dir<13, 256, 2>(lc, data, n_limbs, inverse, st);   // 12.3 M
                default: return launch_ntt_dir<13, 256, 3>(lc, data, n_limbs, inverse, st);  // 13.2 M: 3 CTAs/SM (smem-limited), 80 regs
            }
        } else {
            if (lc.ntt_cfg == 1) return launch_ntt_dir<14, 512, 1>(lc, data, n_limbs, inverse, st);   // whole limb per CTA, 1 CTA/SM
            // CTA pair per limb, 3 CTAs/SM
            return inverse ? launch_ntt_pair_t<true>(lc, data, n_limbs, st) : launch_ntt_pair_t<false>(lc, data, n_limbs, st);
        }
    });
}

cudaError_t launch_mod_switch(const LaunchCtx &lc, const u64 *in, u64 *tau, u64 *out, const MsConsts &K, size_t n_polys, cudaStream_t st) {
    if (n_polys == 0) return cudaSuccess;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value, NT = LOGN == 14 ? 512 : 256, MINB = LOGN == 12 ? 2 : LOGN == 13 ? 3 : 1;
        const size_t smem = Geometry<LOGN>::LIMB_BYTES;
        auto k1 = ms_tau_kernel<LOGN, NT, MINB>;
        auto k2 = ms_limb_kernel<LOGN, NT, MINB>;
        static ConfiguredMask configured;
        cudaError_t e = set_smem_once(configured, lc.device, smem, k1, k2);
        if (e != cudaSuccess) return e;
        const size_t n_items = n_polys * (lc.L - 1);
        k1<<<(unsigned)(n_polys < 0x7fffffffull ? n_polys : 0x7fffffffull), NT, smem, st>>>(in, tau, lc.itw, lc.lt, K, lc.L, n_polys);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        k2<<<(unsigned)(n_items < 0x7fffffffull ? n_items : 0x7fffffffull), NT, smem, st>>>(in, tau, out, lc.tw, lc.lt, K, lc.L, n_items);
        return cudaGetLastError();
    });
}

// in [n_polys][L][N] -> out [n_polys][L-K][N]; tau: n_polys * K * N words of scratch
cudaError_t launch_mod_down_special(const LaunchCtx &lc, const u64 *in, u64 *tau, u64 *out, const MsConsts &K, const GroupConsts &G, size_t n_polys,
                                    cudaStream_t st) {
    if (n_polys == 0) return cudaSuccess;
    if (G.Lq + G.K != lc.L) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value, NT = LOGN == 14 ? 512 : 256, MINB = LOGN == 12 ? 2 : LOGN == 13 ? 3 : 1;
        const size_t smem = Geometry<LOGN>::LIMB_BYTES;
        auto k1 = md_tau_kernel<LOGN, NT, MINB>;
        auto k2 = md_limb_kernel<LOGN, NT, MINB>;
        static ConfiguredMask configured;
        cudaError_t e = set_smem_once(configured, lc.device, smem, k1, k2);
        if (e != cudaSuccess) return e;
        const size_t n_tau = n_polys * G.K, n_items = n_polys * G.Lq;
        k1<<<(unsigned)(n_tau < 0x7fffffffull ? n_tau : 0x7fffffffull), NT, smem, st>>>(in, tau, lc.itw, K, G, n_tau);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        k2<<<(unsigned)(n_items < 0x7fffffffull ? n_items : 0x7fffffffull), NT, smem, st>>>(in, tau, out, lc.tw, lc.lt, K, G, n_items);
        return cudaGetLastError();
    });
}

// ---- CKKS slot encoding
constexpr int CKKS_FFT_NT = 512;

cudaError_t launch_ckks_encode(const LaunchCtx &lc, const Cplx *slots, double *coeffs, u64 *pt, const CkksTables &T, double sc, size_t n_vec,
                               cudaStream_t st) {
    if (n_vec == 0) return cudaSuccess;
    if (n_vec * lc.L * 2 > 0x7fffffffull) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        auto kf = ckks_enc_fft_kernel<LOGN, CKKS_FFT_NT>;
        const size_t smem_fft = ((size_t)1 << (LOGN - 1)) * sizeof(Cplx);
        static ConfiguredMask conf_fft, conf_ntt;
        cudaError_t e = set_smem_once(conf_fft, lc.device, smem_fft, kf);
        if (e != cudaSuccess) return e;
        kf<<<(unsigned)n_vec, CKKS_FFT_NT, smem_fft, st>>>(slots, coeffs, T.tw, T.tj, sc);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        const size_t n_limbs = n_vec * lc.L;
        if constexpr (LOGN == NTT_PAIR_LOGN) {
            auto kn = ckks_enc_ntt_pair_kernel<256, 2>;   // at 3 CTAs per SM (80 registers) the reducing load stage spills
            const size_t smem = Geometry<13>::LIMB_BYTES;   // half a limb
            e = set_smem_once(conf_ntt, lc.device, smem, kn);
            if (e != cudaSuccess) return e;
            kn<<<(unsigned)(2 * n_limbs), 256, smem, st>>>(coeffs, pt, lc.tw, T.pow2, lc.lt, lc.L);
        } else {
            constexpr int MINB = LOGN == 12 ? 2 : 3;
            auto kn = ckks_enc_ntt_kernel<LOGN, 256, MINB>;
            const size_t smem = Geometry<LOGN>::LIMB_BYTES;
            e = set_smem_once(conf_ntt, lc.device, smem, kn);
            if (e != cudaSuccess) return e;
            kn<<<(unsigned)n_limbs, 256, smem, st>>>(coeffs, pt, lc.tw, T.pow2, lc.lt, lc.L);
        }
        return cudaGetLastError();
    });
}

// work: [n_vec][L][N] inverse transforms of the plaintexts (overwritten)
cudaError_t launch_ckks_decode(const LaunchCtx &lc, u64 *work, Cplx *slots, const CkksTables &T, const CkksConsts &K, size_t n_vec, cudaStream_t st) {
    if (n_vec == 0) return cudaSuccess;
    if (n_vec > 0x7fffffffull) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        auto kd = ckks_dec_kernel<LOGN, CKKS_FFT_NT>;
        const size_t smem = ((size_t)1 << (LOGN - 1)) * sizeof(Cplx);
        static ConfiguredMask conf;
        cudaError_t e = set_smem_once(conf, lc.device, smem, kd);
        if (e != cudaSuccess) return e;
        kd<<<(unsigned)n_vec, CKKS_FFT_NT, smem, st>>>(work, slots, T.tw, T.tj, lc.lt, K, lc.L);
        return cudaGetLastError();
    });
}

// ---- BGV slot encoding
constexpr int BGV_NT = 512;

// coeffs: [n_vec][N] words of scratch
cudaError_t launch_bgv_encode(const LaunchCtx &lc, const int64_t *slots, u32 *coeffs, u64 *pt, const BgvTables &T, size_t n_vec, cudaStream_t st) {
    if (n_vec == 0) return cudaSuccess;
    if (n_vec * lc.L * 2 > 0x7fffffffull) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        auto ke = bgv_enc_kernel<LOGN, BGV_NT>;
        const size_t smem_t = ((size_t)1 << LOGN) * sizeof(u32);
        static ConfiguredMask conf_enc, conf_ntt;
        cudaError_t e = set_smem_once(conf_enc, lc.device, smem_t, ke);
        if (e != cudaSuccess) return e;
        ke<<<(unsigned)n_vec, BGV_NT, smem_t, st>>>(slots, coeffs, T);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        const size_t n_limbs = n_vec * lc.L;
        if constexpr (LOGN == NTT_PAIR_LOGN) {
            auto kn = bgv_enc_ntt_pair_kernel<256, 2>;
            const size_t smem = Geometry<13>::LIMB_BYTES;   // half a limb
            e = set_smem_once(conf_ntt, lc.device, smem, kn);
            if (e != cudaSuccess) return e;
            kn<<<(unsigned)(2 * n_limbs), 256, smem, st>>>(coeffs, pt, lc.tw, T.m.t, lc.lt, lc.L);
        } else {
            constexpr int MINB = LOGN == 12 ? 2 : 3;
            auto kn = bgv_enc_ntt_kernel<LOGN, 256, MINB>;
            const size_t smem = Geometry<LOGN>::LIMB_BYTES;
            e = set_smem_once(conf_ntt, lc.device, smem, kn);
            if (e != cudaSuccess) return e;
            kn<<<(unsigned)n_limbs, 256, smem, st>>>(coeffs, pt, lc.tw, T.m.t, lc.lt, lc.L);
        }
        return cudaGetLastError();
    });
}

// work: [n_vec][L][N] inverse transforms of the plaintexts (overwritten)
cudaError_t launch_bgv_decode(const LaunchCtx &lc, u64 *work, u64 *slots, const BgvTables &T, const BgvConsts &K, size_t n_vec, cudaStream_t st) {
    if (n_vec == 0) return cudaSuccess;
    if (n_vec > 0x7fffffffull) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        auto kd = bgv_dec_kernel<LOGN, BGV_NT>;
        const size_t smem = ((size_t)1 << LOGN) * sizeof(u32);
        static ConfiguredMask conf;
        cudaError_t e = set_smem_once(conf, lc.device, smem, kd);
        if (e != cudaSuccess) return e;
        kd<<<(unsigned)n_vec, BGV_NT, smem, st>>>(work, slots, T, lc.lt, K, lc.L);
        return cudaGetLastError();
    });
}

#endif
// Flag, round-mark and mailbox tags are 32-bit round numbers compared by signed difference, so a slot last written more than 2^31
// rounds ago would look "published" (a context that has multiplied 2^31 ciphertexts: an hour of work).  Long before that the
// numbering restarts: flags, marks, mailboxes and hand-back counters are cleared in stream order - after every earlier launch of
// the context (abi.cu orders its calls) and before this one - and the epoch returns to zero.
static cudaError_t epoch_guard(LaunchCtx &lc, size_t batch, cudaStream_t st) {
    if (batch + 1 >= 0x40000000ull) return cudaErrorInvalidValue;
    if ((unsigned long long)lc.ks_epoch + batch + 1 < lc.ks_epoch_limit) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(lc.ks_flags, 0, 2 * lc.ks_slots * sizeof(u32), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(lc.ks_mail, 0, lc.ks_slots * sizeof(u64), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(lc.ks_consumed, 0, lc.ks_slots * sizeof(u32), st);
    if (e != cudaSuccess) return e;
    lc.ks_epoch = 0;
    ++lc.ks_epoch_restarts;
    return cudaSuccess;
}

// the round state every persistent kernel takes (batch, flags, epoch, ticket, mailboxes): its parameter array points here, and
// launch_persistent fills it once the round numbering is settled
struct Rounds {
    size_t batch;
    u32 *flags;
    u32 epoch;
    u32 *ticket;
    u64 *mail;
};

// One launch of a persistent key-switch kernel (256 threads per CTA).  The spin-waits need every CTA of the grid resident, so the
// grid is what fits at once: the resident CTAs (occupancy per SM, or with cluster > 1 whole clusters of that many CTAs), capped by
// DPFHE_KS_OCC per SM when occ_cap, then by lc.ks_slots, rounded down to whole groups of `group` CTAs and to at most `batch`
// groups.  Clears the ticket, and advances the round numbering by the batch + 1 rounds a launch may consume, whether or not the
// launch call succeeded.  cluster == 0: cudaLaunchCooperativeKernel; cluster >= 1 (ks_fused_kernel): cudaLaunchKernelExC,
// cooperative, with the cluster dimension when > 1 and the DPFHE_L2_PERSIST window.
template <class Kern>
static cudaError_t launch_persistent(LaunchCtx &lc, Kern kern, ConfiguredMask &configured, size_t group, size_t smem, size_t batch, Rounds &r,
                                     void **params, cudaStream_t st, bool occ_cap = true, int cluster = 0) {
    constexpr int NT = 256;
    cudaError_t e = set_smem_once(configured, lc.device, smem, kern);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[3];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    int n_attr = cluster > 1 ? 2 : 1;
    size_t G = 0;   // resident CTAs
    if (cluster > 1) {
        cfg.gridDim = dim3(cluster);
        cfg.attrs = attr + 1;
        cfg.numAttrs = 1;
        int clusters = 0;
        e = cudaOccupancyMaxActiveClusters(&clusters, (const void *)kern, &cfg);
        if (e != cudaSuccess) return e;
        G = (size_t)clusters * cluster;
    } else {
        int occ = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, NT, smem);
        if (e != cudaSuccess) return e;
        G = (size_t)lc.num_sms * occ;
    }
    if (G == 0) return cudaErrorLaunchOutOfResources;
    if (occ_cap && lc.ks_occ_cap > 0 && G > (size_t)lc.num_sms * lc.ks_occ_cap) G = (size_t)lc.num_sms * lc.ks_occ_cap;
    if (G > lc.ks_slots) G = lc.ks_slots;
    G = (G / group) * group;
    if (G > batch * group) G = batch * group;
    if (G == 0) return cudaErrorInvalidConfiguration;
    e = epoch_guard(lc, batch, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(lc.ks_ticket, 0, sizeof(u32), st);
    if (e != cudaSuccess) return e;
    r = Rounds{batch, lc.ks_flags, lc.ks_epoch, lc.ks_ticket, lc.ks_mail};
    if (cluster == 0) {
        e = cudaLaunchCooperativeKernel((const void *)kern, dim3((unsigned)G), dim3(NT), params, smem, st);
    } else {
        if (lc.l2_persist && lc.l2_persist_max && lc.ks_window_bytes) {
            // tuning (DPFHE_L2_PERSIST): the digit slots (and at N = 16384 the accumulator rows) are re-read within microseconds,
            // the ciphertext streams never; a persisting access-policy window over the scratch keeps the streams from evicting it
            attr[n_attr].id = cudaLaunchAttributeAccessPolicyWindow;
            attr[n_attr].val.accessPolicyWindow.base_ptr = lc.ks_scratch;
            attr[n_attr].val.accessPolicyWindow.num_bytes = lc.ks_window_bytes;
            const double ratio = (double)lc.l2_persist_max / (double)lc.ks_window_bytes;
            attr[n_attr].val.accessPolicyWindow.hitRatio = (float)(ratio > 1.0 ? 1.0 : ratio);
            attr[n_attr].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
            attr[n_attr].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
            ++n_attr;
        }
        // never launched without the co-residency guarantee: if the runtime refuses the combination, the call returns its error
        cfg.gridDim = dim3((unsigned)G);
        cfg.attrs = attr;
        cfg.numAttrs = (unsigned)n_attr;
        e = cudaLaunchKernelExC(&cfg, (const void *)kern, params);
    }
    lc.ks_epoch += (u32)(batch + 1);
    return e;
}

// the key-switch arguments of the fused, hybrid and grouped kernels: L ciphertext limbs (digits), key rows of Lk limbs.  Set for the
// special-prime kernels (their digit rows and double accumulators); launch_ks resets the fields the fused kernel uses otherwise.
static KsArgs ks_args(const LaunchCtx &lc, const u64 *a, const u64 *b, const u64 *key, const u64 *key_s, u64 *out, u32 L, u32 galois, u32 Lk,
                      bool lift_reduce) {
    KsArgs A;
    A.a = a; A.b = b; A.key = key; A.key_s = key_s; A.out = out; A.scratch = lc.ks_scratch;
    A.tw = lc.tw; A.itw = lc.itw; A.L = L; A.galois = galois; A.Lk = Lk; A.hyb = lc.ks_hyb; A.only = nullptr;
    A.acc = lc.ks_acc_hyb; A.acc_par = 2; A.lift_reduce = lift_reduce ? 1u : 0u;
    return A;
}

// Shoup companions of the first `rows` rows of a switch key [rows][2][L][N] into key_s (same layout)
template <int LOGN>
static cudaError_t launch_key_prepare_t(const LaunchCtx &lc, const u64 *key, u64 *key_s, size_t rows, cudaStream_t st) {
    const size_t n = (size_t)2 * rows * lc.L << LOGN;
    key_prepare_kernel<LOGN><<<ew_grid(lc, n), 256, 0, st>>>(key, key_s, lc.lp, lc.L, n);
    return cudaGetLastError();
}

// grid of the gather kernels (rot_apply, rot_apply_grouped, rot_sum_grouped): `rows` work rows, cut into up to NC / 256 segments
// (nseg) so that small batches still fill the machine several times over, at most 8 CTAs per SM
static inline unsigned gather_grid(const LaunchCtx &lc, size_t rows, u32 &nseg) {
    const size_t want = (size_t)lc.num_sms * 12;
    const u32 max_seg = (1u << (lc.log_n - 1)) / 256;
    nseg = 1;
    while (nseg < max_seg && rows * nseg < want) nseg *= 2;
    const size_t n_items = rows * nseg, cap = (size_t)lc.num_sms * 8;
    return (unsigned)(n_items < cap ? n_items : cap);
}

#if DPFHE_PART_MAIN
cudaError_t launch_key_prepare(const LaunchCtx &lc, const u64 *key, u64 *key_s, u32 rows, cudaStream_t st) {
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) { return launch_key_prepare_t<decltype(lg)::value>(lc, key, key_s, rows, st); });
}

template <int LOGN, int MODE>
static cudaError_t launch_ks_t(LaunchCtx &lc, const KsArgs &A, size_t batch, cudaStream_t st) {
    // N <= 8192: a 4096-point block and two accumulator half-rows, 96 KiB of shared memory -> two CTAs per SM, CTA pairs of a
    // cluster at N = 8192.  N = 16384: 64 KiB (two half-limbs in turn) -> three CTAs per SM.
    constexpr bool BLK = LOGN <= 13;
    constexpr int NT = 256, MINB = BLK ? 2 : 3, PAIR = BLK ? ks_blk_pair<LOGN>() : 1;
    const bool filter = A.only != nullptr;
    if (filter && MODE != KS_ROTATE) return cudaErrorInvalidValue;
    auto kern = ks_fused_kernel<LOGN, NT, MINB, MODE, false>;
    if constexpr (MODE == KS_MUL_RELIN) {   // the per-phase clock counters (DPFHE_KS_PROF, tools/phase_prof.py) exist for ct x ct only
        if (lc.ks_prof) kern = ks_fused_kernel<LOGN, NT, MINB, MODE, true>;
    }
    if (filter) kern = ks_fused_kernel<LOGN, NT, MINB, MODE == KS_ROTATE ? MODE : KS_ROTATE, false, MODE == KS_ROTATE>;
    const size_t smem = BLK ? 3 * Geometry<KS_BLK_LOGN>::LIMB_BYTES : Geometry<13>::LIMB_BYTES;
    static ConfiguredMask configured[3];
    const int variant = filter ? 2 : (lc.ks_prof && MODE == KS_MUL_RELIN ? 1 : 0);
    KsArgs args = A;
    LimbTable lt = lc.lt;
    unsigned long long *prof = lc.ks_prof;
    u32 pf_dist = (u32)lc.ks_prefetch;
    u32 *consumed = !BLK && lc.ks_single ? lc.ks_consumed : nullptr;   // single-buffered digit slots: N = 16384 only
    Rounds r;
    void *params[] = {&args, &lt, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail, &prof, &pf_dist, &consumed};
    return launch_persistent(lc, kern, configured[variant], (size_t)lc.L * PAIR, smem, batch, r, params, st, true, PAIR);
}

cudaError_t launch_ks(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch,
                      u32 galois, cudaStream_t st, const u32 *only, bool key_ready, const u64 *key_s) {
    if (batch == 0) return cudaSuccess;
    return with_log_n(lc.log_n, cudaErrorNotSupported, [&](auto lg) -> cudaError_t {
        constexpr int LOGN = decltype(lg)::value;
        // Shoup companions of the key for this launch (2*L*P words, a few microseconds; batch-amortised)
        if (!key_ready) {
            cudaError_t e = launch_key_prepare_t<LOGN>(lc, key, lc.ks_key_s, lc.L, st);
            if (e != cudaSuccess) return e;
        }
        KsArgs A = ks_args(lc, a, b, key, key_ready && key_s ? key_s : lc.ks_key_s, out, lc.L, galois, lc.L, lc.lift_reduce);
        A.hyb = nullptr; A.only = only; A.acc = lc.ks_acc; A.acc_par = 1;
        switch (mode) {
            case KS_MUL_RELIN: return launch_ks_t<LOGN, KS_MUL_RELIN>(lc, A, batch, st);
            case KS_PLAIN: return launch_ks_t<LOGN, KS_PLAIN>(lc, A, batch, st);
            case KS_ROTATE: return launch_ks_t<LOGN, KS_ROTATE>(lc, A, batch, st);
        }
        return cudaErrorInvalidValue;
    });
}

#endif
#if DPFHE_PART_HYBRID
template <int LOGN, int MODE, bool LV>
static cudaError_t launch_ks_hybrid_t(LaunchCtx &lc, const KsArgs &A, const MsConsts &K, size_t batch, cudaStream_t st) {
    constexpr int NT = 256, MINB = 3;
    auto kern = ks_hybrid_kernel<LOGN, NT, MINB, MODE>;
    if constexpr (LV) kern = ks_hybrid_level_kernel<LOGN, NT, MINB, MODE>;
    static ConfiguredMask configured;
    KsArgs args = A;
    LimbTable lt = lc.lt;
    MsConsts consts = K;
    Rounds r;
    void *params[] = {&args, &lt, &consts, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail};
    // group: L-1 ciphertext limbs + the special limb
    return launch_persistent(lc, kern, configured, lc.L, Geometry<LOGN>::KS_SMEM, batch, r, params, st);
}

// data has L-1 limbs, the key [L-1][2][key_L][N]; lc.ks_hyb must hold (ks_slots / 2 + 1) * KS_HYB_ROWS * N words and lc.ks_acc_hyb
// ks_slots * 2 * 2 * N words.  key_s == nullptr: the top-level call, modes KS_MUL_RELIN, KS_PLAIN and KS_ROTATE, the key's companions
// built here into lc.ks_key_s.  key_s given: the call at level l (DESIGN.md §4.17), modes KS_MUL_RELIN and KS_ROTATE: lc is the level's
// view (L = l + 1 limbs, its own tables), key the top-level key with key_L limbs per row and its companions key_s, built by the caller
// over the top-level rows.
cudaError_t launch_ks_hybrid(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch, u32 galois,
                             const MsConsts &K, cudaStream_t st, const u64 *key_s, u32 key_L) {
    if (batch == 0) return cudaSuccess;
    const bool level = key_s != nullptr;
    if (lc.L < 2 || (level && key_L < lc.L) || !lc.ks_hyb || !lc.ks_acc_hyb) return cudaErrorInvalidValue;
    return with_log_n(lc.log_n, cudaErrorNotSupported, [&](auto lg) -> cudaError_t {
        constexpr int LOGN = decltype(lg)::value;
        if (!level) {
            cudaError_t e = launch_key_prepare_t<LOGN>(lc, key, lc.ks_key_s, lc.L - 1, st);
            if (e != cudaSuccess) return e;
        }
        const KsArgs A = ks_args(lc, a, b, key, level ? key_s : lc.ks_key_s, out, lc.L - 1, galois, level ? key_L : lc.L, lc.lift_reduce);
        switch (mode) {
            case KS_MUL_RELIN:
                return level ? launch_ks_hybrid_t<LOGN, KS_MUL_RELIN, true>(lc, A, K, batch, st) : launch_ks_hybrid_t<LOGN, KS_MUL_RELIN, false>(lc, A, K, batch, st);
            case KS_PLAIN:
                if (!level) return launch_ks_hybrid_t<LOGN, KS_PLAIN, false>(lc, A, K, batch, st);
                break;
            case KS_ROTATE:
                return level ? launch_ks_hybrid_t<LOGN, KS_ROTATE, true>(lc, A, K, batch, st) : launch_ks_hybrid_t<LOGN, KS_ROTATE, false>(lc, A, K, batch, st);
        }
        return cudaErrorInvalidValue;
    });
}

#endif
#if DPFHE_PART_GROUPED
// one launch of a grouped kernel: ks_grouped_kernel (ADD: with the addend), ct_dot_grouped_kernel (MODE = KS_DOT),
// ks_rescale_grouped_kernel (RS) or ks_level_grouped_kernel (LV; RS: with the division by the dropped limb).  Groups of L CTAs:
// every limb of the context, ciphertext and special.
template <int LOGN, int MODE, bool ADD = false, bool RS = false, bool LV = false>
static cudaError_t launch_ks_grouped_t(LaunchCtx &lc, KsArgs A, MsConsts K, GroupConsts G, DotArgs D, RescaleConsts R, const u64 *addend,
                                       size_t batch, cudaStream_t st) {
    constexpr int NT = 256, MINB = 3;
    constexpr size_t smem = Geometry<LOGN>::KS_SMEM;
    static ConfiguredMask configured;
    LimbTable lt = lc.lt;
    Rounds r;
    if constexpr (LV && ADD) {
        void *params[] = {&A, &lt, &K, &G, &D, &R, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail, &addend};
        return launch_persistent(lc, ks_level_horner_kernel<LOGN, NT, MINB>, configured, lc.L, smem, batch, r, params, st);
    } else if constexpr (LV || RS) {
        void *params[] = {&A, &lt, &K, &G, &D, &R, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail};
        if constexpr (LV) return launch_persistent(lc, ks_level_grouped_kernel<LOGN, NT, MINB, MODE, RS>, configured, lc.L, smem, batch, r, params, st);
        else return launch_persistent(lc, ks_rescale_grouped_kernel<LOGN, NT, MINB, MODE>, configured, lc.L, smem, batch, r, params, st);
    } else if constexpr (MODE == KS_DOT) {
        void *params[] = {&A, &lt, &K, &G, &D, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail};
        return launch_persistent(lc, ct_dot_grouped_kernel<LOGN, NT, MINB>, configured, lc.L, smem, batch, r, params, st);
    } else {
        void *params[] = {&A, &lt, &K, &G, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail, &addend};
        return launch_persistent(lc, ks_grouped_kernel<LOGN, NT, MINB, MODE, ADD>, configured, lc.L, smem, batch, r, params, st);
    }
}

// Every grouped key-switching call (data of Gc.Lq = L - K limbs, the key [dnum][2][key rows][N]; scratch requirements as
// launch_ks_hybrid, K <= Lq keeping the special CTAs' rows within lc.ks_hyb):
//   mode KS_MUL_RELIN / KS_PLAIN / KS_ROTATE on a[0], b[0] (galois; addend, KS_ROTATE only: out = rotation + addend), or KS_DOT on
//   the n_terms (1 .. DOT_MAX_TERMS) pairs a[t], b[t] (DESIGN.md §2.18); host arrays of device pointers;
//   R non-null: multiply-and-rescale (DESIGN.md §2.19, modes KS_MUL_RELIN and KS_DOT): out [batch][2][Lq-1][N], divided by
//   P * q_{Lq-1}; the dropped limb's rows and flags are lc.ks_tau_drop, which must hold (ks_slots / 3 + 1) * 4 * N words (a group has
//   L >= 3 CTAs), and one flag per group in the second half of lc.ks_flags, whose words ks_hoistg_kernel uses as round marks in
//   other launches: a tag is always above what an earlier launch left;
//   key_L > 0: the call at level l (DESIGN.md §2.20, §4.17, modes KS_MUL_RELIN, KS_ROTATE, KS_DOT): lc is the level's view (L = l + K
//   limbs, its own tables and Gc built on them), key the top-level key with key_L limbs per row and its companions key_s, built by
//   the caller over the top-level rows of the level's digits.
// key_s == nullptr (top level only): the companions are built here into lc.ks_key_s, one more launch.
static cudaError_t ks_grouped(LaunchCtx &lc, int mode, const u64 *const *a, const u64 *const *b, u32 n_terms, u32 galois, const u64 *addend,
                              const u64 *key, const u64 *key_s, u32 key_L, const RescaleConsts *R, u64 *out, size_t batch, const MsConsts &K,
                              const GroupConsts &Gc, cudaStream_t st) {
    if (batch == 0) return cudaSuccess;
    const bool level = key_L != 0, dot = mode == KS_DOT;
    if (lc.L < 2 || !lc.ks_hyb || !lc.ks_acc_hyb || Gc.Lq + Gc.K != lc.L || Gc.K > Gc.Lq || Gc.K > (u32)KS_MAX_SPECIAL) return cudaErrorInvalidValue;
    if ((level && (key_L < lc.L || !key_s)) || (addend && mode != KS_ROTATE)) return cudaErrorInvalidValue;
    if (R && (mode == KS_ROTATE || lc.L < 3 || Gc.Lq < 2 || !lc.ks_tau_drop)) return cudaErrorInvalidValue;
    if (n_terms < 1 || n_terms > (u32)DOT_MAX_TERMS || (!dot && n_terms != 1)) return cudaErrorInvalidValue;
    DotArgs D{};
    for (u32 t = 0; dot && t < n_terms; ++t) {
        D.a[t] = a[t];
        D.b[t] = b[t];
    }
    if (dot) D.n_terms = n_terms;
    RescaleConsts Rc{};
    if (R) {
        Rc = *R;
        Rc.tau = lc.ks_tau_drop;
        Rc.tau_flag = lc.ks_flags + lc.ks_slots;
    }
    return with_log_n(lc.log_n, cudaErrorNotSupported, [&](auto lg) -> cudaError_t {
        constexpr int LOGN = decltype(lg)::value;
        if (!key_s) {
            cudaError_t e = launch_key_prepare_t<LOGN>(lc, key, lc.ks_key_s, Gc.dnum, st);
            if (e != cudaSuccess) return e;
            key_s = lc.ks_key_s;
        }
        const KsArgs A = ks_args(lc, dot ? nullptr : a[0], dot || !b ? nullptr : b[0], key, key_s, out, Gc.Lq, galois, level ? key_L : lc.L, false);
        if (level) {
            switch (mode) {
                case KS_ROTATE:
                    if (addend) return launch_ks_grouped_t<LOGN, KS_ROTATE, true, false, true>(lc, A, K, Gc, D, Rc, addend, batch, st);
                    return launch_ks_grouped_t<LOGN, KS_ROTATE, false, false, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
                case KS_MUL_RELIN:
                    if (R) return launch_ks_grouped_t<LOGN, KS_MUL_RELIN, false, true, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
                    return launch_ks_grouped_t<LOGN, KS_MUL_RELIN, false, false, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
                case KS_DOT:
                    if (R) return launch_ks_grouped_t<LOGN, KS_DOT, false, true, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
                    return launch_ks_grouped_t<LOGN, KS_DOT, false, false, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
            }
            return cudaErrorInvalidValue;
        }
        if (R) return dot ? launch_ks_grouped_t<LOGN, KS_DOT, false, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st)
                          : launch_ks_grouped_t<LOGN, KS_MUL_RELIN, false, true>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
        switch (mode) {
            case KS_MUL_RELIN: return launch_ks_grouped_t<LOGN, KS_MUL_RELIN>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
            case KS_PLAIN: return launch_ks_grouped_t<LOGN, KS_PLAIN>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
            case KS_ROTATE:
                if (addend) return launch_ks_grouped_t<LOGN, KS_ROTATE, true>(lc, A, K, Gc, D, Rc, addend, batch, st);
                return launch_ks_grouped_t<LOGN, KS_ROTATE>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
            case KS_DOT: return launch_ks_grouped_t<LOGN, KS_DOT>(lc, A, K, Gc, D, Rc, nullptr, batch, st);
        }
        return cudaErrorInvalidValue;
    });
}

// the entry points of ks_grouped: one ct x ct product, plain switch or rotation; the inner product; multiply-and-rescale; level calls
cudaError_t launch_ks_grouped(LaunchCtx &lc, int mode, const u64 *a, const u64 *b, const u64 *key, u64 *out, size_t batch, u32 galois,
                              const MsConsts &K, const GroupConsts &Gc, cudaStream_t st, const u64 *addend, const u64 *key_s) {
    if (batch && mode == KS_DOT) return cudaErrorInvalidValue;
    return ks_grouped(lc, mode, &a, &b, 1, galois, addend, key, key_s, 0, nullptr, out, batch, K, Gc, st);
}

cudaError_t launch_ct_dot_grouped(LaunchCtx &lc, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, u64 *out, size_t batch,
                                  const MsConsts &K, const GroupConsts &Gc, cudaStream_t st, const u64 *key_s) {
    return ks_grouped(lc, KS_DOT, a, b, n_terms, 0, nullptr, key, key_s, 0, nullptr, out, batch, K, Gc, st);
}

cudaError_t launch_ks_rescale_grouped(LaunchCtx &lc, bool dot, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, u64 *out,
                                      size_t batch, const MsConsts &K, const GroupConsts &Gc, const RescaleConsts &R, cudaStream_t st,
                                      const u64 *key_s) {
    return ks_grouped(lc, dot ? KS_DOT : KS_MUL_RELIN, a, b, n_terms, 0, nullptr, key, key_s, 0, &R, out, batch, K, Gc, st);
}

cudaError_t launch_ks_grouped_level(LaunchCtx &lc, int mode, const u64 *const *a, const u64 *const *b, u32 n_terms, const u64 *key, const u64 *key_s,
                                    u32 key_L, u64 *out, size_t batch, u32 galois, const MsConsts &K, const GroupConsts &Gc, const RescaleConsts *R,
                                    cudaStream_t st, const u64 *addend) {
    if (batch && !key_L) return cudaErrorInvalidValue;
    return ks_grouped(lc, mode, a, b, n_terms, galois, addend, key, key_s, key_L, R, out, batch, K, Gc, st);
}

#endif
#if DPFHE_PART_MAIN
// shared-memory plan of pt_inner_kernel: two CTAs per SM (113 KiB each); the plaintext tile takes nb * 128 bytes per
// giant step and the two ciphertext-row buffers 2 * nb * 128 bytes each.  Returns giant steps per launch (0: nb too large).
static constexpr size_t PTI_SMEM_BUDGET = (size_t)113 << 10;
static u32 pt_inner_gmax(u32 nb) {
    const size_t row = (size_t)nb * PTI_COEFFS * 8;
    if (5 * row > PTI_SMEM_BUDGET) return 0;
    u32 gmax = (u32)((PTI_SMEM_BUDGET - 4 * row) / row);
    if (gmax >= 8) gmax -= gmax % 8;   // whole rounds of the CTA's eight warps
    return gmax;
}

// out[g] = sum_b steps[b] o pts[g][b]; returns the number of kernel launches through *launches
cudaError_t launch_pt_inner(const LaunchCtx &lc, const u64 *steps, u32 nb, const u64 *pts, u32 ng, u64 *out, size_t batch, cudaStream_t st,
                            unsigned *launches) {
    *launches = 0;
    if (!batch || !nb || !ng) return cudaSuccess;
    PtInnerArgs A;
    A.steps = steps; A.pts = pts; A.out = out; A.batch = batch; A.L = lc.L; A.nb = nb; A.ng = ng;
    const u32 gmax = pt_inner_gmax(nb);
    if (gmax == 0) return cudaErrorInvalidValue;
    *launches = (ng + gmax - 1) / gmax;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value, NT = 256, MINB = 2;
        auto kern = pt_inner_kernel<LOGN, NT, MINB>;
        static ConfiguredMask configured;
        cudaError_t e = set_smem_once(configured, lc.device, PTI_SMEM_BUDGET, kern);
        if (e != cudaSuccess) return e;
        const size_t row = (size_t)A.nb * PTI_COEFFS * 8;
        const unsigned grid = (unsigned)(lc.L * (((size_t)1 << LOGN) / PTI_COEFFS));
        for (u32 g0 = 0; g0 < A.ng; g0 += gmax) {
            const u32 gcnt = A.ng - g0 < gmax ? A.ng - g0 : gmax;
            kern<<<grid, NT, ((size_t)gcnt + 4) * row, st>>>(A, lc.lt, g0, gcnt);
            e = cudaGetLastError();
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    });
}

// hoisted rotations, step 1: U[ct][j][i] and the zero flags of `batch` ciphertexts (L >= 2)
cudaError_t launch_hoist(LaunchCtx &lc, const u64 *ct, u64 *U, u32 *zero, size_t batch, cudaStream_t st) {
    if (batch == 0) return cudaSuccess;
    HoistArgs A;
    A.ct = ct; A.U = U; A.scratch = lc.ks_scratch; A.zero = zero; A.tw = lc.tw; A.itw = lc.itw; A.L = lc.L;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        static ConfiguredMask configured;
        LimbTable lt = lc.lt;
        Rounds r;
        void *params[] = {&A, &lt, &r.batch, &r.flags, &r.epoch, &r.ticket, &r.mail};
        // groups of L CTAs; DPFHE_KS_OCC does not apply
        return launch_persistent(lc, ks_hoist_kernel<LOGN, 256, 3>, configured, lc.L, Geometry<LOGN>::KS_SMEM, batch, r, params, st, false);
    });
}

#endif
#if DPFHE_PART_GROUPED
// hoisted rotations with grouped hybrid keys, step 1: U [batch][dnum][L][N]
cudaError_t launch_hoist_grouped(LaunchCtx &lc, const u64 *ct, u64 *U, const GroupConsts &G, size_t batch, cudaStream_t st) {
    if (batch == 0) return cudaSuccess;
    if (G.Lq + G.K != lc.L) return cudaErrorInvalidValue;
    HoistGArgs A;
    A.ct = ct; A.U = U; A.scratch = lc.ks_scratch; A.tw = lc.tw; A.itw = lc.itw;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        static ConfiguredMask configured;
        LimbTable lt = lc.lt;
        GroupConsts gc = G;
        u32 *done = lc.ks_flags + lc.ks_slots;   // second half of the flag array: "round finished" marks
        Rounds r;
        void *params[] = {&A, &lt, &gc, &r.batch, &r.flags, &done, &r.epoch, &r.ticket, &r.mail};
        // groups of L CTAs; DPFHE_KS_OCC does not apply
        return launch_persistent(lc, ks_hoistg_kernel<LOGN, 256, 3>, configured, lc.L, Geometry<LOGN>::KS_SMEM, batch, r, params, st, false);
    });
}

// step 2: acc [batch][2][L][N] of one rotation (key companions built here into lc.ks_key_s unless the caller supplies them)
// key_shift > 0: a level view reading a top-level key (rot_apply_grouped_level_kernel, DESIGN.md §4.18), its companions required
cudaError_t launch_rot_apply_grouped(LaunchCtx &lc, const u64 *ct, const u64 *U, const u64 *key, const u64 *key_s, u32 galois, u64 *acc,
                                     const MsConsts &K, const GroupConsts &G, size_t batch, cudaStream_t st, u32 key_shift) {
    if (batch == 0) return cudaSuccess;
    if (key_shift && !key_s) return cudaErrorInvalidValue;
    // two ciphertexts per work item; one at a level, where two spill (the key-row map's registers, DESIGN.md §4.18)
    u32 nseg;
    const unsigned grid = gather_grid(lc, (key_shift ? batch : (batch + 1) / 2) * lc.L, nseg);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        if (!key_s) {
            cudaError_t e = launch_key_prepare_t<LOGN>(lc, key, lc.ks_key_s, G.dnum, st);
            if (e != cudaSuccess) return e;
            key_s = lc.ks_key_s;
        }
        RotApplyGArgs A;
        A.ct = ct; A.U = U; A.key = key; A.key_s = key_s; A.acc = acc; A.galois = galois;
        if (key_shift) rot_apply_grouped_level_kernel<LOGN, 256, 3, 1><<<grid, 256, 0, st>>>(A, lc.lt, K, G, batch, nseg, key_shift);
        else rot_apply_grouped_kernel<LOGN, 256, 3, 2><<<grid, 256, 0, st>>>(A, lc.lt, K, G, batch, nseg);
        return cudaGetLastError();
    });
}

// summed rotations: acc [batch][2][L][N] of n_rot (1 .. ROT_SUM_MAX) rotations with their keys' Shoup companions key_s[m]
// key_shift > 0: a level view reading top-level keys (rot_sum_grouped_level_kernel, DESIGN.md §4.17)
cudaError_t launch_rot_sum_grouped(const LaunchCtx &lc, const u64 *ct, const u64 *U, u32 n_rot, const u64 *const *keys, const u64 *const *key_s,
                                   const u32 *galois, u64 *acc, const MsConsts &K, const GroupConsts &G, size_t batch, cudaStream_t st, u32 key_shift) {
    if (batch == 0) return cudaSuccess;
    if (n_rot < 1 || n_rot > (u32)ROT_SUM_MAX || G.Lq + G.K != lc.L) return cudaErrorInvalidValue;
    RotSumGArgs A;
    memset(&A, 0, sizeof(A));
    A.ct = ct; A.U = U; A.acc = acc; A.n_rot = n_rot;
    for (u32 m = 0; m < n_rot; ++m) {
        A.key[m] = keys[m];
        A.key_s[m] = key_s[m];
        A.galois[m] = galois[m];
    }
    // one ciphertext per work item: with two (the rot_apply_grouped split) the 80 registers of three CTAs per SM spill
    u32 nseg;
    const unsigned grid = gather_grid(lc, batch * lc.L, nseg);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        if (key_shift) rot_sum_grouped_level_kernel<LOGN, 256, 3, 1><<<grid, 256, 0, st>>>(A, lc.lt, K, G, batch, nseg, key_shift);
        else rot_sum_grouped_kernel<LOGN, 256, 3, 1><<<grid, 256, 0, st>>>(A, lc.lt, K, G, batch, nseg);
        return cudaGetLastError();
    });
}

#endif
#if DPFHE_PART_MAIN
// per-rotation constants: Shoup companions of the key (lc.ks_key_s), M = NTT(negmask_g) (in `M`, [L][N]) and kprime [2][L][N]
cudaError_t launch_rot_prepare(LaunchCtx &lc, const u64 *key, u32 galois, const u64 *delta, u64 *M, u64 *kprime, cudaStream_t st, u64 *key_s_out) {
    u64 *key_s = key_s_out ? key_s_out : lc.ks_key_s;   // a caller that keeps the constants of a rotation supplies its own buffer
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        cudaError_t e = launch_key_prepare_t<LOGN>(lc, key, key_s, lc.L, st);
        if (e != cudaSuccess) return e;
        negmask_kernel<LOGN><<<(1u << LOGN) / 256, 256, 0, st>>>(M, galois, lc.L);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        e = launch_ntt(lc, M, 1, false, st);
        if (e != cudaSuccess) return e;
        kprime_kernel<LOGN><<<ew_grid(lc, (size_t)2 * lc.L << LOGN), 256, 0, st>>>(key, M, delta, kprime, lc.lp, lc.L);
        return cudaGetLastError();
    });
}

// hoisted rotations, step 2: one rotation of `batch` ciphertexts from the shared transforms (constants from launch_rot_prepare)
cudaError_t launch_rot_apply(const LaunchCtx &lc, const u64 *ct, const u64 *U, const u64 *key, const u64 *kprime, u32 galois, u64 *out,
                             size_t batch, cudaStream_t st, const u64 *key_s) {
    if (batch == 0) return cudaSuccess;
    RotApplyArgs A;
    A.ct = ct; A.U = U; A.key = key; A.key_s = key_s ? key_s : lc.ks_key_s; A.kprime = kprime; A.out = out; A.L = lc.L; A.galois = galois;
    // tuning variant (DPFHE_ROT_CFG): 0 (default) = two ciphertexts share each key chunk, next digit prefetched;
    // 1 = one ciphertext per item, prefetched; 2 = one ciphertext, no prefetch.
    const int cfg = lc.rot_cfg;
    const size_t cb = cfg == 0 ? 2 : 1;
    u32 nseg;
    const unsigned grid = gather_grid(lc, ((batch + cb - 1) / cb) * lc.L, nseg);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        constexpr int LOGN = decltype(lg)::value;
        if (cfg == 1) rot_apply_kernel<LOGN, 256, 3, 1, true><<<grid, 256, 0, st>>>(A, lc.lt, batch, nseg);
        else if (cfg == 2) rot_apply_kernel<LOGN, 256, 3, 1, false><<<grid, 256, 0, st>>>(A, lc.lt, batch, nseg);
        else rot_apply_kernel<LOGN, 256, 3, 2, true><<<grid, 256, 0, st>>>(A, lc.lt, batch, nseg);
        return cudaGetLastError();
    });
}

cudaError_t launch_pointwise_mul(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *out, size_t n_polys, cudaStream_t st) {
    const size_t n_chunks = n_polys * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!n_chunks) return cudaSuccess;
    auto A = reinterpret_cast<const U64x2 *>(a), B = reinterpret_cast<const U64x2 *>(b);
    auto O = reinterpret_cast<U64x2 *>(out);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        pointwise_mul_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(A, B, O, lc.lp, lc.L, n_chunks);
        return cudaGetLastError();
    });
}

cudaError_t launch_poly_add(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *out, size_t n_polys, cudaStream_t st) {
    const size_t n_chunks = n_polys * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!n_chunks) return cudaSuccess;
    auto A = reinterpret_cast<const U64x2 *>(a), B = reinterpret_cast<const U64x2 *>(b);
    auto O = reinterpret_cast<U64x2 *>(out);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        poly_add_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(A, B, O, lc.lp, lc.L, n_chunks);
        return cudaGetLastError();
    });
}

cudaError_t launch_ct_mul_plain(const LaunchCtx &lc, const u64 *ct, const u64 *pt, u64 *out, size_t batch, cudaStream_t st) {
    const size_t n_chunks = batch * 2 * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!n_chunks) return cudaSuccess;
    auto A = reinterpret_cast<const U64x2 *>(ct), B = reinterpret_cast<const U64x2 *>(pt);
    auto O = reinterpret_cast<U64x2 *>(out);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        ct_mul_plain_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(A, B, O, lc.lp, lc.L, n_chunks);
        return cudaGetLastError();
    });
}

cudaError_t launch_ct_mul_plain_acc(const LaunchCtx &lc, const u64 *ct, const u64 *pt, u64 *acc, size_t batch, cudaStream_t st) {
    const size_t n_chunks = batch * 2 * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!n_chunks) return cudaSuccess;
    auto A = reinterpret_cast<const U64x2 *>(ct), B = reinterpret_cast<const U64x2 *>(pt);
    auto O = reinterpret_cast<U64x2 *>(acc);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        ct_mul_plain_acc_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(A, B, O, lc.lp, lc.L, n_chunks);
        return cudaGetLastError();
    });
}

cudaError_t launch_ct_tensor(const LaunchCtx &lc, const u64 *a, const u64 *b, u64 *d, size_t batch, cudaStream_t st) {
    const size_t items = batch * lc.L * ((size_t)1 << (lc.log_n - 1));
    if (!items) return cudaSuccess;
    auto A = reinterpret_cast<const U64x2 *>(a), B = reinterpret_cast<const U64x2 *>(b);
    auto D = reinterpret_cast<U64x2 *>(d);
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        ct_tensor_kernel<decltype(lg)::value><<<ew_grid(lc, items), 256, 0, st>>>(A, B, D, lc.lp, lc.L, batch);
        return cudaGetLastError();
    });
}

cudaError_t launch_fill_uniform(const LaunchCtx &lc, u64 seed, u64 first_poly, u64 *data, size_t n_polys, cudaStream_t st) {
    const size_t P = (size_t)lc.L << lc.log_n;
    const size_t n_chunks = n_polys * P / 2;
    if (!n_chunks) return cudaSuccess;
    auto O = reinterpret_cast<U64x2 *>(data);
    const u64 first_elem = first_poly * P;
    return with_log_n(lc.log_n, cudaErrorInvalidValue, [&](auto lg) {
        fill_uniform_kernel<decltype(lg)::value><<<ew_grid(lc, n_chunks), 256, 0, st>>>(O, lc.lp, lc.L, seed, first_elem, n_chunks);
        return cudaGetLastError();
    });
}

#endif
}  // namespace DPFHE_VNS
}  // namespace dpfhe
