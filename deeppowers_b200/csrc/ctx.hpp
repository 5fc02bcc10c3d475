// ctx.hpp — the context object behind the C ABI (internal; shared by abi.cu and multi.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <initializer_list>
#include <memory>
#include <vector>

#include "host_params.hpp"
#include "launch.hpp"

constexpr int DPFHE_PIPE_DEPTH = 3;

struct dpfhe_ctx;

// A device buffer that grows on demand and is owned by one context (or by an object built on it).  reserve() replaces it by a
// larger one only after all of the context's earlier work has finished, since any earlier call may still use it; a failed
// allocation leaves it empty, so the next call retries.
class DeviceScratch {
public:
    DeviceScratch() = default;
    DeviceScratch(const DeviceScratch &) = delete;
    DeviceScratch &operator=(const DeviceScratch &) = delete;
    ~DeviceScratch() { release(); }
    int reserve(dpfhe_ctx *ctx, size_t bytes);   // abi.cu
    void release() {
        cudaFree(p_);
        p_ = nullptr;
        bytes_ = 0;
    }
    size_t bytes() const { return bytes_; }
    template <class T = dpfhe::u64>
    T *get() const { return static_cast<T *>(p_); }

private:
    void *p_ = nullptr;
    size_t bytes_ = 0;
};

// The key-switching basis of level l with K special primes (DESIGN.md §2.20, §4.17): {q_0 .. q_{l-1}, p_0 .. p_{K-1}}, its host
// parameters and device tables, and what a context over that basis would pick (arithmetic variant, lift_reduce).  No key: the level
// calls read the context's top-level keys in place.
struct KsLevel {
    unsigned K = 0, l = 0;
    dpfhe::HostParams hp;
    dpfhe::LimbParams *d_lp = nullptr;
    dpfhe::Twiddle *d_tw = nullptr, *d_itw = nullptr;
    dpfhe::LimbTable lt;
    bool lift_reduce = true, fast = false;
    size_t bytes = 0;   // of the device tables
    KsLevel() = default;
    KsLevel(const KsLevel &) = delete;
    KsLevel &operator=(const KsLevel &) = delete;
    ~KsLevel() {
        cudaFree(d_lp);
        cudaFree(d_tw);
        cudaFree(d_itw);
    }
};

struct dpfhe_ctx {
    dpfhe::HostParams hp;
    dpfhe::LaunchCtx lc;
    cudaStream_t stream = nullptr;          // the context's own stream (used when the caller passes NULL)
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    dpfhe::LimbParams *d_lp = nullptr;
    dpfhe::Twiddle *d_tw = nullptr, *d_itw = nullptr;
    size_t device_bytes = 0;
    size_t object_bytes = 0;                // device memory of the counted objects built on the context (polynomial evaluators, slot sums):
                                            //   level tables, keys, scratch; CountedScratch is its one writer
    uint64_t launches = 0;
    // Ordering between calls: every entry point may run on a different stream (the caller's, or the context's own when NULL
    // is passed), but they all share the context's scratch.  Each call makes its stream wait for the previous call's work
    // when that ran on another stream (cur / last_stream / ev_last, see pick() and note_launch() in abi.cu).
    cudaStream_t cur = nullptr, last_stream = nullptr;
    cudaEvent_t ev_last = nullptr;
    bool have_last = false;
    // scratch and tables allocated on first use, released by dpfhe_context_trim (see each_trimmed())
    DeviceScratch ms_tau;                   // dpfhe_mod_switch_down / dpfhe_mod_down_special: [n_polys][K][N]
    DeviceScratch hoist_U, hoist_zero;      // hoisted rotations: shared transforms U [chunk][L][L][N], zero flags [chunk] (u32)
    DeviceScratch hoistg;                   // hoisted rotations with grouped hybrid keys: lifted digits, accumulators and tau' rows of a chunk
    DeviceScratch ckks_tab;                 // CKKS slot encoding: twiddles, 2^e mod q and slot permutation in one allocation
    dpfhe::CkksTables ckks;
    DeviceScratch bgv_tab;                  // BGV slot encoding: the twiddles mod t and slot positions of the plaintext modulus bgv_t
    uint64_t bgv_t = 0;                     //   last used (0: none), rewritten when t changes
    dpfhe::BgvTables bgv;
    DeviceScratch enc_work;                 // both slot encoders (encode: [n_vec][N] coefficients; decode: [n_vec][L][N] inverse transforms)
    DeviceScratch compact_work;             // compact ciphertexts: the level-1 pairs of a compaction, the c1' s rows of a decryption
    DeviceScratch stage_in[DPFHE_PIPE_DEPTH], stage_out[DPFHE_PIPE_DEPTH], stage_key;   // staging of the host-buffer entry points
    // allocated on first use and kept: per-rotation constants of the hoisted rotations, M [L][N] and kprime [2][L][N], and the
    // table delta[j][i] = q_j mod q_i
    DeviceScratch hoist_M, hoist_kprime, hoist_delta;
    // the level bases of the level calls, built at the first call at (K, l), counted in device_bytes, released by dpfhe_context_trim
    std::vector<std::unique_ptr<KsLevel>> ks_levels;
    // the prefix bases {q_0 .. q_{l-1}} of the keyless level calls (DESIGN.md §2.22), by l < L, built at the first call at l: the
    // limb parameters only (no twiddles), from which each call builds its host constants.  Host memory; the device tables are the
    // context's own, read through level_view.
    std::vector<std::unique_ptr<dpfhe::HostParams>> prefix;
    cudaEvent_t ev_h2d[DPFHE_PIPE_DEPTH] = {}, ev_comp[DPFHE_PIPE_DEPTH] = {}, ev_d2h[DPFHE_PIPE_DEPTH] = {};
    size_t N() const { return (size_t)1 << hp.log_n; }
    size_t P() const { return N() * hp.L; }
    // calls f on each buffer that dpfhe_context_trim releases (Self: dpfhe_ctx or const dpfhe_ctx)
    template <class Self, class F>
    static void each_trimmed(Self &c, F f) {
        for (auto *s : {&c.ms_tau, &c.hoist_U, &c.hoist_zero, &c.hoistg, &c.ckks_tab, &c.bgv_tab, &c.enc_work, &c.compact_work, &c.stage_key}) f(*s);
        for (auto &s : c.stage_in) f(s);
        for (auto &s : c.stage_out) f(s);
    }
};

// The device memory of an object built on a context that dpfhe_context_device_bytes reports: a scratch that grows with the batch,
// and the object's fixed allocations (keys, tables), which it makes itself and declares with count_fixed().  Every change of
// ctx->object_bytes happens here, and the destructor takes back all that was counted, so an object can neither reserve without
// counting nor go away without uncounting.
class CountedScratch {
public:
    explicit CountedScratch(dpfhe_ctx *ctx) : ctx_(ctx) {}
    ~CountedScratch() { ctx_->object_bytes -= fixed_ + s_.bytes(); }
    void count_fixed(size_t bytes) {
        fixed_ += bytes;
        ctx_->object_bytes += bytes;
    }
    int reserve(size_t bytes) {
        ctx_->object_bytes -= s_.bytes();
        const int rc = s_.reserve(ctx_, bytes);   // a failed allocation leaves it empty
        ctx_->object_bytes += s_.bytes();
        return rc;
    }
    dpfhe::u64 *get() const { return s_.get(); }

private:
    dpfhe_ctx *ctx_;
    size_t fixed_ = 0;
    DeviceScratch s_;
};
