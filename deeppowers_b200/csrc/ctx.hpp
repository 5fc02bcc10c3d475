// ctx.hpp — the context object behind the C ABI (internal; shared by abi.cu and multi.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "host_params.hpp"
#include "launch.hpp"

constexpr int DPFHE_PIPE_DEPTH = 3;

struct dpfhe_ctx {
    dpfhe::HostParams hp;
    dpfhe::LaunchCtx lc;
    cudaStream_t stream = nullptr;          // the context's own stream (used when the caller passes NULL)
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    dpfhe::LimbParams *d_lp = nullptr;
    dpfhe::Twiddle *d_tw = nullptr, *d_itw = nullptr;
    size_t device_bytes = 0;
    size_t object_bytes = 0;                // device memory of the polynomial evaluators built on the context (keys, tables, scratch)
    uint64_t launches = 0;
    // Ordering between calls: every entry point may run on a different stream (the caller's, or the context's own when NULL
    // is passed), but they all share the context's scratch.  Each call makes its stream wait for the previous call's work
    // when that ran on another stream (cur / last_stream / ev_last, see pick() and note_launch() in abi.cu).
    cudaStream_t cur = nullptr, last_stream = nullptr;
    cudaEvent_t ev_last = nullptr;
    bool have_last = false;
    // staging for the host-buffer entry points (allocated on first use)
    dpfhe::u64 *ms_tau = nullptr;                   // scratch of dpfhe_mod_switch_down: [n_polys][N]
    size_t ms_tau_bytes = 0;
    // hoisted rotations (allocated on first use): shared transforms U [chunk][L][L][N], zero flags [chunk],
    // per-rotation constants M [L][N] and kprime [2][L][N], and the table delta[j][i] = q_j mod q_i
    dpfhe::u64 *hoist_U = nullptr, *hoist_M = nullptr, *hoist_kprime = nullptr, *hoist_delta = nullptr;
    dpfhe::u32 *hoist_zero = nullptr;
    size_t hoist_chunk = 0;                  // ciphertexts the current U / zero buffers hold
    dpfhe::u64 *hoistg_buf = nullptr;        // hoisted rotations with grouped hybrid keys: lifted digits, accumulators and tau' rows of a chunk
    size_t hoistg_bytes = 0;
    // CKKS slot encoding (allocated on first use): twiddles, slot permutation and 2^e mod q tables in one allocation
    void *ckks_tab = nullptr;
    size_t ckks_tab_bytes = 0;
    dpfhe::CkksTables ckks;
    // BGV slot encoding: the twiddles mod t and slot positions of the plaintext modulus bgv_t last used (0: none), in one
    // allocation, replaced when t changes
    void *bgv_tab = nullptr;
    size_t bgv_tab_bytes = 0;
    uint64_t bgv_t = 0;
    dpfhe::BgvTables bgv;
    // scratch rows of both slot encoders (encode: [n_vec][N] coefficients; decode: [n_vec][L][N] inverse transforms)
    void *enc_work = nullptr;
    size_t enc_work_bytes = 0;
    dpfhe::u64 *stage_in[DPFHE_PIPE_DEPTH] = {}, *stage_out[DPFHE_PIPE_DEPTH] = {}, *stage_key = nullptr;
    size_t stage_in_bytes = 0, stage_out_bytes = 0, stage_key_bytes = 0;
    cudaEvent_t ev_h2d[DPFHE_PIPE_DEPTH] = {}, ev_comp[DPFHE_PIPE_DEPTH] = {}, ev_d2h[DPFHE_PIPE_DEPTH] = {};
    size_t N() const { return (size_t)1 << hp.log_n; }
    size_t P() const { return N() * hp.L; }
};

