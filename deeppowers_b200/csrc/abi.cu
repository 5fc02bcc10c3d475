// abi.cu — the extern "C" boundary declared in include/dpfhe.h.
//
// Conventions follow the reference HAL (see the header's citations): cudaSetDevice at the top
// of every call, the context owns its tables/scratch and frees them in destroy, CUDA errors
// are reported with file:line (as hal::CUDADevice::check_cuda_error does) — but as a status
// code plus thread-local message, because exceptions cannot cross a C ABI.
#include <cuda_runtime.h>
#include <sys/random.h>

#include <algorithm>
#include <cerrno>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <string>
#include <vector>

#include "../../include/dpfhe.h"
#include "ctx.hpp"
#include "eval.cuh"
#include "keys.cuh"

using namespace dpfhe;

// sets the thread-local message of dpfhe_last_error() and returns `code` (shared with multi.cu / hostmem.cu: ctx.hpp)
int dpfhe_fail(int code, const char *fmt, ...);

namespace {

thread_local std::string g_err;

#define fail dpfhe_fail

#define CU_TRY(expr)                                                                                          \
    do {                                                                                                      \
        cudaError_t e_ = (expr);                                                                              \
        if (e_ != cudaSuccess)                                                                                \
            return fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: %s (%s)", __FILE__, __LINE__, cudaGetErrorString(e_), #expr); \
    } while (0)

constexpr int PIPE_DEPTH = DPFHE_PIPE_DEPTH;

// launcher of the context's arithmetic variant (launch.hpp): dpfhe::fast when every modulus is k * 2^32 + 1
#define VCALL(fn, lc, ...) ((lc).fast ? fast::fn((lc), __VA_ARGS__) : gen::fn((lc), __VA_ARGS__))

}  // namespace

namespace {

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

#define CHECK_PTR(p)                                                                          \
    do {                                                                                      \
        if (!(p)) return fail(DPFHE_ERR_INVALID, "null pointer: %s", #p);                     \
        if (!aligned16(p)) return fail(DPFHE_ERR_INVALID, "%s must be 16-byte aligned", #p);  \
    } while (0)

// byte ranges [a, a + na) and [b, b + nb) intersect (unified addressing: valid across devices too)
bool overlaps(const void *a, size_t na, const void *b, size_t nb) {
    if (!a || !b || !na || !nb) return false;
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a0 < b0 + nb && b0 < a0 + na;
}

// an element-wise output: it may BE the input (each thread reads its words, then writes them), but not overlap it at another offset
bool overlaps_shifted(const void *out, const void *in, size_t bytes) { return out != in && overlaps(out, bytes, in, bytes); }

int enter(const dpfhe_ctx *ctx) {
    if (!ctx) return fail(DPFHE_ERR_INVALID, "null context");
    CU_TRY(cudaSetDevice(ctx->lc.device));
    return DPFHE_OK;
}

// The stream of this call (NULL = the context's own).  If the previous call ran on a different stream, this one waits for it:
// all calls share the context's scratch (key companions, digit slots, tickets), so they must not overlap.
cudaStream_t pick(dpfhe_ctx *ctx, void *stream) {
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    if (ctx->have_last && ctx->last_stream != st) cudaStreamWaitEvent(st, ctx->ev_last, 0);
    ctx->cur = st;
    return st;
}
// counts `n` launches just issued on the stream chosen by pick() and marks the point later calls have to wait for
void note_launch(dpfhe_ctx *ctx, uint64_t n) {
    ctx->launches += n;
    if (ctx->cur && cudaEventRecord(ctx->ev_last, ctx->cur) == cudaSuccess) {
        ctx->last_stream = ctx->cur;
        ctx->have_last = true;
    }
}

}  // namespace

int DeviceScratch::reserve(dpfhe_ctx *ctx, size_t bytes) {
    if (bytes <= bytes_) return DPFHE_OK;
    if (p_) {
        const int rc = dpfhe_synchronize(ctx);
        if (rc) return rc;
        release();
    }
    void *p = nullptr;
    CU_TRY(cudaMalloc(&p, bytes));
    p_ = p;
    bytes_ = bytes;
    return DPFHE_OK;
}

namespace {

// A device-resident output of the pipeline (dpfhe_seeded.h's uploads): every item of the input is rows of `row_words` words, which
// are copied straight into the output's items (out_item_words each), one row every 2 * row_words words: the c0 / b rows of
// [..][2][L][N] items.  The chunk's compute then runs in place on its items of d, and nothing is staged or downloaded.
struct DeviceOut {
    u64 *d = nullptr;
    size_t row_words = 0;
};

// A device-resident input of the pipeline (dpfhe_compact.h's download): the chunk's compute reads its items of d in place, and nothing
// is uploaded.  The input is the caller's memory, so the first compute waits as DeviceOut's first copy does.
struct DeviceIn {
    const u64 *d = nullptr;
};

// Generic three-stage pipeline over `n_items` items split into chunks:
//   upload(chunk -> stage_in[slot]) on s_h2d, compute on ctx->stream, download(stage_out[slot]) on s_d2h.
// in_item_bytes / out_item_bytes are per item; h_in may be two arrays (a and b) laid out back to back in the stage.
// n_slices > 1: each input is n_slices arrays of n_items items, slice_stride words apart (the operands of an inner product,
// [n_terms][batch] ciphertexts); a chunk stages its items of every slice, [input][slice][chunk_items], slice after slice.
// dev.d: a device-resident output (DeviceOut): upload(chunk -> its items of dev.d) on s_h2d, compute in place on ctx->stream.
// dev_in.d: a device-resident input (DeviceIn): compute(its items of dev_in.d -> stage_out[slot]) on ctx->stream, then the download.
template <class Compute>
int run_pipeline_body(dpfhe_ctx *ctx, const u64 *h_in0, const u64 *h_in1, u64 *h_out, size_t n_items, size_t in_item_words,
                      size_t out_item_words, size_t chunk_items, Compute compute, size_t n_slices, size_t slice_stride, DeviceOut dev,
                      DeviceIn dev_in) {
    if (dev.d) {
        // the output is the caller's memory: the first copy waits for the context's previous call (whatever stream it ran on) and for
        // the work issued before this call on the legacy default stream, which the non-blocking s_h2d does not wait for by itself
        if (ctx->have_last) CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_last, 0));
        CU_TRY(cudaEventRecord(ctx->ev_h2d[0], cudaStreamLegacy));
        CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_h2d[0], 0));
        // each chunk's copy is recorded in its slot's event and waited on by the compute stream at once (a wait takes the event's
        // state when it is issued), so a slot's event can be recorded again for a later chunk; no staging buffer is used
        const size_t row = dev.row_words, rows_per_item = in_item_words / row;
        size_t k = 0;
        for (size_t first = 0; first < n_items; first += chunk_items, ++k) {
            const size_t cnt = n_items - first < chunk_items ? n_items - first : chunk_items;
            const int slot = (int)(k % PIPE_DEPTH);
            u64 *dout = dev.d + first * out_item_words;
            CU_TRY(cudaMemcpy2DAsync(dout, 2 * row * 8, h_in0 + first * in_item_words, row * 8, row * 8, cnt * rows_per_item,
                                     cudaMemcpyHostToDevice, ctx->s_h2d));
            CU_TRY(cudaEventRecord(ctx->ev_h2d[slot], ctx->s_h2d));
            CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[slot], 0));
            const int rc = compute(dout, nullptr, dout, cnt, ctx->stream);
            if (rc) return rc;
        }
        CU_TRY(cudaStreamSynchronize(ctx->stream));
        return DPFHE_OK;
    }
    const size_t n_in = (h_in1 ? 2 : 1) * n_slices;
    int rc = DPFHE_OK;
    for (int k = 0; k < PIPE_DEPTH && !rc && !dev_in.d; ++k) rc = ctx->stage_in[k].reserve(ctx, n_in * chunk_items * in_item_words * 8);
    for (int k = 0; k < PIPE_DEPTH && !rc; ++k) rc = ctx->stage_out[k].reserve(ctx, chunk_items * out_item_words * 8);
    if (rc) return rc;
    if (dev_in.d) {
        if (ctx->have_last) CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_last, 0));
        CU_TRY(cudaEventRecord(ctx->ev_h2d[0], cudaStreamLegacy));
        CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[0], 0));
    }
    size_t k = 0;
    for (size_t first = 0; first < n_items; first += chunk_items, ++k) {
        const size_t cnt = n_items - first < chunk_items ? n_items - first : chunk_items;
        const int slot = (int)(k % PIPE_DEPTH);
        u64 *din0 = nullptr, *din1 = nullptr, *dout = ctx->stage_out[slot].get();
        if (dev_in.d) {
            din0 = const_cast<u64 *>(dev_in.d) + first * in_item_words;   // read only
        } else {
            din0 = ctx->stage_in[slot].get();
            din1 = din0 + n_slices * chunk_items * in_item_words;
            if (k >= PIPE_DEPTH) CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_comp[slot], 0));   // stage_in[slot] free again
            for (size_t s = 0; s < n_slices; ++s) {
                const size_t src = s * slice_stride + first * in_item_words, dst = s * chunk_items * in_item_words;
                CU_TRY(cudaMemcpyAsync(din0 + dst, h_in0 + src, cnt * in_item_words * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
                if (h_in1) CU_TRY(cudaMemcpyAsync(din1 + dst, h_in1 + src, cnt * in_item_words * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
            }
            CU_TRY(cudaEventRecord(ctx->ev_h2d[slot], ctx->s_h2d));
            CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[slot], 0));
        }
        if (k >= PIPE_DEPTH) CU_TRY(cudaStreamWaitEvent(ctx->stream, ctx->ev_d2h[slot], 0));   // stage_out[slot] drained
        rc = compute(din0, din1, dout, cnt, ctx->stream);
        if (rc) return rc;
        CU_TRY(cudaEventRecord(ctx->ev_comp[slot], ctx->stream));
        CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_comp[slot], 0));
        CU_TRY(cudaMemcpyAsync(h_out + first * out_item_words, dout, cnt * out_item_words * 8, cudaMemcpyDeviceToHost, ctx->s_d2h));
        CU_TRY(cudaEventRecord(ctx->ev_d2h[slot], ctx->s_d2h));
    }
    CU_TRY(cudaStreamSynchronize(ctx->s_d2h));
    CU_TRY(cudaStreamSynchronize(ctx->stream));
    return DPFHE_OK;
}

// runs the pipeline; on failure the three streams are drained before returning, so that no copy is still reading or writing
// the caller's host buffers (or the staging slots) when the error is reported
template <class Compute>
int run_pipeline(dpfhe_ctx *ctx, const u64 *h_in0, const u64 *h_in1, u64 *h_out, size_t n_items, size_t in_item_words,
                 size_t out_item_words, size_t chunk_items, Compute compute, size_t n_slices = 1, size_t slice_stride = 0, DeviceOut dev = {},
                 DeviceIn dev_in = {}) {
    const int rc = run_pipeline_body(ctx, h_in0, h_in1, h_out, n_items, in_item_words, out_item_words, chunk_items, compute, n_slices, slice_stride,
                                     dev, dev_in);
    if (rc != DPFHE_OK) {
        const std::string why = g_err;   // the drains below must not replace the message of the failure
        cudaStreamSynchronize(ctx->s_h2d);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->s_d2h);
        cudaGetLastError();
        g_err = why;
    }
    return rc;
}

size_t pick_chunk(const dpfhe_ctx *ctx, size_t item_bytes, size_t n_items) {
    // ~64 MiB per staged operand keeps PCIe transfers long and the staging footprint small
    size_t c = ((size_t)64 << 20) / item_bytes;
    if (c < 1) c = 1;
    // keep at least one full wave of work items per launch where the batch allows it
    const size_t wave = (size_t)ctx->lc.num_sms;
    if (c < wave && n_items >= wave) c = wave;
    if (c > n_items) c = n_items;
    return c;
}

int upload_key(dpfhe_ctx *ctx, const uint64_t *h_key, size_t words) {
    int rc = ctx->stage_key.reserve(ctx, words * 8);
    if (rc) return rc;
    CU_TRY(cudaMemcpyAsync(ctx->stage_key.get(), h_key, words * 8, cudaMemcpyHostToDevice, pick(ctx, nullptr)));
    return DPFHE_OK;
}

int no_check() { return DPFHE_OK; }

// The host-buffer form of an entry point: the host pointers `ptrs` must not be null, then `check()` runs the call's remaining
// argument checks.  The operand every item shares (a key, a plaintext or a secret of `shared_words` words; none when
// shared_words is 0) is uploaded once into the key staging buffer, and the items are pipelined through `compute` in chunks.
// dev.d: the output is that device buffer instead of h_out (DeviceOut); dev_in.d: the input is that device buffer instead of h_in0
// (DeviceIn).
template <class Compute, class Check = int (*)()>
int host_call(dpfhe_ctx *ctx, std::initializer_list<const void *> ptrs, const uint64_t *h_shared, size_t shared_words, const u64 *h_in0,
              const u64 *h_in1, u64 *h_out, size_t n_items, size_t in_item_words, size_t out_item_words, Compute compute, Check check = no_check,
              DeviceOut dev = {}, DeviceIn dev_in = {}) {
    for (const void *p : ptrs)
        if (!p) return fail(DPFHE_ERR_INVALID, "null host pointer");
    int rc = check();
    if (rc) return rc;
    if (shared_words) {
        rc = upload_key(ctx, h_shared, shared_words);
        if (rc) return rc;
    }
    const size_t chunk = pick_chunk(ctx, std::max(in_item_words, out_item_words) * 8, n_items);
    return run_pipeline(ctx, h_in0, h_in1, h_out, n_items, in_item_words, out_item_words, chunk, compute, 1, 0, dev, dev_in);
}

int check_galois(const dpfhe_ctx *ctx, uint64_t galois) {
    if (!(galois & 1) || galois >= ((uint64_t)2 << ctx->hp.log_n)) return fail(DPFHE_ERR_INVALID, "galois element must be odd and < 2N");
    return DPFHE_OK;
}

// the elements and keys of n_rot hoisted rotations
int check_rotations(const dpfhe_ctx *ctx, size_t n_rot, const uint64_t *galois_elts, const uint64_t *const *d_gks) {
    for (size_t r = 0; r < n_rot; ++r) {
        const int rc = check_galois(ctx, galois_elts[r]);
        if (rc) return rc;
        if (!d_gks[r] || !aligned16(d_gks[r])) return fail(DPFHE_ERR_INVALID, "null or misaligned Galois key");
    }
    return DPFHE_OK;
}

// the output of n_rot rotations (out_bytes) against their Galois keys of key_bytes each, which the launches read throughout
int check_keys_apart(const void *out, size_t out_bytes, size_t n_rot, const uint64_t *const *d_gks, size_t key_bytes) {
    for (size_t r = 0; r < n_rot; ++r)
        if (overlaps(out, out_bytes, d_gks[r], key_bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap a Galois key (rotation %zu)", r);
    return DPFHE_OK;
}

// the plaintext modulus of a division by the last K limbs (`what` names them in the message)
int check_t_below_special(const dpfhe_ctx *ctx, unsigned K, uint64_t t_plain, const char *what = "the special prime") {
    for (unsigned k = 0; k < K; ++k)
        if (t_plain >= ctx->hp.limbs[ctx->hp.L - 1 - k].lp.q) return fail(DPFHE_ERR_INVALID, "plaintext modulus must be below %s", what);
    return DPFHE_OK;
}

// Ciphertexts per chunk of the hoisted rotations' scratch (`per_ct` bytes each): at most ~4 GiB at a time, or
// DPFHE_HOIST_CAP_MB (diagnostics / tests: smaller scratch, more chunks).
size_t hoist_chunk(size_t per_ct, size_t batch) {
    size_t cap = (size_t)4 << 30;
    if (const char *e = getenv("DPFHE_HOIST_CAP_MB")) {
        const long mb = atol(e);
        if (mb > 0) cap = (size_t)mb << 20;
    }
    return std::max<size_t>(1, std::min(cap / per_ct, batch));
}

// Chunks of the host forms of the linear layer and the polynomial evaluator: about a fifth of the batch, rounded to whole rounds
// of the persistent key-switch grid (3 CTAs per SM, L CTAs per ciphertext: with grouped keys L = Lq + K, every limb of the
// context).  A chunk that leaves the grid's last round mostly empty costs more than the transfers it hides; the first upload and
// the last download are the only transfers not overlapped with a neighbouring chunk's compute.  `rounds_env` names a variable
// that sets the rounds instead (tuning).  Not capped by the batch.
size_t grid_round_chunk(const dpfhe_ctx *ctx, size_t batch, const char *rounds_env) {
    const size_t groups = std::max<size_t>(1, (size_t)ctx->lc.num_sms * 3 / ctx->hp.L);
    size_t rounds = (batch / 5 + groups / 2) / groups;
    if (const char *e = rounds_env ? getenv(rounds_env) : nullptr) rounds = (size_t)atol(e);
    if (rounds < 1) rounds = 1;
    const size_t chunk = rounds * groups;
    return chunk > 512 ? std::max<size_t>(groups, 512 / groups * groups) : chunk;
}

// the same, unless the variable `items_env` gives the chunk in ciphertexts (tests: several chunks at a small batch)
size_t item_chunk(const dpfhe_ctx *ctx, size_t batch, const char *items_env) {
    if (const char *e = getenv(items_env)) return std::max<size_t>(1, (size_t)atol(e));
    return grid_round_chunk(ctx, batch, nullptr);
}

// The context's launch state restricted to its first l limbs.  That prefix is a basis of its own: the limb constants and twiddles
// are rows indexed by limb with the ciphertext moduli first, and nothing else in the launch state depends on L.  So a view costs
// no device memory, and driven on the stream of the call it keeps the calls' order.
LaunchCtx level_view(const dpfhe_ctx *ctx, unsigned l) {
    LaunchCtx lc = ctx->lc;
    lc.L = l;
    return lc;
}

// The host parameters of the prefix basis {q_0 .. q_{l-1}}: the context's own at l = L, else built once at the first call and kept on
// the context.  Only the limb parameters are copied; the twiddles are the context's rows, read through level_view.  nullptr: out of
// host memory.
const HostParams *prefix_params(dpfhe_ctx *ctx, unsigned l) {
    if (l == ctx->hp.L) return &ctx->hp;
    if (ctx->prefix.size() < ctx->hp.L) ctx->prefix.resize(ctx->hp.L);
    auto &p = ctx->prefix[l];
    if (!p) {
        p.reset(new (std::nothrow) HostParams());
        if (!p) return nullptr;
        p->log_n = ctx->hp.log_n;
        p->L = l;
        p->limbs.resize(l);
        for (unsigned i = 0; i < l; ++i) {
            p->limbs[i].lp = ctx->hp.limbs[i].lp;
            p->limbs[i].psi = ctx->hp.limbs[i].psi;
        }
    }
    return p.get();
}

// the level of a keyless level call (DESIGN.md §2.22): 1 <= level <= L
int check_prefix_level(const dpfhe_ctx *ctx, unsigned level) {
    if (level < 1 || level > ctx->hp.L) return fail(DPFHE_ERR_INVALID, "level %u is outside [1, %u], the context's limbs", level, ctx->hp.L);
    return DPFHE_OK;
}

// rc, the result of a call at `level`; a failure's message is made to name the level
int level_failure(unsigned level, int rc) {
    if (rc != DPFHE_OK && g_err.compare(0, 6, "level ") != 0) g_err = "level " + std::to_string(level) + ": " + g_err;
    return rc;
}

// A keyless level call: the context and the level checked, then call(), the body on the prefix of `level` limbs, whose failures
// name the level
template <class Call>
int prefix_call(dpfhe_ctx *ctx, unsigned level, Call call) {
    int rc = enter(ctx);
    if (!rc) rc = check_prefix_level(ctx, level);
    if (rc) return rc;
    return level_failure(level, call());
}

// n grouped keys [n][dnum][2][L][N] on the device, back to back, and their Shoup companions in a second allocation of the same
// layout; keys[k] / key_s[k] point at key k.  Copyable: whoever holds it calls release().
struct PreparedKeys {
    u64 *d_keys = nullptr, *d_key_s = nullptr;
    std::vector<const u64 *> keys, key_s;
    size_t bytes = 0;   // of both allocations
    void release() {
        cudaFree(d_keys);
        cudaFree(d_key_s);
        *this = PreparedKeys();
    }
};

// Allocates both arrays, has `upload(d_keys)` copy the keys up (all of them, or the rows a level keeps) and issues the companions'
// launches on `st` with the launch state `lc`, one per key; the caller waits for them.  On failure nothing stays allocated.
template <class Upload>
int prepare_keys(dpfhe_ctx *ctx, const LaunchCtx &lc, size_t n, size_t dnum, cudaStream_t st, const char *what, Upload upload, PreparedKeys &pk) {
    const size_t key_words = dnum * 2 * lc.L * ((size_t)1 << lc.log_n);
    cudaError_t e = cudaMalloc(&pk.d_keys, n * key_words * 8);
    if (e == cudaSuccess) e = cudaMalloc(&pk.d_key_s, n * key_words * 8);
    if (e == cudaSuccess) e = upload(pk.d_keys);
    for (size_t k = 0; k < n && e == cudaSuccess; ++k) {
        pk.keys.push_back(pk.d_keys + k * key_words);
        pk.key_s.push_back(pk.d_key_s + k * key_words);
        e = VCALL(launch_key_prepare, lc, pk.keys[k], pk.d_key_s + k * key_words, (u32)dnum, st);
        note_launch(ctx, 1);
    }
    if (e != cudaSuccess) {
        pk.release();
        return fail(DPFHE_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
    }
    pk.bytes = 2 * n * key_words * 8;
    return DPFHE_OK;
}

// ---- The lifecycle of a library object built on a context (DESIGN.md §4.14).  Obj provides: ctx; `what`, the message for a null
// handle; in_words() / out_words(), the words of a ciphertext in and out; reserve(batch), the scratch of an application;
// apply_on(d_ct, d_out, batch, stream), the launches; host_chunk(batch), the ciphertexts per chunk of the host form (capped by the
// batch here); and a destructor that frees its device memory.

template <class Obj>
int object_apply(Obj *obj, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    if (!obj) return fail(DPFHE_ERR_INVALID, "%s", Obj::what);
    int rc = enter(obj->ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (overlaps(d_out, batch * obj->out_words() * 8, d_ct, batch * obj->in_words() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = obj->reserve(batch);
    if (rc) return rc;
    return obj->apply_on(d_ct, d_out, batch, stream);
}

// host buffers: chunks of the batch pipelined through apply_on (upload / compute / download overlapped)
template <class Obj>
int object_apply_host(Obj *obj, const uint64_t *h_ct, uint64_t *h_out, size_t batch) {
    if (!obj) return fail(DPFHE_ERR_INVALID, "%s", Obj::what);
    int rc = enter(obj->ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    if (!h_ct || !h_out) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const size_t chunk = std::min(obj->host_chunk(batch), batch);
    rc = obj->reserve(chunk);
    if (rc) return rc;
    return run_pipeline(obj->ctx, h_ct, nullptr, h_out, batch, obj->in_words(), obj->out_words(), chunk,
                        [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int { return obj->apply_on(din, dout, cnt, st); });
}

// waits for the context's work, which may still use the object's buffers
template <class Obj>
void object_destroy(Obj *obj) {
    if (!obj) return;
    cudaSetDevice(obj->ctx->lc.device);
    dpfhe_synchronize(obj->ctx);
    delete obj;
}

// The end of a constructor (rc: the result of everything before): waits for the launches on `st` that prepared the object's
// constants and hands the object out, or deletes it and reports the failure.
template <class Obj>
int object_finish(Obj *obj, int rc, cudaStream_t st, const char *what, Obj **out) {
    if (rc == DPFHE_OK) {
        const cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = fail(DPFHE_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
    }
    if (rc != DPFHE_OK) {
        delete obj;   // cudaFree waits for the device
        return rc;
    }
    *out = obj;
    return DPFHE_OK;
}

// The device tables of a modulus basis: limb constants d_lp [L] (also copied into lt, for the kernels' parameter blocks) and the
// forward and inverse twiddles [L][N]; adds their size to `bytes`.  lift_reduce: the key-switch kernels reduce the lifted
// digits unless every modulus is below twice the smallest (or always, with DPFHE_LIFT_REDUCE set).
int upload_basis(const HostParams &hp, LimbParams *&d_lp, Twiddle *&d_tw, Twiddle *&d_itw, LimbTable &lt, bool &lift_reduce, size_t &bytes) {
    const size_t L = hp.L, N = (size_t)1 << hp.log_n;
    CU_TRY(cudaMalloc(&d_lp, L * sizeof(LimbParams)));
    CU_TRY(cudaMalloc(&d_tw, L * N * sizeof(Twiddle)));
    CU_TRY(cudaMalloc(&d_itw, L * N * sizeof(Twiddle)));
    bytes += L * sizeof(LimbParams) + 2 * L * N * sizeof(Twiddle);
    memset(&lt, 0, sizeof(lt));
    uint64_t qmin = ~0ull, qmax = 0;
    for (size_t l = 0; l < L; ++l) {
        lt.lp[l] = hp.limbs[l].lp;
        qmin = std::min(qmin, lt.lp[l].q);
        qmax = std::max(qmax, lt.lp[l].q);
        CU_TRY(cudaMemcpy(d_tw + l * N, hp.limbs[l].tw.data(), N * sizeof(Twiddle), cudaMemcpyHostToDevice));
        CU_TRY(cudaMemcpy(d_itw + l * N, hp.limbs[l].itw.data(), N * sizeof(Twiddle), cudaMemcpyHostToDevice));
    }
    CU_TRY(cudaMemcpy(d_lp, lt.lp, L * sizeof(LimbParams), cudaMemcpyHostToDevice));
    lift_reduce = !(qmax < 2 * qmin) || getenv("DPFHE_LIFT_REDUCE") != nullptr;
    return DPFHE_OK;
}

}  // namespace

int dpfhe_fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

extern "C" {

const char *dpfhe_last_error(void) { return g_err.c_str(); }
const char *dpfhe_version(void) { return "dpfhe 0.1 sm_90a"; }

int dpfhe_context_create(const dpfhe_params *p, int device_id, dpfhe_ctx **out) {
    if (!p || !out) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    int n_dev = 0;
    cudaError_t ce = cudaGetDeviceCount(&n_dev);
    if (ce != cudaSuccess || n_dev <= 0)
        return fail(DPFHE_ERR_CUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                    ce == cudaSuccess ? "device count is 0" : cudaGetErrorString(ce));
    if (device_id < 0 || device_id >= n_dev) return fail(DPFHE_ERR_INVALID, "device_id %d out of range [0,%d)", device_id, n_dev);
    dpfhe_ctx *ctx = new (std::nothrow) dpfhe_ctx();
    if (!ctx) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    std::string msg = build_host_params(p->log_n, p->n_limbs, p->moduli, ctx->hp);
    if (!msg.empty()) {
        delete ctx;
        return fail(DPFHE_ERR_INVALID, "%s", msg.c_str());
    }
    ctx->lc.device = device_id;
#define CTX_TRY(expr)                                                                                              \
    do {                                                                                                           \
        cudaError_t e_ = (expr);                                                                                   \
        if (e_ != cudaSuccess) {                                                                                   \
            int rc_ = fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: %s (%s)", __FILE__, __LINE__, cudaGetErrorString(e_), #expr); \
            dpfhe_context_destroy(ctx);                                                                            \
            return rc_;                                                                                            \
        }                                                                                                          \
    } while (0)
    CTX_TRY(cudaSetDevice(device_id));
    cudaDeviceProp prop;
    CTX_TRY(cudaGetDeviceProperties(&prop, device_id));
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 only
        dpfhe_context_destroy(ctx);
        return fail(DPFHE_ERR_INVALID, "device %d is sm_%d%d; this build targets sm_90a only", device_id, prop.major, prop.minor);
    }
    CTX_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    CTX_TRY(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
    CTX_TRY(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
    for (int k = 0; k < PIPE_DEPTH; ++k) {
        CTX_TRY(cudaEventCreateWithFlags(&ctx->ev_h2d[k], cudaEventDisableTiming));
        CTX_TRY(cudaEventCreateWithFlags(&ctx->ev_comp[k], cudaEventDisableTiming));
        CTX_TRY(cudaEventCreateWithFlags(&ctx->ev_d2h[k], cudaEventDisableTiming));
    }
    CTX_TRY(cudaEventCreateWithFlags(&ctx->ev_last, cudaEventDisableTiming));
    const size_t N = ctx->N(), L = ctx->hp.L;
    LaunchCtx &lc = ctx->lc;
    const int rc = upload_basis(ctx->hp, ctx->d_lp, ctx->d_tw, ctx->d_itw, lc.lt, lc.lift_reduce, ctx->device_bytes);
    if (rc) {
        dpfhe_context_destroy(ctx);
        return rc;
    }
    lc.num_sms = prop.multiProcessorCount;
    lc.log_n = ctx->hp.log_n;
    lc.L = ctx->hp.L;
    lc.fast = true;
    for (size_t l = 0; l < L; ++l) lc.fast = lc.fast && lc.lt.lp[l].nqh != 0;
    if (getenv("DPFHE_FORCE_GENERIC")) lc.fast = false;   // diagnostics: run fast-class moduli through the generic kernels
    lc.lp = ctx->d_lp;
    if (const char *env = getenv("DPFHE_NTT_CFG")) lc.ntt_cfg = atoi(env);
    if (const char *env = getenv("DPFHE_NTT_TMA")) lc.ntt_tma = atoi(env);
    if (const char *env = getenv("DPFHE_EPOCH_LIMIT")) lc.ks_epoch_limit = strtoull(env, nullptr, 10);
    if (const char *env = getenv("DPFHE_ROT_CFG")) lc.rot_cfg = atoi(env);
    if (const char *env = getenv("DPFHE_KS_OCC")) lc.ks_occ_cap = atoi(env);
    if (const char *env = getenv("DPFHE_KS_PF")) lc.ks_prefetch = atoi(env);
    lc.tw = ctx->d_tw;
    lc.itw = ctx->d_itw;
    // digit-exchange scratch for the fused key-switch kernel: one slot per resident CTA, two parities
    lc.ks_slots = (size_t)lc.num_sms * 4;
    // digit slots and, at N = 16384, accumulator rows: ONE allocation, so that a single L2 access-policy window can cover the
    // whole cross-phase working set of the fused kernel (launch_ks_t).  At N <= 8192 the accumulators live in shared memory.
    const size_t ks_parts = ctx->hp.log_n > 13 ? 2 : 1;
    CTX_TRY(cudaMalloc(&lc.ks_scratch, ks_parts * lc.ks_slots * 2 * N * 8));
    lc.ks_acc = ks_parts > 1 ? lc.ks_scratch + lc.ks_slots * 2 * N : nullptr;
    lc.ks_window_bytes = ks_parts * lc.ks_slots * 2 * N * 8;
    {
        int max_persist = 0, max_window = 0;
        cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, device_id);
        cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, device_id);
        lc.l2_persist_max = (size_t)(max_persist > 0 ? max_persist : 0);
        if ((size_t)max_window < lc.ks_window_bytes) lc.ks_window_bytes = (size_t)(max_window > 0 ? max_window : 0);
        if (const char *env = getenv("DPFHE_L2_PERSIST")) lc.l2_persist = atoi(env);
        if (lc.l2_persist && lc.l2_persist_max) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, lc.l2_persist_max);
    }
    CTX_TRY(cudaMalloc(&lc.ks_key_s, 2 * L * L * N * 8));
    ctx->device_bytes += 2 * L * L * N * 8;
    CTX_TRY(cudaMalloc(&lc.ks_flags, 2 * lc.ks_slots * sizeof(u32)));   // digit flags, then the "round finished" marks of ks_hoistg_kernel
    CTX_TRY(cudaMemset(lc.ks_flags, 0, 2 * lc.ks_slots * sizeof(u32)));
    CTX_TRY(cudaMalloc(&lc.ks_consumed, lc.ks_slots * sizeof(u32)));
    CTX_TRY(cudaMemset(lc.ks_consumed, 0, lc.ks_slots * sizeof(u32)));
    if (const char *env = getenv("DPFHE_KS_SINGLE")) lc.ks_single = atoi(env);
    CTX_TRY(cudaMalloc(&lc.ks_ticket, 64));
    CTX_TRY(cudaMalloc(&lc.ks_mail, lc.ks_slots * sizeof(u64)));
    CTX_TRY(cudaMemset(lc.ks_mail, 0, lc.ks_slots * sizeof(u64)));
    ctx->device_bytes += ks_parts * lc.ks_slots * 2 * N * 8 + lc.ks_slots * (2 * sizeof(u32) + sizeof(u64)) + 64;
    if (getenv("DPFHE_KS_PROF")) {   // diagnostics: per-phase cycle counters of the fused kernel
        CTX_TRY(cudaMalloc(&lc.ks_prof, lc.ks_slots * 16 * sizeof(unsigned long long)));
        ctx->device_bytes += lc.ks_slots * 16 * sizeof(unsigned long long);
        CTX_TRY(cudaMemset(lc.ks_prof, 0, lc.ks_slots * 16 * sizeof(unsigned long long)));
    }
    CTX_TRY(cudaDeviceSynchronize());
#undef CTX_TRY
    *out = ctx;
    return DPFHE_OK;
}

void dpfhe_context_destroy(dpfhe_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->lc.device);
    cudaDeviceSynchronize();
    cudaFree(ctx->d_lp);
    cudaFree(ctx->d_tw);
    cudaFree(ctx->d_itw);
    cudaFree(ctx->lc.ks_scratch);   // ks_acc is the second half of the same allocation
    cudaFree(ctx->lc.ks_acc_hyb);
    cudaFree(ctx->lc.ks_flags);
    cudaFree(ctx->lc.ks_consumed);
    cudaFree(ctx->lc.ks_key_s);
    cudaFree(ctx->lc.ks_ticket);
    cudaFree(ctx->lc.ks_mail);
    cudaFree(ctx->lc.ks_prof);
    cudaFree(ctx->lc.ks_hyb);
    cudaFree(ctx->lc.ks_tau_drop);
    ctx->ks_levels.clear();
    for (int k = 0; k < PIPE_DEPTH; ++k) {
        if (ctx->ev_h2d[k]) cudaEventDestroy(ctx->ev_h2d[k]);
        if (ctx->ev_comp[k]) cudaEventDestroy(ctx->ev_comp[k]);
        if (ctx->ev_d2h[k]) cudaEventDestroy(ctx->ev_d2h[k]);
    }
    if (ctx->ev_last) cudaEventDestroy(ctx->ev_last);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
    delete ctx;   // frees the scratch
}

int dpfhe_get_modulus(const dpfhe_ctx *ctx, uint32_t limb, uint64_t *q) {
    if (!ctx || !q || limb >= ctx->hp.L) return fail(DPFHE_ERR_INVALID, "bad argument");
    *q = ctx->hp.limbs[limb].lp.q;
    return DPFHE_OK;
}
int dpfhe_get_psi(const dpfhe_ctx *ctx, uint32_t limb, uint64_t *psi) {
    if (!ctx || !psi || limb >= ctx->hp.L) return fail(DPFHE_ERR_INVALID, "bad argument");
    *psi = ctx->hp.limbs[limb].psi;
    return DPFHE_OK;
}
int dpfhe_get_root_powers(const dpfhe_ctx *ctx, uint32_t limb, int inverse, uint64_t *h_out) {
    if (!ctx || !h_out || limb >= ctx->hp.L) return fail(DPFHE_ERR_INVALID, "bad argument");
    const auto &v = inverse ? ctx->hp.limbs[limb].inv_root_powers : ctx->hp.limbs[limb].root_powers;
    memcpy(h_out, v.data(), v.size() * sizeof(uint64_t));
    return DPFHE_OK;
}
size_t dpfhe_context_device_bytes(const dpfhe_ctx *ctx) {
    if (!ctx) return 0;
    size_t n = ctx->device_bytes;   // tables, key companions, digit slots, accumulators, flags (+ hybrid rows)
    dpfhe_ctx::each_trimmed(*ctx, [&](const DeviceScratch &s) { n += s.bytes(); });
    n += ctx->hoist_M.bytes() + ctx->hoist_kprime.bytes() + ctx->hoist_delta.bytes();
    n += ctx->object_bytes;         // polynomial evaluators and slot sums: level tables, keys, scratch (CountedScratch)
    return n;
}

// frees the scratch that grows with use (hoisted-rotation transforms, modulus-switch rows, encoding tables, host staging, the level
// bases of the level calls); it comes back on demand
int dpfhe_context_trim(dpfhe_ctx *ctx) {
    int rc = enter(ctx);
    if (rc) return rc;
    rc = dpfhe_synchronize(ctx);
    if (rc) return rc;
    dpfhe_ctx::each_trimmed(*ctx, [](DeviceScratch &s) { s.release(); });
    for (const auto &v : ctx->ks_levels) ctx->device_bytes -= v->bytes;
    ctx->ks_levels.clear();   // the level bases come back at the next level call
    ctx->ckks = CkksTables();
    ctx->bgv_t = 0;
    ctx->bgv = BgvTables();
    return DPFHE_OK;
}
uint64_t dpfhe_launch_count(const dpfhe_ctx *ctx) { return ctx ? ctx->launches : 0; }

int dpfhe_ntt_fwd(dpfhe_ctx *ctx, uint64_t *d_data, size_t n_polys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_data);
    CU_TRY(VCALL(launch_ntt, ctx->lc, d_data, n_polys, false, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_ntt_inv(dpfhe_ctx *ctx, uint64_t *d_data, size_t n_polys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_data);
    CU_TRY(VCALL(launch_ntt, ctx->lc, d_data, n_polys, true, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

int dpfhe_poly_mul_pointwise(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out, size_t n_polys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_a); CHECK_PTR(d_b); CHECK_PTR(d_out);
    const size_t bytes = n_polys * ctx->P() * 8;
    if (overlaps_shifted(d_out, d_a, bytes) || overlaps_shifted(d_out, d_b, bytes))
        return fail(DPFHE_ERR_INVALID, "output must be an input or not overlap it");
    CU_TRY(VCALL(launch_pointwise_mul, ctx->lc, d_a, d_b, d_out, n_polys, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

int dpfhe_poly_add(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_out, size_t n_polys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_a); CHECK_PTR(d_b); CHECK_PTR(d_out);
    const size_t bytes = n_polys * ctx->P() * 8;
    if (overlaps_shifted(d_out, d_a, bytes) || overlaps_shifted(d_out, d_b, bytes))
        return fail(DPFHE_ERR_INVALID, "output must be an input or not overlap it");
    CU_TRY(VCALL(launch_poly_add, ctx->lc, d_a, d_b, d_out, n_polys, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

int dpfhe_ct_tensor(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, uint64_t *d_d, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_a); CHECK_PTR(d_b); CHECK_PTR(d_d);
    const size_t in_bytes = batch * 2 * ctx->P() * 8, out_bytes = batch * 3 * ctx->P() * 8;
    if (overlaps(d_d, out_bytes, d_a, in_bytes) || overlaps(d_d, out_bytes, d_b, in_bytes))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    CU_TRY(VCALL(launch_ct_tensor, ctx->lc, d_a, d_b, d_d, batch, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

static int ks_common(dpfhe_ctx *ctx, int mode, const uint64_t *a, const uint64_t *b, const uint64_t *key, uint64_t *out,
                     size_t batch, uint64_t galois, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(a); CHECK_PTR(key); CHECK_PTR(out);
    if (mode == KS_MUL_RELIN) CHECK_PTR(b);
    rc = mode == KS_ROTATE ? check_galois(ctx, galois) : DPFHE_OK;
    if (rc) return rc;
    {   // the output rows are written while other work items still read their inputs: no overlap at all, not only out == in;
        // every work item reads the key [L][2][L][N]
        const size_t ct_bytes = 2 * ctx->P() * 8, in_bytes = batch * (mode == KS_PLAIN ? ct_bytes / 2 : ct_bytes);
        if (overlaps(out, batch * ct_bytes, a, in_bytes) || overlaps(out, batch * ct_bytes, b, in_bytes))
            return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
        if (overlaps(out, batch * ct_bytes, key, ctx->hp.L * ct_bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap the key");
    }
    CU_TRY(VCALL(launch_ks, ctx->lc, mode, a, b, key, out, batch, (u32)galois, pick(ctx, stream)));
    note_launch(ctx, 2);   // key_prepare_kernel + ks_fused_kernel
    return DPFHE_OK;
}

int dpfhe_keyswitch(dpfhe_ctx *ctx, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out, size_t batch, void *stream) {
    return ks_common(ctx, KS_PLAIN, d_d, nullptr, d_key, d_out, batch, 0, stream);
}
int dpfhe_ct_mul_relin(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk, uint64_t *d_out,
                       size_t batch, void *stream) {
    return ks_common(ctx, KS_MUL_RELIN, d_a, d_b, d_evk, d_out, batch, 0, stream);
}
int dpfhe_rotate(dpfhe_ctx *ctx, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk, uint64_t *d_out, size_t batch,
                 void *stream) {
    return ks_common(ctx, KS_ROTATE, d_ct, nullptr, d_gk, d_out, batch, galois_elt, stream);
}

// hybrid (special-prime) variants: the context's last limb is the special prime, data carries L-1 limbs
// n_special = K: the last K limbs are special primes and the digits are groups of K limbs (DESIGN.md §2.11); K = 1 is §2.10
static int check_special(const dpfhe_ctx *ctx, unsigned n_special) {
    const unsigned L = ctx->hp.L;
    if (L < 2) return fail(DPFHE_ERR_INVALID, "hybrid key switching needs a special prime: create the context with at least two limbs");
    if (n_special < 1 || n_special > (unsigned)KS_MAX_SPECIAL || 2 * n_special > L)
        return fail(DPFHE_ERR_INVALID, "n_special must be between 1 and %d and at most half of the context's %u limbs", KS_MAX_SPECIAL, L);
    return DPFHE_OK;
}

// a call with grouped special-prime keys that ends in a division by the special primes with plaintext modulus t_plain
static int check_grouped(const dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain) {
    const int rc = check_special(ctx, n_special);
    return rc ? rc : check_t_below_special(ctx, n_special, t_plain);
}

// digits of a key: groups of n_special limbs of the L - n_special ciphertext moduli; n_special = 0: per-limb digits, L of them
static size_t key_digits(const dpfhe_ctx *ctx, unsigned n_special) {
    const unsigned L = ctx->hp.L;
    return n_special ? (L - n_special + n_special - 1) / n_special : L;
}

// bytes of one switch key [digits][2][L][N] of the context: what every work item of a key-switching launch reads
static size_t grouped_key_bytes(const dpfhe_ctx *ctx, unsigned n_special) { return key_digits(ctx, n_special) * 2 * ctx->P() * 8; }

// the special-prime accumulator and tau' rows of the hybrid / grouped key-switch kernels, allocated at the first call that needs them
static int ensure_hyb(dpfhe_ctx *ctx) {
    if (ctx->lc.ks_hyb) return DPFHE_OK;
    u64 *hyb = nullptr;
    const size_t hyb_bytes = (ctx->lc.ks_slots / 2 + 1) * KS_HYB_ROWS * ctx->N() * sizeof(u64), acc_bytes = ctx->lc.ks_slots * 4 * ctx->N() * sizeof(u64);
    CU_TRY(cudaMalloc(&hyb, hyb_bytes));
    ctx->lc.ks_hyb = hyb;
    CU_TRY(cudaMalloc(&ctx->lc.ks_acc_hyb, acc_bytes));
    ctx->device_bytes += hyb_bytes + acc_bytes;
    return DPFHE_OK;
}

static int ks_hybrid_common(dpfhe_ctx *ctx, unsigned n_special, int mode, const uint64_t *a, const uint64_t *b, const uint64_t *key,
                            uint64_t *out, size_t batch, uint64_t galois, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(a); CHECK_PTR(key); CHECK_PTR(out);
    if (mode == KS_MUL_RELIN) CHECK_PTR(b);
    const unsigned L = ctx->hp.L;
    rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    rc = mode == KS_ROTATE ? check_galois(ctx, galois) : DPFHE_OK;
    if (rc) return rc;
    {
        const size_t ct_bytes = 2 * (size_t)(L - n_special) * ctx->N() * 8, in_bytes = batch * (mode == KS_PLAIN ? ct_bytes / 2 : ct_bytes);
        if (overlaps(out, batch * ct_bytes, a, in_bytes) || overlaps(out, batch * ct_bytes, b, in_bytes))
            return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
        if (overlaps(out, batch * ct_bytes, key, grouped_key_bytes(ctx, n_special))) return fail(DPFHE_ERR_INVALID, "output must not overlap the key");
    }
    rc = ensure_hyb(ctx);
    if (rc) return rc;
    MsConsts K;
    if (n_special == 1) {
        build_ms_consts(ctx->hp, t_plain, K);
        CU_TRY(VCALL(launch_ks_hybrid, ctx->lc, mode, a, b, key, out, batch, (u32)galois, K, pick(ctx, stream)));
    } else {
        GroupConsts G;
        build_group_consts(ctx->hp, n_special, t_plain, G, K);
        CU_TRY(VCALL(launch_ks_grouped, ctx->lc, mode, a, b, key, out, batch, (u32)galois, K, G, pick(ctx, stream)));
    }
    note_launch(ctx, 2);   // key_prepare_kernel + ks_hybrid_kernel / ks_grouped_kernel
    return DPFHE_OK;
}
int dpfhe_keyswitch_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out, size_t batch,
                            uint64_t t_plain, void *stream) {
    return ks_hybrid_common(ctx, n_special, KS_PLAIN, d_d, nullptr, d_key, d_out, batch, 0, t_plain, stream);
}
int dpfhe_ct_mul_relin_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk,
                               uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return ks_hybrid_common(ctx, n_special, KS_MUL_RELIN, d_a, d_b, d_evk, d_out, batch, 0, t_plain, stream);
}
int dpfhe_rotate_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk, uint64_t *d_out,
                         size_t batch, uint64_t t_plain, void *stream) {
    return ks_hybrid_common(ctx, n_special, KS_ROTATE, d_ct, nullptr, d_gk, d_out, batch, galois_elt, t_plain, stream);
}
// The argument checks of a call on n_terms operand pairs (d_as[i], d_bs[i]) [batch][2][Lq][N] with grouped keys, in this order: the
// pair table, the key and output pointers, check() (the call's own checks of n_special and t_plain), then, for a non-empty batch, the
// output [batch][2][Lq - drop][N] against every operand: the output rows are written while other work items still read their inputs,
// so no overlap at all.  An empty batch passes once the checks before the overlap have.  level: the operands' limbs of a level call
// (DESIGN.md §2.20), 0 for the top level Lq = L - n_special.
extern "C++" {   // a template inside the C entry points' linkage block
template <class Check>
static int check_pairs(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                       const uint64_t *d_evk, uint64_t *d_out, size_t batch, unsigned drop, Check check, unsigned level = 0) {
    if (n_terms < 1 || n_terms > (size_t)DOT_MAX_TERMS) return fail(DPFHE_ERR_INVALID, "n_terms must be in [1, %d]", DOT_MAX_TERMS);
    if (!d_as || !d_bs) return fail(DPFHE_ERR_INVALID, "null argument");
    for (size_t i = 0; i < n_terms; ++i)
        if (!d_as[i] || !d_bs[i] || !aligned16(d_as[i]) || !aligned16(d_bs[i])) return fail(DPFHE_ERR_INVALID, "null or misaligned operand of pair %zu", i);
    CHECK_PTR(d_evk); CHECK_PTR(d_out);
    const int rc = check();
    if (rc || batch == 0) return rc;
    const size_t Lq = level ? level : ctx->hp.L - n_special, in_bytes = batch * 2 * Lq * ctx->N() * 8, out_bytes = batch * 2 * (Lq - drop) * ctx->N() * 8;
    for (size_t i = 0; i < n_terms; ++i)
        if (overlaps(d_out, out_bytes, d_as[i], in_bytes) || overlaps(d_out, out_bytes, d_bs[i], in_bytes))
            return fail(DPFHE_ERR_INVALID, "output must not overlap an operand (pair %zu)", i);
    if (overlaps(d_out, out_bytes, d_evk, grouped_key_bytes(ctx, n_special))) return fail(DPFHE_ERR_INVALID, "output must not overlap the key");
    return DPFHE_OK;
}
}

// Encrypted inner product (DESIGN.md §2.18): the tensor products of n_terms pairs summed before one relinearisation.  Every
// n_special runs the grouped kernel (with one special prime its digits are single limbs and it computes what the hybrid kernel does).
int dpfhe_ct_dot_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                         const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    rc = check_pairs(ctx, n_special, n_terms, d_as, d_bs, d_evk, d_out, batch, 0, [&] { return check_grouped(ctx, n_special, t_plain); });
    if (rc || batch == 0) return rc;
    rc = ensure_hyb(ctx);
    if (rc) return rc;
    MsConsts K;
    GroupConsts G;
    build_group_consts(ctx->hp, n_special, t_plain, G, K);
    CU_TRY(VCALL(launch_ct_dot_grouped, ctx->lc, d_as, d_bs, (u32)n_terms, d_evk, d_out, batch, K, G, pick(ctx, stream)));
    note_launch(ctx, 2);   // key_prepare_kernel + ct_dot_grouped_kernel
    return DPFHE_OK;
}

// the dropped limb's y_qbar rows of multiply-and-rescale (DESIGN.md §4.16), allocated at the first such call: one block of
// [2 parities][2][N] per group of the grid, whose groups have L >= 3 CTAs
static int ensure_tau_drop(dpfhe_ctx *ctx) {
    if (ctx->lc.ks_tau_drop) return DPFHE_OK;
    u64 *rows = nullptr;
    const size_t bytes = (ctx->lc.ks_slots / 3 + 1) * 4 * ctx->N() * sizeof(u64);
    CU_TRY(cudaMalloc(&rows, bytes));
    ctx->lc.ks_tau_drop = rows;
    ctx->device_bytes += bytes;
    return DPFHE_OK;
}

// the checks of a multiply-and-rescale call beyond its operands: those of the grouped product, at least two ciphertext limbs (one
// is kept) and t_plain below the dropped modulus as well as the special primes
static int check_rescale(const dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain) {
    int rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    if (ctx->hp.L - n_special < 2)
        return fail(DPFHE_ERR_INVALID, "multiply-and-rescale needs at least two ciphertext limbs: the context has %u limbs, %u of them special",
                    ctx->hp.L, n_special);
    return check_t_below_special(ctx, n_special + 1, t_plain, "the special primes and the dropped modulus");
}

// Multiply-and-rescale (DESIGN.md §2.19): dot = false is the ct x ct product of d_as[0] and d_bs[0] (n_terms = 1), dot = true the
// inner product of n_terms pairs; relinearised and divided by P * q_{Lq-1} in one kernel.  out: [batch][2][Lq-1][N].
static int rescale_common(dpfhe_ctx *ctx, unsigned n_special, bool dot, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                          const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    rc = check_pairs(ctx, n_special, n_terms, d_as, d_bs, d_evk, d_out, batch, 1, [&] { return check_rescale(ctx, n_special, t_plain); });
    if (rc || batch == 0) return rc;
    rc = ensure_hyb(ctx);
    if (rc) return rc;
    rc = ensure_tau_drop(ctx);
    if (rc) return rc;
    MsConsts K;
    GroupConsts G;
    RescaleConsts R;
    build_rescale_consts(ctx->hp, n_special, t_plain, G, K, R);
    CU_TRY(VCALL(launch_ks_rescale_grouped, ctx->lc, dot, d_as, d_bs, (u32)n_terms, d_evk, d_out, batch, K, G, R, pick(ctx, stream)));
    note_launch(ctx, 2);   // key_prepare_kernel + ks_rescale_grouped_kernel
    return DPFHE_OK;
}
int dpfhe_ct_mul_relin_rescale_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk,
                                       uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return rescale_common(ctx, n_special, false, 1, &d_a, &d_b, d_evk, d_out, batch, t_plain, stream);
}
int dpfhe_ct_dot_rescale_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *const *d_as, const uint64_t *const *d_bs,
                                 const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return rescale_common(ctx, n_special, true, n_terms, d_as, d_bs, d_evk, d_out, batch, t_plain, stream);
}

// ---- calls at level l on the top-level context (DESIGN.md §2.20, §4.17) ----------------------------------------------------------
// A level-l call is the same call on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the top-level key restricted to the level's
// digits and rows.  It runs on the level's view of this context: the level's own tables (KsLevel, built at the first call at (K, l)),
// the context's scratch and round numbering, and the top-level key read in place through the kernels' key-row map.

// the checks of a level call beyond those of the unrescaled top-level call (check_grouped), after them: K <= l <= Lq; with the
// rescale also l >= 2 and t_plain below q_{l-1}
static int check_level(const dpfhe_ctx *ctx, unsigned K, unsigned level, bool rescale, uint64_t t_plain) {
    const unsigned Lq = ctx->hp.L - K;
    if (level < K || level > Lq)
        return fail(DPFHE_ERR_INVALID, "level %u is outside [%u, %u]: a level call needs at least n_special = %u ciphertext limbs and at most the "
                    "context's %u", level, K, Lq, K, Lq);
    if (!rescale) return DPFHE_OK;
    if (level < 2) return fail(DPFHE_ERR_INVALID, "level %u: multiply-and-rescale needs at least two ciphertext limbs", level);
    if (t_plain >= ctx->hp.limbs[level - 1].lp.q)
        return fail(DPFHE_ERR_INVALID, "level %u: plaintext modulus must be below the dropped modulus q_%u", level, level - 1);
    return DPFHE_OK;
}

// the level state of (K, l), l < Lq: found, or built and uploaded (its bytes counted in device_bytes until dpfhe_context_trim)
static int level_state(dpfhe_ctx *ctx, unsigned K, unsigned l, const KsLevel *&out) {
    for (const auto &v : ctx->ks_levels)
        if (v->K == K && v->l == l) {
            out = v.get();
            return DPFHE_OK;
        }
    std::unique_ptr<KsLevel> v(new (std::nothrow) KsLevel());
    if (!v) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    v->K = K;
    v->l = l;
    const unsigned Lq = ctx->hp.L - K;
    std::vector<uint64_t> mod(l + K);
    for (unsigned i = 0; i < l; ++i) mod[i] = ctx->hp.limbs[i].lp.q;
    for (unsigned k = 0; k < K; ++k) mod[l + k] = ctx->hp.limbs[Lq + k].lp.q;
    const std::string msg = build_host_params(ctx->hp.log_n, l + K, mod.data(), v->hp);
    if (!msg.empty()) return fail(DPFHE_ERR_INVALID, "level %u: %s", l, msg.c_str());
    const int rc = upload_basis(v->hp, v->d_lp, v->d_tw, v->d_itw, v->lt, v->lift_reduce, v->bytes);
    if (rc) return rc;   // the destructor frees what was allocated
    // the arithmetic variant a context over this basis picks (dpfhe_context_create)
    v->fast = getenv("DPFHE_FORCE_GENERIC") == nullptr;
    for (unsigned i = 0; i < l + K; ++i) v->fast = v->fast && v->lt.lp[i].nqh != 0;
    ctx->device_bytes += v->bytes;
    out = v.get();
    ctx->ks_levels.push_back(std::move(v));
    return DPFHE_OK;
}

// the launch state of a level: the context's, with the level's basis and tables
static LaunchCtx level_ks_view(const dpfhe_ctx *ctx, const KsLevel &v) {
    LaunchCtx lc = ctx->lc;
    lc.L = v.l + v.K;
    lc.lp = v.d_lp;
    lc.lt = v.lt;
    lc.tw = v.d_tw;
    lc.itw = v.d_itw;
    lc.lift_reduce = v.lift_reduce;
    lc.fast = v.fast;
    return lc;
}

// runs launch(lc) on the level's view and carries the round numbering back to the context: the next key switch on any view continues
// from there
extern "C++" {   // a template inside the C entry points' linkage block
template <class Launch>
static cudaError_t on_level_view(dpfhe_ctx *ctx, const KsLevel &v, Launch launch) {
    LaunchCtx lc = level_ks_view(ctx, v);
    const cudaError_t e = launch(lc);
    ctx->lc.ks_epoch = lc.ks_epoch;
    ctx->lc.ks_epoch_restarts = lc.ks_epoch_restarts;
    return e;
}
}

// A key-switching call at level l < Lq once its arguments are checked: the level state, the top-level key's companions over the
// digits g < ceil(l / K) (the context's launch state, into lc.ks_key_s) and the kernel on the level's view.  mode KS_MUL_RELIN /
// KS_ROTATE (as[0], bs[0]; galois) or KS_DOT (n_terms pairs); rescale: divided by P * q_{l-1}.  K = 1 without the pairs and the
// rescale is the one-special-prime kernel, as at the top level.  Two launches.
static int level_launch(dpfhe_ctx *ctx, unsigned K, unsigned l, int mode, bool rescale, size_t n_terms, const uint64_t *const *as,
                        const uint64_t *const *bs, const uint64_t *key, uint64_t *out, size_t batch, uint64_t galois, uint64_t t_plain, void *stream) {
    const KsLevel *v = nullptr;
    int rc = level_state(ctx, K, l, v);
    if (!rc) rc = ensure_hyb(ctx);
    if (!rc && rescale) rc = ensure_tau_drop(ctx);
    if (rc) return rc;
    MsConsts Kc;
    GroupConsts G;
    RescaleConsts R;
    const bool hybrid = K == 1 && mode != KS_DOT && !rescale;
    if (hybrid) build_ms_consts(v->hp, t_plain, Kc);
    else if (rescale) build_rescale_consts(v->hp, K, t_plain, G, Kc, R);
    else build_group_consts(v->hp, K, t_plain, G, Kc);
    cudaStream_t st = pick(ctx, stream);
    CU_TRY(VCALL(launch_key_prepare, ctx->lc, key, ctx->lc.ks_key_s, (u32)((l + K - 1) / K), st));
    const u32 key_L = ctx->hp.L;
    CU_TRY(on_level_view(ctx, *v, [&](LaunchCtx &lc) {
        if (hybrid) return VCALL(launch_ks_hybrid, lc, mode, as[0], bs ? bs[0] : nullptr, key, out, batch, (u32)galois, Kc, st, lc.ks_key_s, key_L);
        return VCALL(launch_ks_grouped_level, lc, mode, as, bs, (u32)n_terms, key, lc.ks_key_s, key_L, out, batch, (u32)galois, Kc, G,
                     rescale ? &R : nullptr, st);
    }));
    note_launch(ctx, 2);   // key_prepare_kernel + the kernel
    return DPFHE_OK;
}

// ct x ct product and rotation at level l: ks_hybrid_common's checks, in its order, with the operands' sizes of the level
static int level_single(dpfhe_ctx *ctx, unsigned n_special, unsigned level, int mode, const uint64_t *a, const uint64_t *b, const uint64_t *key,
                        uint64_t *out, size_t batch, uint64_t galois, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(a); CHECK_PTR(key); CHECK_PTR(out);
    if (mode == KS_MUL_RELIN) CHECK_PTR(b);
    rc = check_grouped(ctx, n_special, t_plain);
    if (!rc) rc = check_level(ctx, n_special, level, false, t_plain);
    if (!rc && mode == KS_ROTATE) rc = check_galois(ctx, galois);
    if (rc) return rc;
    if (level == ctx->hp.L - n_special) return ks_hybrid_common(ctx, n_special, mode, a, b, key, out, batch, galois, t_plain, stream);
    const size_t ct_bytes = 2 * (size_t)level * ctx->N() * 8;
    if (overlaps(out, batch * ct_bytes, a, batch * ct_bytes) || overlaps(out, batch * ct_bytes, b, batch * ct_bytes))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    if (overlaps(out, batch * ct_bytes, key, grouped_key_bytes(ctx, n_special))) return fail(DPFHE_ERR_INVALID, "output must not overlap the key");
    return level_launch(ctx, n_special, level, mode, false, 1, &a, &b, key, out, batch, galois, t_plain, stream);
}

// the calls on operand pairs at level l: check_pairs with the level's checks and sizes, then the top-level call at l = Lq
static int level_pairs(dpfhe_ctx *ctx, unsigned n_special, unsigned level, bool rescale, bool dot, size_t n_terms, const uint64_t *const *d_as,
                       const uint64_t *const *d_bs, const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    rc = check_pairs(ctx, n_special, n_terms, d_as, d_bs, d_evk, d_out, batch, rescale ? 1 : 0, [&] {
        const int r = check_grouped(ctx, n_special, t_plain);
        return r ? r : check_level(ctx, n_special, level, rescale, t_plain);
    }, level);
    if (rc || batch == 0) return rc;
    if (level == ctx->hp.L - n_special) {
        if (rescale) return rescale_common(ctx, n_special, dot, n_terms, d_as, d_bs, d_evk, d_out, batch, t_plain, stream);
        if (dot) return dpfhe_ct_dot_grouped(ctx, n_special, n_terms, d_as, d_bs, d_evk, d_out, batch, t_plain, stream);
        return dpfhe_ct_mul_relin_grouped(ctx, n_special, d_as[0], d_bs[0], d_evk, d_out, batch, t_plain, stream);
    }
    return level_launch(ctx, n_special, level, dot ? KS_DOT : KS_MUL_RELIN, rescale, n_terms, d_as, d_bs, d_evk, d_out, batch, 0, t_plain, stream);
}

int dpfhe_ct_mul_relin_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_a, const uint64_t *d_b,
                                     const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return level_single(ctx, n_special, level, KS_MUL_RELIN, d_a, d_b, d_evk, d_out, batch, 0, t_plain, stream);
}
int dpfhe_rotate_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk,
                               uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return level_single(ctx, n_special, level, KS_ROTATE, d_ct, nullptr, d_gk, d_out, batch, galois_elt, t_plain, stream);
}
int dpfhe_ct_dot_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *const *d_as,
                               const uint64_t *const *d_bs, const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return level_pairs(ctx, n_special, level, false, true, n_terms, d_as, d_bs, d_evk, d_out, batch, t_plain, stream);
}
int dpfhe_ct_mul_relin_rescale_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_a, const uint64_t *d_b,
                                             const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return level_pairs(ctx, n_special, level, true, false, 1, &d_a, &d_b, d_evk, d_out, batch, t_plain, stream);
}
int dpfhe_ct_dot_rescale_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *const *d_as,
                                       const uint64_t *const *d_bs, const uint64_t *d_evk, uint64_t *d_out, size_t batch, uint64_t t_plain,
                                       void *stream) {
    return level_pairs(ctx, n_special, level, true, true, n_terms, d_as, d_bs, d_evk, d_out, batch, t_plain, stream);
}

int dpfhe_grouped_digits(const dpfhe_ctx *ctx, unsigned n_special, unsigned *digits) {
    if (!ctx || !digits) return fail(DPFHE_ERR_INVALID, "null argument");
    int rc = check_special(ctx, n_special);
    if (rc) return rc;
    *digits = (unsigned)key_digits(ctx, n_special);
    return DPFHE_OK;
}
int dpfhe_keyswitch_hybrid(dpfhe_ctx *ctx, const uint64_t *d_d, const uint64_t *d_key, uint64_t *d_out, size_t batch, uint64_t t_plain,
                           void *stream) {
    return dpfhe_keyswitch_grouped(ctx, 1, d_d, d_key, d_out, batch, t_plain, stream);
}
int dpfhe_ct_mul_relin_hybrid(dpfhe_ctx *ctx, const uint64_t *d_a, const uint64_t *d_b, const uint64_t *d_evk, uint64_t *d_out,
                              size_t batch, uint64_t t_plain, void *stream) {
    return dpfhe_ct_mul_relin_grouped(ctx, 1, d_a, d_b, d_evk, d_out, batch, t_plain, stream);
}
int dpfhe_rotate_hybrid(dpfhe_ctx *ctx, const uint64_t *d_ct, uint64_t galois_elt, const uint64_t *d_gk, uint64_t *d_out, size_t batch,
                        uint64_t t_plain, void *stream) {
    return dpfhe_rotate_grouped(ctx, 1, d_ct, galois_elt, d_gk, d_out, batch, t_plain, stream);
}

// Hoisted rotations: n_rot rotations of the SAME ciphertexts.  Bit-identical to n_rot calls of dpfhe_rotate; the digit
// decomposition and its L(L-1) forward transforms are done once per ciphertext (kernels.cu: ks_hoist_kernel), each
// rotation is then gathers + multiply-accumulates (rot_apply_kernel).  Ciphertexts whose digit has a zero coefficient
// (where the shared-transform identity does not hold) are recomputed by the ordinary rotate kernel.
// prepared: optional per-rotation constants kept by the caller (a linear layer applies the same rotations to every batch):
// for rotation r, prepared[2r] = the key's Shoup companions [L][2][L][N], prepared[2r+1] = kprime [2][L][N].
static int ensure_hoist_consts(dpfhe_ctx *ctx) {
    const size_t L = ctx->hp.L, P = ctx->P();
    if (ctx->hoist_delta.bytes()) return DPFHE_OK;   // allocated last
    int rc = ctx->hoist_M.reserve(ctx, P * sizeof(u64));
    if (!rc) rc = ctx->hoist_kprime.reserve(ctx, 2 * P * sizeof(u64));
    if (!rc) rc = ctx->hoist_delta.reserve(ctx, L * L * sizeof(u64));
    if (rc) return rc;
    std::vector<u64> delta(L * L);
    for (size_t j = 0; j < L; ++j)
        for (size_t i = 0; i < L; ++i) delta[j * L + i] = ctx->hp.limbs[j].lp.q % ctx->hp.limbs[i].lp.q;
    CU_TRY(cudaMemcpy(ctx->hoist_delta.get(), delta.data(), delta.size() * sizeof(u64), cudaMemcpyHostToDevice));
    return DPFHE_OK;
}

static int rotate_hoisted_impl(dpfhe_ctx *ctx, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts, const uint64_t *const *d_gks,
                               const uint64_t *const *prepared, uint64_t *d_out, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0 || n_rot == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (!galois_elts || !d_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    const size_t N = ctx->N(), L = ctx->hp.L, P = ctx->P();
    rc = check_rotations(ctx, n_rot, galois_elts, d_gks);
    if (rc) return rc;
    if (overlaps(d_out, n_rot * batch * 2 * P * 8, d_ct, batch * 2 * P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = check_keys_apart(d_out, n_rot * batch * 2 * P * 8, n_rot, d_gks, L * 2 * P * 8);
    if (rc) return rc;
    cudaStream_t st = pick(ctx, stream);
    // scratch: the shared transforms and zero flags of a chunk of the batch
    const size_t per_ct = L * L * N * sizeof(u64), chunk = hoist_chunk(per_ct, batch);
    rc = ctx->hoist_U.reserve(ctx, chunk * per_ct);
    if (!rc) rc = ctx->hoist_zero.reserve(ctx, chunk * sizeof(u32));
    if (!rc) rc = ensure_hoist_consts(ctx);
    if (rc) return rc;
    u64 *U = ctx->hoist_U.get(), *M = ctx->hoist_M.get(), *kp = ctx->hoist_kprime.get(), *delta = ctx->hoist_delta.get();
    u32 *zero = ctx->hoist_zero.get<u32>();
    for (size_t first = 0; first < batch; first += chunk) {
        const size_t cnt = batch - first < chunk ? batch - first : chunk;
        const u64 *in = d_ct + first * 2 * P;
        CU_TRY(cudaMemsetAsync(zero, 0, cnt * sizeof(u32), st));
        if (L > 1) {
            CU_TRY(VCALL(launch_hoist, ctx->lc, in, U, zero, cnt, st));
            note_launch(ctx, 1);
        }
        for (size_t r = 0; r < n_rot; ++r) {
            u64 *out = d_out + (r * batch + first) * 2 * P;
            const u64 *key_s = prepared ? prepared[2 * r] : nullptr, *kprime = prepared ? prepared[2 * r + 1] : kp;
            if (!prepared) {
                CU_TRY(VCALL(launch_rot_prepare, ctx->lc, d_gks[r], (u32)galois_elts[r], delta, M, kp, st));
                note_launch(ctx, 4);   // key_prepare, negmask, ntt, kprime
            }
            CU_TRY(VCALL(launch_rot_apply, ctx->lc, in, L > 1 ? U : nullptr, d_gks[r], kprime, (u32)galois_elts[r], out, cnt, st, key_s));
            note_launch(ctx, 1);
            if (L > 1) {
                CU_TRY(VCALL(launch_ks, ctx->lc, KS_ROTATE, in, nullptr, d_gks[r], out, cnt, (u32)galois_elts[r], st, zero, true, key_s));
                note_launch(ctx, 1);
            }
        }
    }
    return DPFHE_OK;
}

int dpfhe_rotate_hoisted(dpfhe_ctx *ctx, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts, const uint64_t *const *d_gks,
                         uint64_t *d_out, size_t batch, void *stream) {
    return rotate_hoisted_impl(ctx, d_ct, n_rot, galois_elts, d_gks, nullptr, d_out, batch, stream);
}

// Hoisted rotations with grouped hybrid keys (DESIGN.md §2.11b): the mod-up of c1 is done once per ciphertext
// (ks_hoistg_kernel), every rotation is then gathers + multiply-accumulates over all L limbs (rot_apply_grouped_kernel) and
// the division by P (md_tau / md_limb kernels).  Same plaintexts as n_rot calls of dpfhe_rotate_grouped, not the same bits.
// key_s: optional Shoup companions of every key, kept by the caller (a linear layer applies the same rotations to every batch);
// nullptr = built per rotation into the context's scratch (one more launch each).
// lv: the rotations at that level (DESIGN.md §2.21), on its view, reading top-level keys; companions the caller does not give are
// built with the context's launch state over the level's ceil(l / K) digits, as level_launch builds them.
static int rotate_hoisted_grouped_impl(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                                       const uint64_t *const *d_gks, const uint64_t *const *key_s, uint64_t *d_out, size_t batch, uint64_t t_plain,
                                       void *stream, const KsLevel *lv = nullptr) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0 || n_rot == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (!galois_elts || !d_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    const size_t N = ctx->N(), L = lv ? lv->l + n_special : ctx->hp.L, Lq = L - n_special, Pq = Lq * N, dnum = (Lq + n_special - 1) / n_special;
    rc = check_rotations(ctx, n_rot, galois_elts, d_gks);
    if (rc) return rc;
    if (overlaps(d_out, n_rot * batch * 2 * Pq * 8, d_ct, batch * 2 * Pq * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = check_keys_apart(d_out, n_rot * batch * 2 * Pq * 8, n_rot, d_gks, grouped_key_bytes(ctx, n_special));
    if (rc) return rc;
    cudaStream_t st = pick(ctx, stream);
    // scratch per ciphertext of a chunk: lifted digits [dnum][L][N], accumulators [2][L][N], tau' rows [2][K][N]
    const size_t u_words = dnum * L * N, acc_words = 2 * L * N, tau_words = 2 * (size_t)n_special * N;
    const size_t per_ct = (u_words + acc_words + tau_words) * sizeof(u64), chunk = hoist_chunk(per_ct, batch);
    rc = ctx->hoistg.reserve(ctx, chunk * per_ct);
    if (rc) return rc;
    u64 *U = ctx->hoistg.get(), *acc = U + chunk * u_words, *tau = acc + chunk * acc_words;
    MsConsts K;
    GroupConsts G;
    build_group_consts(lv ? lv->hp : ctx->hp, n_special, t_plain, G, K);
    const u32 key_shift = (u32)(ctx->hp.L - L);
    auto on_view = [&](auto launch) { return lv ? on_level_view(ctx, *lv, launch) : launch(ctx->lc); };
    for (size_t first = 0; first < batch; first += chunk) {
        const size_t cnt = batch - first < chunk ? batch - first : chunk;
        const u64 *in = d_ct + first * 2 * Pq;
        CU_TRY(on_view([&](LaunchCtx &lc) { return VCALL(launch_hoist_grouped, lc, in, U, G, cnt, st); }));
        note_launch(ctx, 1);
        for (size_t r = 0; r < n_rot; ++r) {
            u64 *out = d_out + (r * batch + first) * 2 * Pq;
            const u64 *ks = key_s ? key_s[r] : nullptr;
            if (lv && !ks) {
                CU_TRY(VCALL(launch_key_prepare, ctx->lc, d_gks[r], ctx->lc.ks_key_s, (u32)dnum, st));
                ks = ctx->lc.ks_key_s;
            }
            CU_TRY(on_view([&](LaunchCtx &lc) {
                cudaError_t e = VCALL(launch_rot_apply_grouped, lc, in, U, d_gks[r], ks, (u32)galois_elts[r], acc, K, G, cnt, st, key_shift);
                if (e == cudaSuccess) e = VCALL(launch_mod_down_special, lc, acc, tau, out, K, G, 2 * cnt, st);
                return e;
            }));
            note_launch(ctx, key_s ? 3 : 4);   // (key_prepare,) rot_apply_grouped, md_tau, md_limb
        }
    }
    return DPFHE_OK;
}

int dpfhe_rotate_hoisted_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                                 const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    return rotate_hoisted_grouped_impl(ctx, n_special, d_ct, n_rot, galois_elts, d_gks, nullptr, d_out, batch, t_plain, stream);
}

// hoisted rotations at level l (DESIGN.md §2.21): the checks of dpfhe_rotate_hoisted_grouped with the level's sizes, then the level's;
// l = Lq is the top-level call
int dpfhe_rotate_hoisted_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, size_t n_rot,
                                       const uint64_t *galois_elts, const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain,
                                       void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0 || n_rot == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (!galois_elts || !d_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    rc = check_grouped(ctx, n_special, t_plain);
    if (!rc) rc = check_level(ctx, n_special, level, false, t_plain);
    if (!rc) rc = check_rotations(ctx, n_rot, galois_elts, d_gks);
    if (rc) return rc;
    const size_t ct_bytes = batch * 2 * (size_t)level * ctx->N() * 8;
    if (overlaps(d_out, n_rot * ct_bytes, d_ct, ct_bytes)) return fail(DPFHE_ERR_INVALID, "level %u: output must not overlap the input", level);
    rc = check_keys_apart(d_out, n_rot * ct_bytes, n_rot, d_gks, grouped_key_bytes(ctx, n_special));
    if (rc) return rc;
    const KsLevel *lv = nullptr;
    if (level < ctx->hp.L - n_special) rc = level_state(ctx, n_special, level, lv);
    if (rc) return rc;
    return rotate_hoisted_grouped_impl(ctx, n_special, d_ct, n_rot, galois_elts, d_gks, nullptr, d_out, batch, t_plain, stream, lv);
}

// Summed rotations (DESIGN.md §2.17).  Scratch in ctx->hoistg: `head` words first (the key companions of a dpfhe_rotate_sum_grouped
// call; 0 for a slot-sum object, which keeps its own), then per ciphertext of a chunk the lifted digits [dnum][L][N], the summed
// accumulators [2][L][N] and the tau' rows [2][K][N].
// lv: a level call's basis (DESIGN.md §2.20), nullptr for the top level
static size_t rotate_sum_per_ct(const dpfhe_ctx *ctx, unsigned K, const KsLevel *lv = nullptr) {
    const size_t N = ctx->N(), L = lv ? lv->l + K : ctx->hp.L, dnum = (L - K + K - 1) / K;
    return (dnum * L * N + 2 * L * N + 2 * (size_t)K * N) * sizeof(u64);
}

static int rotate_sum_reserve(dpfhe_ctx *ctx, unsigned K, size_t head, size_t batch, const KsLevel *lv = nullptr) {
    const size_t per_ct = rotate_sum_per_ct(ctx, K, lv);
    return ctx->hoistg.reserve(ctx, head * sizeof(u64) + hoist_chunk(per_ct, batch) * per_ct);
}

// one stage: per chunk of the batch the mod-up of c1 (ks_hoistg_kernel), the summed multiply-accumulate of every rotation
// (rot_sum_grouped_kernel) and the division by P (md_tau, md_limb); 4 launches.  The scratch is reserved by the caller.  lv: the
// stage at that level (DESIGN.md §2.20), on its view, with the top-level keys and their companions.
static int rotate_sum_stage(dpfhe_ctx *ctx, unsigned K, size_t head, const u64 *d_ct, u32 n_rot, const u32 *galois, const u64 *const *keys,
                            const u64 *const *key_s, u64 *d_out, size_t batch, const MsConsts &Kc, const GroupConsts &G, cudaStream_t st,
                            const KsLevel *lv = nullptr) {
    const size_t N = ctx->N(), L = lv ? lv->l + K : ctx->hp.L, Pq = (L - K) * N, dnum = (L - K + K - 1) / K;
    const size_t u_words = dnum * L * N, acc_words = 2 * L * N, per_ct = rotate_sum_per_ct(ctx, K, lv), chunk = hoist_chunk(per_ct, batch);
    if (ctx->hoistg.bytes() < head * sizeof(u64) + chunk * per_ct) return fail(DPFHE_ERR_INVALID, "summed rotations: scratch not reserved");
    u64 *U = ctx->hoistg.get() + head, *acc = U + chunk * u_words, *tau = acc + chunk * acc_words;
    const u32 key_shift = (u32)(ctx->hp.L - L);
    for (size_t first = 0; first < batch; first += chunk) {
        const size_t cnt = batch - first < chunk ? batch - first : chunk;
        const u64 *in = d_ct + first * 2 * Pq;
        auto launch = [&](LaunchCtx &lc) {
            cudaError_t e = VCALL(launch_hoist_grouped, lc, in, U, G, cnt, st);
            if (e == cudaSuccess) e = VCALL(launch_rot_sum_grouped, lc, in, U, n_rot, keys, key_s, galois, acc, Kc, G, cnt, st, key_shift);
            if (e == cudaSuccess) e = VCALL(launch_mod_down_special, lc, acc, tau, d_out + first * 2 * Pq, Kc, G, 2 * cnt, st);
            return e;
        };
        CU_TRY(lv ? on_level_view(ctx, *lv, launch) : launch(ctx->lc));
        note_launch(ctx, 4);   // ks_hoistg, rot_sum_grouped, md_tau, md_limb
    }
    return DPFHE_OK;
}

// the checks of dpfhe_rotate_hoisted_grouped, and 1 <= n_rot <= 15
static int check_rotate_sum(dpfhe_ctx *ctx, unsigned n_special, size_t n_rot, const uint64_t *galois_elts, uint64_t t_plain) {
    if (!galois_elts) return fail(DPFHE_ERR_INVALID, "null argument");
    int rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    if (n_rot < 1 || n_rot > (size_t)ROT_SUM_MAX) return fail(DPFHE_ERR_INVALID, "summed rotations take 1 to %d rotations", ROT_SUM_MAX);
    for (size_t r = 0; r < n_rot; ++r) {
        rc = check_galois(ctx, galois_elts[r]);
        if (rc) return rc;
    }
    return DPFHE_OK;
}

// what a dpfhe_rotate_sum_grouped call shares between its chunks: the Shoup companions of its n_rot keys (at the head of
// ctx->hoistg, built once per call), the Galois elements and the constants of the division by P
struct RotSumPrep {
    const u64 *key_s[ROT_SUM_MAX];
    u32 galois[ROT_SUM_MAX];
    size_t head = 0;
    MsConsts K;
    GroupConsts G;
};

// reserves the scratch of chunks of up to `batch` ciphertexts and builds the companions (n_rot launches)
// lv: at that level (DESIGN.md §2.20): the companions of the top-level keys' rows of the level's digits, the level's constants
static int rotate_sum_prepare(dpfhe_ctx *ctx, unsigned n_special, size_t n_rot, const uint64_t *galois_elts, const uint64_t *const *d_gks,
                              uint64_t t_plain, size_t batch, cudaStream_t st, RotSumPrep &pr, const KsLevel *lv = nullptr) {
    const size_t dnum = lv ? (lv->l + n_special - 1) / n_special : key_digits(ctx, n_special), key_words = dnum * 2 * ctx->P();
    pr.head = n_rot * key_words;
    int rc = rotate_sum_reserve(ctx, n_special, pr.head, batch, lv);
    if (rc) return rc;
    u64 *key_s = ctx->hoistg.get();
    for (size_t r = 0; r < n_rot; ++r) {
        CU_TRY(VCALL(launch_key_prepare, ctx->lc, d_gks[r], key_s + r * key_words, (u32)dnum, st));
        note_launch(ctx, 1);
        pr.key_s[r] = key_s + r * key_words;
        pr.galois[r] = (u32)galois_elts[r];
    }
    build_group_consts(lv ? lv->hp : ctx->hp, n_special, t_plain, pr.G, pr.K);
    return DPFHE_OK;
}

int dpfhe_rotate_sum_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                             const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (!d_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    rc = check_rotate_sum(ctx, n_special, n_rot, galois_elts, t_plain);
    if (!rc) rc = check_rotations(ctx, n_rot, galois_elts, d_gks);
    if (rc) return rc;
    const size_t ct_bytes = batch * 2 * (ctx->hp.L - n_special) * ctx->N() * 8;
    if (overlaps(d_out, ct_bytes, d_ct, ct_bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = check_keys_apart(d_out, ct_bytes, n_rot, d_gks, grouped_key_bytes(ctx, n_special));
    if (rc) return rc;
    cudaStream_t st = pick(ctx, stream);
    RotSumPrep pr;
    rc = rotate_sum_prepare(ctx, n_special, n_rot, galois_elts, d_gks, t_plain, batch, st, pr);
    if (rc) return rc;
    return rotate_sum_stage(ctx, n_special, pr.head, d_ct, (u32)n_rot, pr.galois, d_gks, pr.key_s, d_out, batch, pr.K, pr.G, st);
}

// summed rotations at level l (DESIGN.md §2.20): the checks of dpfhe_rotate_sum_grouped, then the level's; the level's scratch
// and constants, the top-level keys' companions over its digits and the stage on its view
int dpfhe_rotate_sum_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *d_ct, size_t n_rot, const uint64_t *galois_elts,
                                   const uint64_t *const *d_gks, uint64_t *d_out, size_t batch, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (!d_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    rc = check_rotate_sum(ctx, n_special, n_rot, galois_elts, t_plain);
    if (!rc) rc = check_rotations(ctx, n_rot, galois_elts, d_gks);
    if (!rc) rc = check_level(ctx, n_special, level, false, t_plain);
    if (rc) return rc;
    if (level == ctx->hp.L - n_special) return dpfhe_rotate_sum_grouped(ctx, n_special, d_ct, n_rot, galois_elts, d_gks, d_out, batch, t_plain, stream);
    const size_t ct_bytes = batch * 2 * (size_t)level * ctx->N() * 8;
    if (overlaps(d_out, ct_bytes, d_ct, ct_bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = check_keys_apart(d_out, ct_bytes, n_rot, d_gks, grouped_key_bytes(ctx, n_special));
    if (rc) return rc;
    const KsLevel *lv = nullptr;
    rc = level_state(ctx, n_special, level, lv);
    if (rc) return rc;
    cudaStream_t st = pick(ctx, stream);
    RotSumPrep pr;
    rc = rotate_sum_prepare(ctx, n_special, n_rot, galois_elts, d_gks, t_plain, batch, st, pr, lv);
    if (rc) return rc;
    return rotate_sum_stage(ctx, n_special, pr.head, d_ct, (u32)n_rot, pr.galois, d_gks, pr.key_s, d_out, batch, pr.K, pr.G, st, lv);
}

int dpfhe_rotate_sum_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_ct, size_t n_rot, const uint64_t *galois_elts,
                                  const uint64_t *h_gks, uint64_t *h_out, size_t batch, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    if (!h_ct || !h_gks || !h_out) return fail(DPFHE_ERR_INVALID, "null host pointer");
    rc = check_rotate_sum(ctx, n_special, n_rot, galois_elts, t_plain);
    if (rc) return rc;
    const size_t key_words = key_digits(ctx, n_special) * 2 * ctx->P(), Pq = (ctx->hp.L - n_special) * ctx->N();
    rc = upload_key(ctx, h_gks, n_rot * key_words);
    if (rc) return rc;
    const u64 *keys[ROT_SUM_MAX];
    for (size_t r = 0; r < n_rot; ++r) keys[r] = ctx->stage_key.get() + r * key_words;
    const size_t chunk = pick_chunk(ctx, 2 * Pq * 8, batch);
    RotSumPrep pr;   // the companions once, for every chunk
    rc = rotate_sum_prepare(ctx, n_special, n_rot, galois_elts, keys, t_plain, chunk, pick(ctx, nullptr), pr);
    if (rc) return rc;
    return run_pipeline(ctx, h_ct, nullptr, h_out, batch, 2 * Pq, 2 * Pq, chunk, [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
        return rotate_sum_stage(ctx, n_special, pr.head, din, (u32)n_rot, pr.galois, keys, pr.key_s, dout, cnt, pr.K, pr.G, pick(ctx, st));
    });
}

// on the prefix of L limbs (DESIGN.md §2.22); L = hp.L is dpfhe_ct_mul_plain
static int ct_mul_plain_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_pt); CHECK_PTR(d_out);
    const size_t P = L * ctx->N(), ct_bytes = batch * 2 * P * 8;
    if (overlaps_shifted(d_out, d_ct, ct_bytes)) return fail(DPFHE_ERR_INVALID, "output must be the input or not overlap it");
    if (overlaps(d_out, ct_bytes, d_pt, P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the plaintext");
    CU_TRY(VCALL(launch_ct_mul_plain, level_view(ctx, L), d_ct, d_pt, d_out, batch, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_ct_mul_plain(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch, void *stream) {
    return ct_mul_plain_at(ctx, ctx ? ctx->hp.L : 0, d_ct, d_pt, d_out, batch, stream);
}

int dpfhe_ct_mul_plain_acc(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_acc, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_pt); CHECK_PTR(d_acc);
    const size_t ct_bytes = batch * 2 * ctx->P() * 8;
    if (overlaps(d_acc, ct_bytes, d_ct, ct_bytes)) return fail(DPFHE_ERR_INVALID, "accumulator must not overlap the input");
    if (overlaps(d_acc, ct_bytes, d_pt, ctx->P() * 8)) return fail(DPFHE_ERR_INVALID, "accumulator must not overlap the plaintext");
    CU_TRY(VCALL(launch_ct_mul_plain_acc, ctx->lc, d_ct, d_pt, d_acc, batch, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

int dpfhe_ct_mul_plain_inner(dpfhe_ctx *ctx, const uint64_t *d_steps, size_t n_steps, const uint64_t *d_pts, size_t n_groups, uint64_t *d_out,
                             size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0 || n_groups == 0) return DPFHE_OK;
    CHECK_PTR(d_steps); CHECK_PTR(d_pts); CHECK_PTR(d_out);
    if (n_steps == 0 || n_steps > 128) return fail(DPFHE_ERR_INVALID, "n_steps must be in [1, 128]");
    if (n_groups > 65535) return fail(DPFHE_ERR_INVALID, "n_groups must be below 65536");
    if (overlaps(d_out, n_groups * batch * 2 * ctx->P() * 8, d_steps, n_steps * batch * 2 * ctx->P() * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    if (overlaps(d_out, n_groups * batch * 2 * ctx->P() * 8, d_pts, n_groups * n_steps * ctx->P() * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap the plaintexts");
    unsigned launches = 0;
    CU_TRY(VCALL(launch_pt_inner, ctx->lc, d_steps, (u32)n_steps, d_pts, (u32)n_groups, d_out, batch, pick(ctx, stream), &launches));
    note_launch(ctx, launches);
    return DPFHE_OK;
}

// The modulus switch of [n_polys][L][N] on the prefix of L = level limbs (DESIGN.md §2.22): its view and host parameters; L = hp.L is
// dpfhe_mod_switch_down
static int mod_switch_down_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_in); CHECK_PTR(d_out);
    if (L < 2) return fail(DPFHE_ERR_INVALID, "mod_switch_down needs at least two limbs");
    const size_t N = ctx->N();
    if (overlaps(d_out, n_polys * (size_t)(L - 1) * N * 8, d_in, n_polys * L * N * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    const uint64_t ql = ctx->hp.limbs[L - 1].lp.q;
    if (t_plain >= ql || (t_plain && t_plain % ql == 0)) return fail(DPFHE_ERR_INVALID, "plaintext modulus must be below the dropped modulus");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    rc = ctx->ms_tau.reserve(ctx, n_polys * N * 8);
    if (rc) return rc;
    MsConsts K;
    build_ms_consts(*hp, t_plain, K);
    CU_TRY(VCALL(launch_mod_switch, level_view(ctx, L), d_in, ctx->ms_tau.get(), d_out, K, n_polys, pick(ctx, stream)));
    note_launch(ctx, 2);
    return DPFHE_OK;
}

int dpfhe_mod_switch_down(dpfhe_ctx *ctx, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain, void *stream) {
    return mod_switch_down_at(ctx, ctx ? ctx->hp.L : 0, d_in, d_out, n_polys, t_plain, stream);
}

// division by the product of the last n_special limbs (DESIGN.md §2.11); n_special = 1 is dpfhe_mod_switch_down
int dpfhe_mod_down_special(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain,
                           void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_in); CHECK_PTR(d_out);
    const unsigned L = ctx->hp.L;
    if (n_special < 1 || n_special > (unsigned)KS_MAX_SPECIAL || n_special >= L)
        return fail(DPFHE_ERR_INVALID, "n_special must be between 1 and %d and below the context's %u limbs", KS_MAX_SPECIAL, L);
    if (overlaps(d_out, n_polys * (size_t)(L - n_special) * ctx->N() * 8, d_in, n_polys * ctx->P() * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    rc = check_t_below_special(ctx, n_special, t_plain, "the dropped moduli");
    if (rc) return rc;
    rc = ctx->ms_tau.reserve(ctx, n_polys * n_special * ctx->N() * 8);
    if (rc) return rc;
    MsConsts K;
    GroupConsts G;
    build_group_consts(ctx->hp, n_special, t_plain, G, K);
    CU_TRY(VCALL(launch_mod_down_special, ctx->lc, d_in, ctx->ms_tau.get(), d_out, K, G, n_polys, pick(ctx, stream)));
    note_launch(ctx, 2);
    return DPFHE_OK;
}

int dpfhe_fill_uniform(dpfhe_ctx *ctx, uint64_t seed, uint64_t first_poly, uint64_t *d_data, size_t n_polys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    CHECK_PTR(d_data);
    CU_TRY(VCALL(launch_fill_uniform, ctx->lc, seed, first_poly, d_data, n_polys, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

// ---------------------------------------------------------------- host-buffer entry points

static int ntt_host(dpfhe_ctx *ctx, uint64_t *h_data, size_t n_polys, bool inverse) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    if (!h_data) return fail(DPFHE_ERR_INVALID, "null pointer: h_data");
    const size_t P = ctx->P();
    return host_call(ctx, {}, nullptr, 0, h_data, nullptr, h_data, n_polys, P, P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         CU_TRY(VCALL(launch_ntt, ctx->lc, din, cnt, inverse, st));
                         note_launch(ctx, 1);
                         CU_TRY(cudaMemcpyAsync(dout, din, cnt * P * 8, cudaMemcpyDeviceToDevice, st));
                         return DPFHE_OK;
                     });
}
int dpfhe_ntt_fwd_host(dpfhe_ctx *ctx, uint64_t *h_data, size_t n_polys) { return ntt_host(ctx, h_data, n_polys, false); }
int dpfhe_ntt_inv_host(dpfhe_ctx *ctx, uint64_t *h_data, size_t n_polys) { return ntt_host(ctx, h_data, n_polys, true); }

int dpfhe_ct_mul_relin_host(dpfhe_ctx *ctx, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk, uint64_t *h_out, size_t batch) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t P = ctx->P();
    return host_call(ctx, {h_a, h_b, h_evk, h_out}, h_evk, 2 * ctx->hp.L * P, h_a, h_b, h_out, batch, 2 * P, 2 * P,
                     [&](u64 *da, u64 *db, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ks_common(ctx, KS_MUL_RELIN, da, db, ctx->stage_key.get(), dout, cnt, 0, st);
                     });
}

int dpfhe_rotate_host(dpfhe_ctx *ctx, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk, uint64_t *h_out, size_t batch) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t P = ctx->P();
    return host_call(ctx, {h_ct, h_gk, h_out}, h_gk, 2 * ctx->hp.L * P, h_ct, nullptr, h_out, batch, 2 * P, 2 * P,
                     [&](u64 *dc, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ks_common(ctx, KS_ROTATE, dc, nullptr, ctx->stage_key.get(), dout, cnt, galois_elt, st);
                     });
}

int dpfhe_ct_mul_relin_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk,
                                    uint64_t *h_out, size_t batch, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t Pq = (ctx->hp.L - n_special) * ctx->N();   // words of a ciphertext polynomial (L - K limbs)
    return host_call(ctx, {h_a, h_b, h_evk, h_out}, h_evk, 2 * key_digits(ctx, n_special) * ctx->P(), h_a, h_b, h_out, batch, 2 * Pq, 2 * Pq,
                     [&](u64 *da, u64 *db, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ks_hybrid_common(ctx, n_special, KS_MUL_RELIN, da, db, ctx->stage_key.get(), dout, cnt, 0, t_plain, st);
                     },
                     [&] { return check_special(ctx, n_special); });
}

// Host form of a call on operand pairs (the inner product, multiply-and-rescale): h_as, h_bs [n_terms][batch][2][Lq][N], h_out
// [batch][2][Lq - drop][N].  The key is uploaded once and the batch pipelined in chunks, each chunk uploading its ciphertexts of
// every pair.  A chunk stages 2 n_terms operands per ciphertext, so its size is budgeted on all of them; where the batch allows, it
// is a whole number of rounds of the persistent grid.  check(): the call's own checks of n_special and t_plain; call(as, bs, dout,
// cnt, st): the device form on one chunk.
extern "C++" {   // a template inside the C entry points' linkage block
template <class Check, class Call>
static int pairs_host(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs, const uint64_t *h_evk,
                      uint64_t *h_out, size_t batch, unsigned drop, Check check, Call call, unsigned level = 0) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_terms < 1 || n_terms > (size_t)DOT_MAX_TERMS) return fail(DPFHE_ERR_INVALID, "n_terms must be in [1, %d]", DOT_MAX_TERMS);
    if (!h_as || !h_bs || !h_evk || !h_out) return fail(DPFHE_ERR_INVALID, "null host pointer");
    rc = check();
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    // words of an operand / output (level: the operands' limbs of a level call, whose key is still the top-level one)
    const size_t Lq = level ? level : ctx->hp.L - n_special, ctw = 2 * Lq * ctx->N(), outw = 2 * (Lq - drop) * ctx->N();
    rc = upload_key(ctx, h_evk, 2 * key_digits(ctx, n_special) * ctx->P());
    if (rc) return rc;
    size_t chunk = std::max<size_t>(1, ((size_t)64 << 20) / (n_terms * ctw * 8));   // ~64 MiB per staged operand side, as pick_chunk
    const size_t round = std::max<size_t>(1, (size_t)ctx->lc.num_sms * 3 / (Lq + n_special));   // ciphertexts per round of the grid (3 CTAs per SM)
    if (chunk > round) chunk -= chunk % round;
    if (chunk > batch) chunk = batch;
    return run_pipeline(
        ctx, h_as, h_bs, h_out, batch, ctw, outw, chunk,
        [&](u64 *da, u64 *db, u64 *dout, size_t cnt, cudaStream_t st) {
            const u64 *as[DOT_MAX_TERMS], *bs[DOT_MAX_TERMS];
            for (size_t t = 0; t < n_terms; ++t) {
                as[t] = da + t * chunk * ctw;
                bs[t] = db + t * chunk * ctw;
            }
            return call(as, bs, dout, cnt, st);
        },
        n_terms, batch * ctw);
}
}

int dpfhe_ct_dot_grouped_host(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs, const uint64_t *h_evk,
                              uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return pairs_host(ctx, n_special, n_terms, h_as, h_bs, h_evk, h_out, batch, 0, [&] { return check_grouped(ctx, n_special, t_plain); },
                      [&](const u64 *const *as, const u64 *const *bs, u64 *dout, size_t cnt, cudaStream_t st) {
                          return dpfhe_ct_dot_grouped(ctx, n_special, n_terms, as, bs, ctx->stage_key.get(), dout, cnt, t_plain, st);
                      });
}

// host forms of multiply-and-rescale: the pipeline of the inner product's, with Lq - 1 limbs per output ciphertext
static int rescale_host(dpfhe_ctx *ctx, unsigned n_special, bool dot, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs, const uint64_t *h_evk,
                        uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return pairs_host(ctx, n_special, n_terms, h_as, h_bs, h_evk, h_out, batch, 1, [&] { return check_rescale(ctx, n_special, t_plain); },
                      [&](const u64 *const *as, const u64 *const *bs, u64 *dout, size_t cnt, cudaStream_t st) {
                          return rescale_common(ctx, n_special, dot, n_terms, as, bs, ctx->stage_key.get(), dout, cnt, t_plain, st);
                      });
}
int dpfhe_ct_mul_relin_rescale_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk,
                                            uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return rescale_host(ctx, n_special, false, 1, h_a, h_b, h_evk, h_out, batch, t_plain);
}
int dpfhe_ct_dot_rescale_grouped_host(dpfhe_ctx *ctx, unsigned n_special, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs,
                                      const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return rescale_host(ctx, n_special, true, n_terms, h_as, h_bs, h_evk, h_out, batch, t_plain);
}

// host forms of multiply-and-rescale at level l (DESIGN.md §2.20): the top-level key uploaded once, operands of l limbs and outputs of
// l - 1 limbs pipelined in chunks
static int rescale_level_host(dpfhe_ctx *ctx, unsigned n_special, unsigned level, bool dot, size_t n_terms, const uint64_t *h_as, const uint64_t *h_bs,
                              const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return pairs_host(ctx, n_special, n_terms, h_as, h_bs, h_evk, h_out, batch, 1, [&] {
        const int rc = check_grouped(ctx, n_special, t_plain);
        return rc ? rc : check_level(ctx, n_special, level, true, t_plain);
    }, [&](const u64 *const *as, const u64 *const *bs, u64 *dout, size_t cnt, cudaStream_t st) {
        return level_pairs(ctx, n_special, level, true, dot, n_terms, as, bs, ctx->stage_key.get(), dout, cnt, t_plain, st);
    }, level);
}
int dpfhe_ct_mul_relin_rescale_grouped_level_host(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *h_a, const uint64_t *h_b,
                                                  const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return rescale_level_host(ctx, n_special, level, false, 1, h_a, h_b, h_evk, h_out, batch, t_plain);
}
int dpfhe_ct_dot_rescale_grouped_level_host(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t n_terms, const uint64_t *h_as,
                                            const uint64_t *h_bs, const uint64_t *h_evk, uint64_t *h_out, size_t batch, uint64_t t_plain) {
    return rescale_level_host(ctx, n_special, level, true, n_terms, h_as, h_bs, h_evk, h_out, batch, t_plain);
}

int dpfhe_rotate_grouped_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk,
                              uint64_t *h_out, size_t batch, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t Pq = (ctx->hp.L - n_special) * ctx->N();
    return host_call(ctx, {h_ct, h_gk, h_out}, h_gk, 2 * key_digits(ctx, n_special) * ctx->P(), h_ct, nullptr, h_out, batch, 2 * Pq, 2 * Pq,
                     [&](u64 *dc, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ks_hybrid_common(ctx, n_special, KS_ROTATE, dc, nullptr, ctx->stage_key.get(), dout, cnt, galois_elt, t_plain, st);
                     },
                     [&] { return check_special(ctx, n_special); });
}

int dpfhe_ct_mul_relin_hybrid_host(dpfhe_ctx *ctx, const uint64_t *h_a, const uint64_t *h_b, const uint64_t *h_evk, uint64_t *h_out,
                                   size_t batch, uint64_t t_plain) {
    return dpfhe_ct_mul_relin_grouped_host(ctx, 1, h_a, h_b, h_evk, h_out, batch, t_plain);
}

int dpfhe_rotate_hybrid_host(dpfhe_ctx *ctx, const uint64_t *h_ct, uint64_t galois_elt, const uint64_t *h_gk, uint64_t *h_out,
                             size_t batch, uint64_t t_plain) {
    return dpfhe_rotate_grouped_host(ctx, 1, h_ct, galois_elt, h_gk, h_out, batch, t_plain);
}

int dpfhe_mod_switch_down_host(dpfhe_ctx *ctx, const uint64_t *h_in, uint64_t *h_out, size_t n_polys, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    const size_t P = ctx->P(), Pq = (ctx->hp.L - 1) * ctx->N();
    return host_call(ctx, {h_in, h_out}, nullptr, 0, h_in, nullptr, h_out, n_polys, P, Pq,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return dpfhe_mod_switch_down(ctx, din, dout, cnt, t_plain, st);
                     },
                     [&] { return ctx->hp.L < 2 ? fail(DPFHE_ERR_INVALID, "mod_switch_down needs at least two limbs") : DPFHE_OK; });
}

int dpfhe_mod_down_special_host(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_in, uint64_t *h_out, size_t n_polys, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_polys == 0) return DPFHE_OK;
    const size_t P = ctx->P(), Pq = (ctx->hp.L - n_special) * ctx->N();
    return host_call(ctx, {h_in, h_out}, nullptr, 0, h_in, nullptr, h_out, n_polys, P, Pq,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return dpfhe_mod_down_special(ctx, n_special, din, dout, cnt, t_plain, st);
                     },
                     [&] {
                         return n_special < 1 || n_special >= ctx->hp.L
                                    ? fail(DPFHE_ERR_INVALID, "n_special must be at least 1 and below the context's limbs") : DPFHE_OK;
                     });
}

int dpfhe_ct_mul_plain_host(dpfhe_ctx *ctx, const uint64_t *h_ct, const uint64_t *h_pt, uint64_t *h_out, size_t batch) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t P = ctx->P();
    return host_call(ctx, {h_ct, h_pt, h_out}, h_pt, P, h_ct, nullptr, h_out, batch, 2 * P, 2 * P,
                     [&](u64 *dc, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         CU_TRY(VCALL(launch_ct_mul_plain, ctx->lc, dc, ctx->stage_key.get(), dout, cnt, st));
                         note_launch(ctx, 1);
                         return DPFHE_OK;
                     });
}

// ---------------------------------------------------------------- CKKS slot encoding (DESIGN.md §2.12)

// the context's encoding tables (built and uploaded once) and `need` bytes of the slot encoders' scratch
static int ckks_prepare(dpfhe_ctx *ctx, size_t need) {
    if (!ctx->ckks_tab.bytes()) {
        std::vector<Cplx> tw;
        std::vector<uint32_t> tj;
        std::vector<uint64_t> pow2;
        build_ckks_tables(ctx->hp, tw, tj, pow2);
        const size_t b_tw = tw.size() * sizeof(Cplx), b_tj = tj.size() * 4, b_p2 = pow2.size() * 8;
        const int rc = ctx->ckks_tab.reserve(ctx, b_tw + b_tj + b_p2);
        if (rc) return rc;
        unsigned char *base = ctx->ckks_tab.get<unsigned char>();
        if (cudaMemcpy(base, tw.data(), b_tw, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(base + b_tw, pow2.data(), b_p2, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(base + b_tw + b_p2, tj.data(), b_tj, cudaMemcpyHostToDevice) != cudaSuccess) {
            ctx->ckks_tab.release();
            return fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: uploading the CKKS tables failed", __FILE__, __LINE__);
        }
        ctx->ckks.tw = (const Cplx *)base;
        ctx->ckks.pow2 = (const u64 *)(base + b_tw);
        ctx->ckks.tj = (const u32 *)(base + b_tw + b_p2);
    }
    return ctx->enc_work.reserve(ctx, need);
}

static bool valid_scale(double scale) { return scale > 0.0 && scale <= 1.7976931348623157e308; }   // finite and positive (NaN fails both)

// The bodies below take L, the limbs of the prefix basis they run on (DESIGN.md §2.22): its view of the context, its host parameters,
// buffers and checks sized by it.  L = hp.L is the top-level call.
static int ckks_encode_at(dpfhe_ctx *ctx, unsigned L, const double *d_slots, uint64_t *d_pt, size_t n_vec, double scale, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!valid_scale(scale)) return fail(DPFHE_ERR_INVALID, "scale must be finite and positive");
    if (n_vec == 0) return DPFHE_OK;
    CHECK_PTR(d_slots); CHECK_PTR(d_pt);
    if (overlaps(d_pt, n_vec * L * ctx->N() * 8, d_slots, n_vec * ctx->N() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    cudaStream_t st = pick(ctx, stream);
    rc = ckks_prepare(ctx, n_vec * ctx->N() * sizeof(double));
    if (rc) return rc;
    const double sc = scale * (2.0 / (double)ctx->N());
    CU_TRY(VCALL(launch_ckks_encode, level_view(ctx, L), (const Cplx *)d_slots, ctx->enc_work.get<double>(), d_pt, ctx->ckks, sc, n_vec, st));
    note_launch(ctx, 2);   // ckks_enc_fft_kernel + ckks_enc_ntt(_pair)_kernel
    return DPFHE_OK;
}
int dpfhe_ckks_encode(dpfhe_ctx *ctx, const double *d_slots, uint64_t *d_pt, size_t n_vec, double scale, void *stream) {
    return ckks_encode_at(ctx, ctx ? ctx->hp.L : 0, d_slots, d_pt, n_vec, scale, stream);
}

static int ckks_decode_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_pt, double *d_slots, size_t n_vec, double scale, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!valid_scale(scale)) return fail(DPFHE_ERR_INVALID, "scale must be finite and positive");
    if (n_vec == 0) return DPFHE_OK;
    CHECK_PTR(d_pt); CHECK_PTR(d_slots);
    const size_t bytes = n_vec * L * ctx->N() * 8;
    if (overlaps(d_slots, n_vec * ctx->N() * 8, d_pt, bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    cudaStream_t st = pick(ctx, stream);
    rc = ckks_prepare(ctx, bytes);
    if (rc) return rc;
    const LaunchCtx lc = level_view(ctx, L);
    u64 *work = ctx->enc_work.get();
    CU_TRY(cudaMemcpyAsync(work, d_pt, bytes, cudaMemcpyDeviceToDevice, st));   // the caller's plaintexts stay unchanged
    CU_TRY(VCALL(launch_ntt, lc, work, n_vec, true, st));
    CkksConsts K;
    build_ckks_consts(*hp, scale, K);
    CU_TRY(VCALL(launch_ckks_decode, lc, work, (Cplx *)d_slots, ctx->ckks, K, n_vec, st));
    note_launch(ctx, 2);   // inverse transform + ckks_dec_kernel
    return DPFHE_OK;
}
int dpfhe_ckks_decode(dpfhe_ctx *ctx, const uint64_t *d_pt, double *d_slots, size_t n_vec, double scale, void *stream) {
    return ckks_decode_at(ctx, ctx ? ctx->hp.L : 0, d_pt, d_slots, n_vec, scale, stream);
}

static int ckks_encode_host_at(dpfhe_ctx *ctx, unsigned L, const double *h_slots, uint64_t *h_pt, size_t n_vec, double scale) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!valid_scale(scale)) return fail(DPFHE_ERR_INVALID, "scale must be finite and positive");
    if (n_vec == 0) return DPFHE_OK;
    const size_t P = L * ctx->N(), S = ctx->N();   // words of a plaintext, and of a slot vector (N/2 complex doubles)
    return host_call(ctx, {h_slots, h_pt}, nullptr, 0, (const u64 *)h_slots, nullptr, h_pt, n_vec, S, P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ckks_encode_at(ctx, L, (const double *)din, dout, cnt, scale, st);
                     });
}
int dpfhe_ckks_encode_host(dpfhe_ctx *ctx, const double *h_slots, uint64_t *h_pt, size_t n_vec, double scale) {
    return ckks_encode_host_at(ctx, ctx ? ctx->hp.L : 0, h_slots, h_pt, n_vec, scale);
}

static int ckks_decode_host_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *h_pt, double *h_slots, size_t n_vec, double scale) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!valid_scale(scale)) return fail(DPFHE_ERR_INVALID, "scale must be finite and positive");
    if (n_vec == 0) return DPFHE_OK;
    const size_t P = L * ctx->N(), S = ctx->N();
    return host_call(ctx, {h_slots, h_pt}, nullptr, 0, h_pt, nullptr, (u64 *)h_slots, n_vec, P, S,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return ckks_decode_at(ctx, L, din, (double *)dout, cnt, scale, st);
                     });
}
int dpfhe_ckks_decode_host(dpfhe_ctx *ctx, const uint64_t *h_pt, double *h_slots, size_t n_vec, double scale) {
    return ckks_decode_host_at(ctx, ctx ? ctx->hp.L : 0, h_pt, h_slots, n_vec, scale);
}

// ---------------------------------------------------------------- BGV slot encoding (DESIGN.md §2.13)

#define CHECK_T(t)                                                                                                \
    do {                                                                                                          \
        if (!bgv_plain_modulus_valid(ctx->hp.log_n, (t)))                                                         \
            return fail(DPFHE_ERR_INVALID, "plaintext modulus %llu is not a prime below 2^31 that is 1 mod 2N",  \
                        (unsigned long long)(t));                                                                 \
    } while (0)

// the tables of plaintext modulus t (kept for the last t used: built and uploaded on first use and whenever t changes) and
// `need` bytes of scratch
static int bgv_prepare(dpfhe_ctx *ctx, uint64_t t, size_t need) {
    if (ctx->bgv_t != t) {
        std::vector<uint32_t> tab;
        BgvTables T;
        if (!build_bgv_tables(ctx->hp, t, tab, T)) return fail(DPFHE_ERR_INVALID, "invalid plaintext modulus");
        int rc = ctx->bgv_tab.bytes() ? dpfhe_synchronize(ctx) : DPFHE_OK;   // earlier calls may still read the old tables
        if (rc) return rc;
        ctx->bgv_t = 0;
        ctx->bgv = BgvTables();
        const size_t bytes = tab.size() * sizeof(uint32_t);
        rc = ctx->bgv_tab.reserve(ctx, bytes);
        if (rc) return rc;
        if (cudaMemcpy(ctx->bgv_tab.get<void>(), tab.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
            ctx->bgv_tab.release();
            return fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: uploading the BGV tables failed", __FILE__, __LINE__);
        }
        T.tw = ctx->bgv_tab.get<const u32>();
        T.pos = T.tw + 4 * ctx->N();
        ctx->bgv = T;
        ctx->bgv_t = t;
    }
    return ctx->enc_work.reserve(ctx, need);
}

// on the prefix of L limbs (DESIGN.md §2.22), as the CKKS bodies above
static int bgv_encode_at(dpfhe_ctx *ctx, unsigned L, const int64_t *d_slots, uint64_t *d_pt, size_t n_vec, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_T(t_plain);
    if (n_vec == 0) return DPFHE_OK;
    CHECK_PTR(d_slots); CHECK_PTR(d_pt);
    if (overlaps(d_pt, n_vec * L * ctx->N() * 8, d_slots, n_vec * ctx->N() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    cudaStream_t st = pick(ctx, stream);
    rc = bgv_prepare(ctx, t_plain, n_vec * ctx->N() * sizeof(u32));
    if (rc) return rc;
    CU_TRY(VCALL(launch_bgv_encode, level_view(ctx, L), d_slots, ctx->enc_work.get<u32>(), d_pt, ctx->bgv, n_vec, st));
    note_launch(ctx, 2);   // bgv_enc_kernel + bgv_enc_ntt(_pair)_kernel
    return DPFHE_OK;
}
int dpfhe_bgv_encode(dpfhe_ctx *ctx, const int64_t *d_slots, uint64_t *d_pt, size_t n_vec, uint64_t t_plain, void *stream) {
    return bgv_encode_at(ctx, ctx ? ctx->hp.L : 0, d_slots, d_pt, n_vec, t_plain, stream);
}

static int bgv_decode_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_pt, uint64_t *d_slots, size_t n_vec, uint64_t t_plain, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_T(t_plain);
    if (n_vec == 0) return DPFHE_OK;
    CHECK_PTR(d_pt); CHECK_PTR(d_slots);
    const size_t bytes = n_vec * L * ctx->N() * 8;
    if (overlaps(d_slots, n_vec * ctx->N() * 8, d_pt, bytes)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    cudaStream_t st = pick(ctx, stream);
    rc = bgv_prepare(ctx, t_plain, bytes);
    if (rc) return rc;
    const LaunchCtx lc = level_view(ctx, L);
    u64 *work = ctx->enc_work.get();
    CU_TRY(cudaMemcpyAsync(work, d_pt, bytes, cudaMemcpyDeviceToDevice, st));   // the caller's plaintexts stay unchanged
    CU_TRY(VCALL(launch_ntt, lc, work, n_vec, true, st));
    BgvConsts K;
    build_bgv_consts(*hp, t_plain, K);
    CU_TRY(VCALL(launch_bgv_decode, lc, work, d_slots, ctx->bgv, K, n_vec, st));
    note_launch(ctx, 2);   // inverse transform + bgv_dec_kernel
    return DPFHE_OK;
}
int dpfhe_bgv_decode(dpfhe_ctx *ctx, const uint64_t *d_pt, uint64_t *d_slots, size_t n_vec, uint64_t t_plain, void *stream) {
    return bgv_decode_at(ctx, ctx ? ctx->hp.L : 0, d_pt, d_slots, n_vec, t_plain, stream);
}

static int bgv_encode_host_at(dpfhe_ctx *ctx, unsigned L, const int64_t *h_slots, uint64_t *h_pt, size_t n_vec, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_T(t_plain);
    if (n_vec == 0) return DPFHE_OK;
    const size_t P = L * ctx->N(), S = ctx->N();   // words of a plaintext, and of a slot vector
    return host_call(ctx, {h_slots, h_pt}, nullptr, 0, (const u64 *)h_slots, nullptr, h_pt, n_vec, S, P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return bgv_encode_at(ctx, L, (const int64_t *)din, dout, cnt, t_plain, st);
                     });
}
int dpfhe_bgv_encode_host(dpfhe_ctx *ctx, const int64_t *h_slots, uint64_t *h_pt, size_t n_vec, uint64_t t_plain) {
    return bgv_encode_host_at(ctx, ctx ? ctx->hp.L : 0, h_slots, h_pt, n_vec, t_plain);
}

static int bgv_decode_host_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *h_pt, uint64_t *h_slots, size_t n_vec, uint64_t t_plain) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_T(t_plain);
    if (n_vec == 0) return DPFHE_OK;
    const size_t P = L * ctx->N(), S = ctx->N();
    return host_call(ctx, {h_slots, h_pt}, nullptr, 0, h_pt, nullptr, h_slots, n_vec, P, S,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return bgv_decode_at(ctx, L, din, dout, cnt, t_plain, st);
                     });
}
int dpfhe_bgv_decode_host(dpfhe_ctx *ctx, const uint64_t *h_pt, uint64_t *h_slots, size_t n_vec, uint64_t t_plain) {
    return bgv_decode_host_at(ctx, ctx ? ctx->hp.L : 0, h_pt, h_slots, n_vec, t_plain);
}
#undef CHECK_T

// ---------------------------------------------------------------- key generation, encryption, decryption (DESIGN.md §2.14)

int dpfhe_random_seed(uint8_t seed[32]) {
    if (!seed) return fail(DPFHE_ERR_INVALID, "null seed");
    size_t got = 0;
    while (got < 32) {
        const ssize_t r = getrandom(seed + got, 32 - got, 0);
        if (r < 0) {
            if (errno == EINTR) continue;
            return fail(DPFHE_ERR_OS, "getrandom failed: %s", strerror(errno));
        }
        got += (size_t)r;
    }
    return DPFHE_OK;
}

#define CHECK_SEED(s) \
    do { if (!(s)) return fail(DPFHE_ERR_INVALID, "null seed"); } while (0)

int dpfhe_secret_keygen(dpfhe_ctx *ctx, const uint8_t seed[32], uint64_t *d_sk, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    CHECK_PTR(d_sk);
    KeyArgs A = build_key_args(ctx->hp, seed, 0, 1);
    A.out = d_sk;
    CU_TRY(VCALL(launch_keys, ctx->lc, KM_SECRET, A, 1, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

static int check_key_special(const dpfhe_ctx *ctx, unsigned n_special) { return n_special ? check_special(ctx, n_special) : DPFHE_OK; }

int dpfhe_relin_keygen(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t *d_key,
                       void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    CHECK_PTR(d_sk); CHECK_PTR(d_key);
    KeyArgs A = build_key_args(ctx->hp, seed, n_special, t_plain);
    if (overlaps(d_key, (size_t)A.ndig * 2 * ctx->P() * 8, d_sk, ctx->P() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    A.s = d_sk;
    A.out = d_key;
    CU_TRY(VCALL(launch_keys, ctx->lc, KM_RELIN, A, A.ndig, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

int dpfhe_galois_keygen(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, size_t n_elts, const uint64_t *galois_elts,
                        const uint8_t seed[32], uint64_t *d_keys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (n_elts == 0) return DPFHE_OK;
    if (!galois_elts) return fail(DPFHE_ERR_INVALID, "null galois_elts");
    for (size_t e = 0; e < n_elts; ++e) {
        rc = check_galois(ctx, galois_elts[e]);
        if (rc) return rc;
    }
    CHECK_PTR(d_sk); CHECK_PTR(d_keys);
    KeyArgs A = build_key_args(ctx->hp, seed, n_special, t_plain);
    A.s = d_sk;
    const size_t key_words = (size_t)A.ndig * 2 * ctx->P();
    if (overlaps(d_keys, n_elts * key_words * 8, d_sk, ctx->P() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    cudaStream_t st = pick(ctx, stream);
    uint64_t launches = 0;
    for (size_t e0 = 0; e0 < n_elts; e0 += KEYS_MAX_ELTS) {
        const size_t cnt = std::min<size_t>(KEYS_MAX_ELTS, n_elts - e0);
        for (size_t e = 0; e < cnt; ++e) A.galois[e] = galois_elts[e0 + e];
        A.out = d_keys + e0 * key_words;
        CU_TRY(VCALL(launch_keys, ctx->lc, KM_GALOIS, A, cnt * A.ndig, st));
        ++launches;
    }
    note_launch(ctx, launches);
    return DPFHE_OK;
}

// encryption and decryption on the prefix of L limbs (DESIGN.md §2.22): the first L rows of the secret, which are the prefix basis's
// own secret; L = hp.L is the top-level call
static int encrypt_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                      const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_sk); CHECK_PTR(d_pt); CHECK_PTR(d_ct);
    const size_t P = L * ctx->N();
    if (overlaps(d_ct, n * 2 * P * 8, d_pt, n * P * 8) || overlaps(d_ct, n * 2 * P * 8, d_sk, P * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    KeyArgs A = build_key_args(*hp, seed, 0, t_plain);
    A.s = d_sk;
    A.pt = d_pt;
    A.out = d_ct;
    A.item0 = first_index;
    CU_TRY(VCALL(launch_keys, level_view(ctx, L), KM_ENC, A, n, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_encrypt(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index, const uint64_t *d_pt,
                  uint64_t *d_ct, size_t n, void *stream) {
    return encrypt_at(ctx, ctx ? ctx->hp.L : 0, t_plain, d_sk, seed, first_index, d_pt, d_ct, n, stream);
}

// the public key (b, a) = (-a s + t NTT(e), a): the encryption of zero with its own nonce domains and item 0
int dpfhe_public_keygen(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t *d_pk, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    CHECK_PTR(d_sk); CHECK_PTR(d_pk);
    if (overlaps(d_pk, 2 * ctx->P() * 8, d_sk, ctx->P() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    KeyArgs A = build_key_args(ctx->hp, seed, 0, t_plain);
    A.s = d_sk;
    A.out = d_pk;
    CU_TRY(VCALL(launch_keys, ctx->lc, KM_PUBLIC_KEY, A, 1, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

// d_pk is the context's public key [2][hp.L][N] at every L: the prefix reads the first L rows of each component
static int encrypt_public_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *d_pk, const uint8_t seed[32], uint64_t first_index,
                             const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_pk); CHECK_PTR(d_pt); CHECK_PTR(d_ct);
    const size_t P = L * ctx->N();
    if (overlaps(d_ct, n * 2 * P * 8, d_pt, n * P * 8) || overlaps(d_ct, n * 2 * P * 8, d_pk, 2 * ctx->P() * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    KeyArgs A = build_key_args(*hp, seed, 0, t_plain);
    A.s = d_pk;   // b at s, a at s + pk_a
    A.pk_a = (u32)ctx->P();
    A.pt = d_pt;
    A.out = d_ct;
    A.item0 = first_index;
    CU_TRY(VCALL(launch_keys, level_view(ctx, L), KM_ENC_PUBLIC, A, n, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_encrypt_public(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_pk, const uint8_t seed[32], uint64_t first_index,
                         const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream) {
    return encrypt_public_at(ctx, ctx ? ctx->hp.L : 0, t_plain, d_pk, seed, first_index, d_pt, d_ct, n, stream);
}

static int decrypt_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_sk, const uint64_t *d_ct, unsigned n_comp, uint64_t *d_pt, size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_comp != 2 && n_comp != 3) return fail(DPFHE_ERR_INVALID, "n_comp must be 2 or 3");
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_sk); CHECK_PTR(d_ct); CHECK_PTR(d_pt);
    const size_t P = L * ctx->N();
    if (overlaps(d_pt, n * P * 8, d_sk, P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    if (overlaps(d_pt, n * P * 8, d_ct, n * n_comp * P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    CU_TRY(VCALL(launch_decrypt, level_view(ctx, L), d_ct, d_sk, d_pt, n_comp, n, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_decrypt(dpfhe_ctx *ctx, const uint64_t *d_sk, const uint64_t *d_ct, unsigned n_comp, uint64_t *d_pt, size_t n, void *stream) {
    return decrypt_at(ctx, ctx ? ctx->hp.L : 0, d_sk, d_ct, n_comp, d_pt, n, stream);
}

// host forms of the key generators: a device buffer of their own, the call, a copy out (synchronous)
static int keygen_host(dpfhe_ctx *ctx, const uint64_t *h_sk, size_t out_words, uint64_t *h_out,
                       int (*call)(dpfhe_ctx *, const uint64_t *, uint64_t *, const void *), const void *arg) {
    if (!h_out) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const size_t sk_words = h_sk ? ctx->P() : 0;
    u64 *d = nullptr;
    CU_TRY(cudaMalloc(&d, (sk_words + out_words) * 8));
    cudaStream_t st = pick(ctx, nullptr);
    int rc = DPFHE_OK;
    if (h_sk && cudaMemcpyAsync(d, h_sk, sk_words * 8, cudaMemcpyHostToDevice, st) != cudaSuccess)
        rc = fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: uploading the secret failed", __FILE__, __LINE__);
    if (!rc) rc = call(ctx, h_sk ? d : nullptr, d + sk_words, arg);
    if (!rc && cudaMemcpyAsync(h_out, d + sk_words, out_words * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess)
        rc = fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: copying the result out failed", __FILE__, __LINE__);
    const cudaError_t e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (!rc && e != cudaSuccess) rc = fail(DPFHE_ERR_CUDA, "CUDA error at %s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e));
    return rc;
}

struct KeygenHostArgs {
    unsigned n_special;
    uint64_t t_plain;
    const uint8_t *seed;
    size_t n_elts;
    const uint64_t *galois_elts;
};

int dpfhe_secret_keygen_host(dpfhe_ctx *ctx, const uint8_t seed[32], uint64_t *h_sk) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    return keygen_host(ctx, nullptr, ctx->P(), h_sk,
                       [](dpfhe_ctx *c, const uint64_t *, uint64_t *out, const void *a) {
                           return dpfhe_secret_keygen(c, (const uint8_t *)a, out, nullptr);
                       }, seed);
}

int dpfhe_relin_keygen_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t *h_key) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (!h_sk) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const KeygenHostArgs args{n_special, t_plain, seed, 0, nullptr};
    return keygen_host(ctx, h_sk, key_digits(ctx, n_special) * 2 * ctx->P(), h_key,
                       [](dpfhe_ctx *c, const uint64_t *sk, uint64_t *out, const void *a) {
                           const KeygenHostArgs &k = *(const KeygenHostArgs *)a;
                           return dpfhe_relin_keygen(c, k.n_special, k.t_plain, sk, k.seed, out, nullptr);
                       }, &args);
}

int dpfhe_galois_keygen_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, size_t n_elts, const uint64_t *galois_elts,
                             const uint8_t seed[32], uint64_t *h_keys) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (n_elts == 0) return DPFHE_OK;
    if (!h_sk) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const KeygenHostArgs args{n_special, t_plain, seed, n_elts, galois_elts};
    return keygen_host(ctx, h_sk, n_elts * key_digits(ctx, n_special) * 2 * ctx->P(), h_keys,
                       [](dpfhe_ctx *c, const uint64_t *sk, uint64_t *out, const void *a) {
                           const KeygenHostArgs &k = *(const KeygenHostArgs *)a;
                           return dpfhe_galois_keygen(c, k.n_special, k.t_plain, sk, k.n_elts, k.galois_elts, k.seed, out, nullptr);
                       }, &args);
}

// host forms on the prefix of L limbs: the secret's first L rows staged once
static int encrypt_host_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                           const uint64_t *h_pt, uint64_t *h_ct, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    const size_t P = L * ctx->N();
    uint64_t next = first_index;   // the chunks run in order: ciphertext k keeps item number first_index + k
    return host_call(ctx, {h_sk, h_pt, h_ct}, h_sk, P, h_pt, nullptr, h_ct, n, P, 2 * P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         const int r = encrypt_at(ctx, L, t_plain, ctx->stage_key.get(), seed, next, din, dout, cnt, st);
                         next += cnt;
                         return r;
                     });
}
int dpfhe_encrypt_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index, const uint64_t *h_pt,
                       uint64_t *h_ct, size_t n) {
    return encrypt_host_at(ctx, ctx ? ctx->hp.L : 0, t_plain, h_sk, seed, first_index, h_pt, h_ct, n);
}

int dpfhe_public_keygen_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t *h_pk) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (!h_sk) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const KeygenHostArgs args{0, t_plain, seed, 0, nullptr};
    return keygen_host(ctx, h_sk, 2 * ctx->P(), h_pk,
                       [](dpfhe_ctx *c, const uint64_t *sk, uint64_t *out, const void *a) {
                           const KeygenHostArgs &k = *(const KeygenHostArgs *)a;
                           return dpfhe_public_keygen(c, k.t_plain, sk, k.seed, out, nullptr);
                       }, &args);
}

// the public key (2P words of the top level, whatever L) is the staged shared operand; item numbers continue across chunks as in
// dpfhe_encrypt_host
static int encrypt_public_host_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *h_pk, const uint8_t seed[32], uint64_t first_index,
                                  const uint64_t *h_pt, uint64_t *h_ct, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    const size_t P = L * ctx->N();
    uint64_t next = first_index;
    return host_call(ctx, {h_pk, h_pt, h_ct}, h_pk, 2 * ctx->P(), h_pt, nullptr, h_ct, n, P, 2 * P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         const int r = encrypt_public_at(ctx, L, t_plain, ctx->stage_key.get(), seed, next, din, dout, cnt, st);
                         next += cnt;
                         return r;
                     });
}
int dpfhe_encrypt_public_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_pk, const uint8_t seed[32], uint64_t first_index,
                              const uint64_t *h_pt, uint64_t *h_ct, size_t n) {
    return encrypt_public_host_at(ctx, ctx ? ctx->hp.L : 0, t_plain, h_pk, seed, first_index, h_pt, h_ct, n);
}

static int decrypt_host_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *h_sk, const uint64_t *h_ct, unsigned n_comp, uint64_t *h_pt, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_comp != 2 && n_comp != 3) return fail(DPFHE_ERR_INVALID, "n_comp must be 2 or 3");
    if (n == 0) return DPFHE_OK;
    const size_t P = L * ctx->N();
    return host_call(ctx, {h_sk, h_ct, h_pt}, h_sk, P, h_ct, nullptr, h_pt, n, n_comp * P, P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return decrypt_at(ctx, L, ctx->stage_key.get(), din, n_comp, dout, cnt, st);
                     });
}
int dpfhe_decrypt_host(dpfhe_ctx *ctx, const uint64_t *h_sk, const uint64_t *h_ct, unsigned n_comp, uint64_t *h_pt, size_t n) {
    return decrypt_host_at(ctx, ctx ? ctx->hp.L : 0, h_sk, h_ct, n_comp, h_pt, n);
}

// ---- the keyless calls at level l (DESIGN.md §2.22): each is, bit for bit, the call it is named after on a context over the prefix
// basis {q_0 .. q_{l-1}}, run on this context's view of that prefix.  1 <= level <= L.
int dpfhe_ckks_encode_level(dpfhe_ctx *ctx, unsigned level, const double *d_slots, uint64_t *d_pt, size_t n_vec, double scale, void *stream) {
    return prefix_call(ctx, level, [&] { return ckks_encode_at(ctx, level, d_slots, d_pt, n_vec, scale, stream); });
}
int dpfhe_ckks_decode_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_pt, double *d_slots, size_t n_vec, double scale, void *stream) {
    return prefix_call(ctx, level, [&] { return ckks_decode_at(ctx, level, d_pt, d_slots, n_vec, scale, stream); });
}
int dpfhe_ckks_encode_level_host(dpfhe_ctx *ctx, unsigned level, const double *h_slots, uint64_t *h_pt, size_t n_vec, double scale) {
    return prefix_call(ctx, level, [&] { return ckks_encode_host_at(ctx, level, h_slots, h_pt, n_vec, scale); });
}
int dpfhe_ckks_decode_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_pt, double *h_slots, size_t n_vec, double scale) {
    return prefix_call(ctx, level, [&] { return ckks_decode_host_at(ctx, level, h_pt, h_slots, n_vec, scale); });
}
int dpfhe_bgv_encode_level(dpfhe_ctx *ctx, unsigned level, const int64_t *d_slots, uint64_t *d_pt, size_t n_vec, uint64_t t_plain, void *stream) {
    return prefix_call(ctx, level, [&] { return bgv_encode_at(ctx, level, d_slots, d_pt, n_vec, t_plain, stream); });
}
int dpfhe_bgv_decode_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_pt, uint64_t *d_slots, size_t n_vec, uint64_t t_plain, void *stream) {
    return prefix_call(ctx, level, [&] { return bgv_decode_at(ctx, level, d_pt, d_slots, n_vec, t_plain, stream); });
}
int dpfhe_bgv_encode_level_host(dpfhe_ctx *ctx, unsigned level, const int64_t *h_slots, uint64_t *h_pt, size_t n_vec, uint64_t t_plain) {
    return prefix_call(ctx, level, [&] { return bgv_encode_host_at(ctx, level, h_slots, h_pt, n_vec, t_plain); });
}
int dpfhe_bgv_decode_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_pt, uint64_t *h_slots, size_t n_vec, uint64_t t_plain) {
    return prefix_call(ctx, level, [&] { return bgv_decode_host_at(ctx, level, h_pt, h_slots, n_vec, t_plain); });
}
int dpfhe_encrypt_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                        const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream) {
    return prefix_call(ctx, level, [&] { return encrypt_at(ctx, level, t_plain, d_sk, seed, first_index, d_pt, d_ct, n, stream); });
}
int dpfhe_encrypt_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                             const uint64_t *h_pt, uint64_t *h_ct, size_t n) {
    return prefix_call(ctx, level, [&] { return encrypt_host_at(ctx, level, t_plain, h_sk, seed, first_index, h_pt, h_ct, n); });
}
int dpfhe_encrypt_public_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_pk, const uint8_t seed[32], uint64_t first_index,
                               const uint64_t *d_pt, uint64_t *d_ct, size_t n, void *stream) {
    return prefix_call(ctx, level, [&] { return encrypt_public_at(ctx, level, t_plain, d_pk, seed, first_index, d_pt, d_ct, n, stream); });
}
int dpfhe_encrypt_public_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_pk, const uint8_t seed[32],
                                    uint64_t first_index, const uint64_t *h_pt, uint64_t *h_ct, size_t n) {
    return prefix_call(ctx, level, [&] { return encrypt_public_host_at(ctx, level, t_plain, h_pk, seed, first_index, h_pt, h_ct, n); });
}
int dpfhe_decrypt_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_sk, const uint64_t *d_ct, unsigned n_comp, uint64_t *d_pt, size_t n,
                        void *stream) {
    return prefix_call(ctx, level, [&] { return decrypt_at(ctx, level, d_sk, d_ct, n_comp, d_pt, n, stream); });
}
int dpfhe_decrypt_level_host(dpfhe_ctx *ctx, unsigned level, const uint64_t *h_sk, const uint64_t *h_ct, unsigned n_comp, uint64_t *h_pt,
                             size_t n) {
    return prefix_call(ctx, level, [&] { return decrypt_host_at(ctx, level, h_sk, h_ct, n_comp, h_pt, n); });
}
int dpfhe_ct_mul_plain_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch,
                             void *stream) {
    return prefix_call(ctx, level, [&] { return ct_mul_plain_at(ctx, level, d_ct, d_pt, d_out, batch, stream); });
}
int dpfhe_mod_switch_down_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_in, uint64_t *d_out, size_t n_polys, uint64_t t_plain,
                                void *stream) {
    return prefix_call(ctx, level, [&] { return mod_switch_down_at(ctx, level, d_in, d_out, n_polys, t_plain, stream); });
}
// ---------------------------------------------------------------- seeded ciphertexts and switch keys (DESIGN.md §2.23)

static void seed_words(const uint8_t b[32], u32 w[8]) {
    for (int i = 0; i < 8; ++i) w[i] = (u32)b[4 * i] | (u32)b[4 * i + 1] << 8 | (u32)b[4 * i + 2] << 16 | (u32)b[4 * i + 3] << 24;
}

// a_seed of the key owner's seed: words 0..7 of its ChaCha20 block at counter 0, nonce (KD_PUBLIC_SEED, 0, 0)
static void public_seed_words(const uint8_t seed[32], u32 a_seed[8]) {
    u32 key[8], w[16];
    seed_words(seed, key);
    gen::chacha20_block(key, 0, key_nonce0(KD_PUBLIC_SEED, 0, 0, 0), 0, 0, w);
    for (int i = 0; i < 8; ++i) a_seed[i] = w[i];
}

int dpfhe_seeded_public_seed(const uint8_t seed[32], uint8_t a_seed[32]) {
    if (!seed || !a_seed) return fail(DPFHE_ERR_INVALID, "null seed");
    u32 w[8];
    public_seed_words(seed, w);
    for (int i = 0; i < 32; ++i) a_seed[i] = (uint8_t)(w[i / 4] >> (8 * (i % 4)));
    return DPFHE_OK;
}

// the key arguments of a seeded launch: build_key_args' with the public seed a_seed (words) of the `a` rows
static SeededKeyArgs seeded_args(const HostParams &hp, const uint8_t seed[32], unsigned K, uint64_t t_plain, const u32 a_seed[8]) {
    SeededKeyArgs A;
    static_cast<KeyArgs &>(A) = build_key_args(hp, seed, K, t_plain);
    for (int i = 0; i < 8; ++i) A.a_seed[i] = a_seed[i];
    return A;
}

// the key arguments of an expansion over the first L limbs: only a_seed, K, ndig and the uniform reduction's constants are read
static SeededKeyArgs expand_args(const HostParams &hp, const uint8_t a_seed[32], unsigned K) {
    u32 w[8];
    seed_words(a_seed, w);
    return seeded_args(hp, a_seed, K, 0, w);
}

static int encrypt_seeded_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index,
                             const uint64_t *d_pt, uint64_t *d_c0, size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_sk); CHECK_PTR(d_pt); CHECK_PTR(d_c0);
    const size_t P = L * ctx->N();
    if (overlaps(d_c0, n * P * 8, d_pt, n * P * 8) || overlaps(d_c0, n * P * 8, d_sk, P * 8))
        return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    u32 a_seed[8];
    public_seed_words(seed, a_seed);
    SeededKeyArgs A = seeded_args(*hp, seed, 0, t_plain, a_seed);
    A.s = d_sk;
    A.pt = d_pt;
    A.out = d_c0;
    A.item0 = first_index;
    CU_TRY(VCALL(launch_keys, level_view(ctx, L), KM_ENC_SEEDED, A, n, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

static int encrypt_seeded_host_at(dpfhe_ctx *ctx, unsigned L, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                                  const uint64_t *h_pt, uint64_t *h_c0, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    if (n == 0) return DPFHE_OK;
    const size_t P = L * ctx->N();
    uint64_t next = first_index;   // as dpfhe_encrypt_host: ciphertext k keeps item number first_index + k across chunks
    return host_call(ctx, {h_sk, h_pt, h_c0}, h_sk, P, h_pt, nullptr, h_c0, n, P, P,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         const int r = encrypt_seeded_at(ctx, L, t_plain, ctx->stage_key.get(), seed, next, din, dout, cnt, st);
                         next += cnt;
                         return r;
                     });
}

static int expand_ciphertexts_at(dpfhe_ctx *ctx, unsigned L, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *d_c0, uint64_t *d_ct,
                                 size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(a_seed);
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_c0); CHECK_PTR(d_ct);
    const size_t P = L * ctx->N();
    if (overlaps(d_ct, n * 2 * P * 8, d_c0, n * P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    SeededKeyArgs A = expand_args(*hp, a_seed, 0);
    A.item0 = first_index;
    CU_TRY(VCALL(launch_expand_seeded, level_view(ctx, L), false, A, d_c0, d_ct, n, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}

// host c0 rows straight into d_ct's c0 rows, chunk by chunk, each chunk's c1 rows expanded in place behind its copy
static int upload_seeded_ciphertexts_at(dpfhe_ctx *ctx, unsigned L, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *h_c0,
                                        uint64_t *d_ct, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(a_seed);
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_ct);
    const HostParams *hp = prefix_params(ctx, L);
    if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    const size_t P = L * ctx->N();
    SeededKeyArgs A = expand_args(*hp, a_seed, 0);
    A.item0 = first_index;
    const LaunchCtx lc = level_view(ctx, L);
    return host_call(ctx, {h_c0}, nullptr, 0, h_c0, nullptr, nullptr, n, P, 2 * P,
                     [&](u64 *, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         CU_TRY(VCALL(launch_expand_seeded, lc, false, A, nullptr, dout, cnt, pick(ctx, st)));
                         A.item0 += cnt;
                         note_launch(ctx, 1);
                         return DPFHE_OK;
                     }, no_check, DeviceOut{d_ct, P});
}

int dpfhe_encrypt_seeded(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t first_index, const uint64_t *d_pt,
                         uint64_t *d_c0, size_t n, void *stream) {
    return encrypt_seeded_at(ctx, ctx ? ctx->hp.L : 0, t_plain, d_sk, seed, first_index, d_pt, d_c0, n, stream);
}
int dpfhe_encrypt_seeded_host(dpfhe_ctx *ctx, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32], uint64_t first_index,
                              const uint64_t *h_pt, uint64_t *h_c0, size_t n) {
    return encrypt_seeded_host_at(ctx, ctx ? ctx->hp.L : 0, t_plain, h_sk, seed, first_index, h_pt, h_c0, n);
}
int dpfhe_encrypt_seeded_level(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32],
                               uint64_t first_index, const uint64_t *d_pt, uint64_t *d_c0, size_t n, void *stream) {
    return prefix_call(ctx, level, [&] { return encrypt_seeded_at(ctx, level, t_plain, d_sk, seed, first_index, d_pt, d_c0, n, stream); });
}
int dpfhe_encrypt_seeded_level_host(dpfhe_ctx *ctx, unsigned level, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32],
                                    uint64_t first_index, const uint64_t *h_pt, uint64_t *h_c0, size_t n) {
    return prefix_call(ctx, level, [&] { return encrypt_seeded_host_at(ctx, level, t_plain, h_sk, seed, first_index, h_pt, h_c0, n); });
}
int dpfhe_expand_ciphertexts(dpfhe_ctx *ctx, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *d_c0, uint64_t *d_ct, size_t n,
                             void *stream) {
    return expand_ciphertexts_at(ctx, ctx ? ctx->hp.L : 0, a_seed, first_index, d_c0, d_ct, n, stream);
}
int dpfhe_expand_ciphertexts_level(dpfhe_ctx *ctx, unsigned level, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *d_c0,
                                   uint64_t *d_ct, size_t n, void *stream) {
    return prefix_call(ctx, level, [&] { return expand_ciphertexts_at(ctx, level, a_seed, first_index, d_c0, d_ct, n, stream); });
}
int dpfhe_upload_seeded_ciphertexts(dpfhe_ctx *ctx, const uint8_t a_seed[32], uint64_t first_index, const uint64_t *h_c0, uint64_t *d_ct,
                                    size_t n) {
    return upload_seeded_ciphertexts_at(ctx, ctx ? ctx->hp.L : 0, a_seed, first_index, h_c0, d_ct, n);
}
int dpfhe_upload_seeded_ciphertexts_level(dpfhe_ctx *ctx, unsigned level, const uint8_t a_seed[32], uint64_t first_index,
                                          const uint64_t *h_c0, uint64_t *d_ct, size_t n) {
    return prefix_call(ctx, level, [&] { return upload_seeded_ciphertexts_at(ctx, level, a_seed, first_index, h_c0, d_ct, n); });
}

// seeded relinearisation key (galois_elts = nullptr, n_elts = 1) or Galois keys: the b rows [n_elts][dnum][L][N]
static int switch_keygen_seeded(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, size_t n_elts,
                                const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *d_b, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (n_elts == 0) return DPFHE_OK;
    for (size_t e = 0; galois_elts && e < n_elts; ++e) {
        rc = check_galois(ctx, galois_elts[e]);
        if (rc) return rc;
    }
    CHECK_PTR(d_sk); CHECK_PTR(d_b);
    u32 a_seed[8];
    public_seed_words(seed, a_seed);
    SeededKeyArgs A = seeded_args(ctx->hp, seed, n_special, t_plain, a_seed);
    A.s = d_sk;
    const size_t key_words = (size_t)A.ndig * ctx->P();
    if (overlaps(d_b, n_elts * key_words * 8, d_sk, ctx->P() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    cudaStream_t st = pick(ctx, stream);
    uint64_t launches = 0;
    for (size_t e0 = 0; e0 < n_elts; e0 += KEYS_MAX_ELTS) {
        const size_t cnt = std::min<size_t>(KEYS_MAX_ELTS, n_elts - e0);
        for (size_t e = 0; galois_elts && e < cnt; ++e) A.galois[e] = galois_elts[e0 + e];
        A.out = d_b + e0 * key_words;
        CU_TRY(VCALL(launch_keys, ctx->lc, galois_elts ? KM_GALOIS_SEEDED : KM_RELIN_SEEDED, A, cnt * A.ndig, st));
        ++launches;
    }
    note_launch(ctx, launches);
    return DPFHE_OK;
}

int dpfhe_relin_keygen_seeded(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, const uint8_t seed[32], uint64_t *d_b,
                              void *stream) {
    return switch_keygen_seeded(ctx, n_special, t_plain, d_sk, 1, nullptr, seed, d_b, stream);
}
int dpfhe_galois_keygen_seeded(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *d_sk, size_t n_elts,
                               const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *d_b, void *stream) {
    if (ctx && n_elts && !galois_elts) return fail(DPFHE_ERR_INVALID, "null galois_elts");
    return switch_keygen_seeded(ctx, n_special, t_plain, d_sk, n_elts, galois_elts, seed, d_b, stream);
}
int dpfhe_relin_keygen_seeded_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, const uint8_t seed[32],
                                   uint64_t *h_b) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (!h_sk) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const KeygenHostArgs args{n_special, t_plain, seed, 0, nullptr};
    return keygen_host(ctx, h_sk, key_digits(ctx, n_special) * ctx->P(), h_b,
                       [](dpfhe_ctx *c, const uint64_t *sk, uint64_t *out, const void *a) {
                           const KeygenHostArgs &k = *(const KeygenHostArgs *)a;
                           return dpfhe_relin_keygen_seeded(c, k.n_special, k.t_plain, sk, k.seed, out, nullptr);
                       }, &args);
}
int dpfhe_galois_keygen_seeded_host(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_sk, size_t n_elts,
                                    const uint64_t *galois_elts, const uint8_t seed[32], uint64_t *h_b) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(seed);
    rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (n_elts == 0) return DPFHE_OK;
    if (!galois_elts) return fail(DPFHE_ERR_INVALID, "null galois_elts");
    for (size_t e = 0; e < n_elts; ++e) {
        rc = check_galois(ctx, galois_elts[e]);
        if (rc) return rc;
    }
    if (!h_sk) return fail(DPFHE_ERR_INVALID, "null host pointer");
    const KeygenHostArgs args{n_special, t_plain, seed, n_elts, galois_elts};
    return keygen_host(ctx, h_sk, n_elts * key_digits(ctx, n_special) * ctx->P(), h_b,
                       [](dpfhe_ctx *c, const uint64_t *sk, uint64_t *out, const void *a) {
                           const KeygenHostArgs &k = *(const KeygenHostArgs *)a;
                           return dpfhe_galois_keygen_seeded(c, k.n_special, k.t_plain, sk, k.n_elts, k.galois_elts, k.seed, out, nullptr);
                       }, &args);
}

// the checks every expansion of switch keys makes before its first copy or launch: K and the item numbers
static int check_key_items(const dpfhe_ctx *ctx, unsigned n_special, size_t n_keys, const uint64_t *items) {
    int rc = check_key_special(ctx, n_special);
    if (rc) return rc;
    if (n_keys && !items) return fail(DPFHE_ERR_INVALID, "null items");
    for (size_t e = 0; e < n_keys; ++e)
        if (items[e] && (rc = check_galois(ctx, items[e]))) return rc;
    return DPFHE_OK;
}

// n_keys seeded keys' b rows (src, [n_keys][dnum][L][N]; nullptr: already in place in dst) -> dst [n_keys][dnum][2][L][N], one launch per
// KEYS_MAX_ELTS keys; returns the launches
static cudaError_t launch_expand_keys(dpfhe_ctx *ctx, SeededKeyArgs &A, size_t n_keys, const uint64_t *items, const u64 *src, u64 *dst, cudaStream_t st,
                                      uint64_t &launches) {
    const size_t key_words = (size_t)A.ndig * ctx->P();
    for (size_t e0 = 0; e0 < n_keys; e0 += KEYS_MAX_ELTS) {
        const size_t cnt = std::min<size_t>(KEYS_MAX_ELTS, n_keys - e0);
        for (size_t e = 0; e < cnt; ++e) A.galois[e] = items[e0 + e];
        const cudaError_t err = VCALL(launch_expand_seeded, ctx->lc, true, A, src ? src + e0 * key_words : nullptr, dst + e0 * 2 * key_words,
                                      cnt * A.ndig, st);
        if (err != cudaSuccess) return err;
        ++launches;
    }
    return cudaSuccess;
}

int dpfhe_expand_switch_keys(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                             const uint64_t *d_b, uint64_t *d_keys, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(a_seed);
    rc = check_key_items(ctx, n_special, n_keys, items);
    if (rc || n_keys == 0) return rc;
    CHECK_PTR(d_b); CHECK_PTR(d_keys);
    const size_t key_words = key_digits(ctx, n_special) * ctx->P();
    if (overlaps(d_keys, n_keys * 2 * key_words * 8, d_b, n_keys * key_words * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    SeededKeyArgs A = expand_args(ctx->hp, a_seed, n_special);
    uint64_t launches = 0;
    CU_TRY(launch_expand_keys(ctx, A, n_keys, items, d_b, d_keys, pick(ctx, stream), launches));
    note_launch(ctx, launches);
    return DPFHE_OK;
}

int dpfhe_upload_seeded_switch_keys(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                                    const uint64_t *h_b, uint64_t *d_keys) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(a_seed);
    rc = check_key_items(ctx, n_special, n_keys, items);
    if (rc || n_keys == 0) return rc;
    CHECK_PTR(d_keys);
    const size_t key_words = key_digits(ctx, n_special) * ctx->P();
    SeededKeyArgs A = expand_args(ctx->hp, a_seed, n_special);
    size_t next = 0;
    return host_call(ctx, {h_b}, nullptr, 0, h_b, nullptr, nullptr, n_keys, key_words, 2 * key_words,
                     [&](u64 *, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         uint64_t launches = 0;
                         CU_TRY(launch_expand_keys(ctx, A, cnt, items + next, nullptr, dout, pick(ctx, st), launches));
                         note_launch(ctx, launches);
                         next += cnt;
                         return DPFHE_OK;
                     }, no_check, DeviceOut{d_keys, ctx->P()});
}

int dpfhe_expand_switch_keys_host(dpfhe_ctx *ctx, unsigned n_special, const uint8_t a_seed[32], size_t n_keys, const uint64_t *items,
                                  const uint64_t *h_b, uint64_t *h_keys) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_SEED(a_seed);
    rc = check_key_items(ctx, n_special, n_keys, items);
    if (rc || n_keys == 0) return rc;
    const size_t key_words = key_digits(ctx, n_special) * ctx->P();
    if (overlaps(h_keys, n_keys * 2 * key_words * 8, h_b, n_keys * key_words * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    SeededKeyArgs A = expand_args(ctx->hp, a_seed, n_special);
    size_t next = 0;
    return host_call(ctx, {h_b, h_keys}, nullptr, 0, h_b, nullptr, h_keys, n_keys, key_words, 2 * key_words,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         uint64_t launches = 0;
                         CU_TRY(launch_expand_keys(ctx, A, cnt, items + next, din, dout, pick(ctx, st), launches));
                         note_launch(ctx, launches);
                         next += cnt;
                         return DPFHE_OK;
                     });
}

// ---------------------------------------------------------------- compact ciphertexts (DESIGN.md §2.24)

// the checks on bits and t_plain (level 1), and the switch's constants
static int compact_args(const dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, CompactArgs &A) {
    const uint64_t q = ctx->hp.limbs[0].lp.q;
    // compared without a sum, so that no `bits` wraps past the range check; every shift below is then by less than 64
    if (bits < 2 || bits >= 64 - ctx->hp.log_n || ((uint64_t)ctx->N() << bits) >= q)
        return fail(DPFHE_ERR_INVALID, "bits must be at least 2 with N 2^bits below q0");
    if (t_plain && (!(t_plain & 1) || t_plain < 3 || t_plain >= (uint64_t)1 << (bits - 1)))
        return fail(DPFHE_ERR_INVALID, "plaintext modulus must be 0 or odd with 3 <= t < 2^(bits-1)");
    build_compact_args(q, ctx->hp.log_n, bits, t_plain, A);
    return DPFHE_OK;
}

// every check of a compaction at `level` (1 <= level <= L checked by the caller) before its first launch
static int check_compact(const dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, CompactArgs &A) {
    int rc = compact_args(ctx, bits, t_plain, A);
    if (rc || !t_plain) return rc;
    for (unsigned k = level; k >= 2; --k) {   // the checks of dpfhe_mod_switch_down_level at k
        const uint64_t ql = ctx->hp.limbs[k - 1].lp.q;
        if (t_plain >= ql || t_plain % ql == 0) return fail(DPFHE_ERR_INVALID, "plaintext modulus must be below the dropped modulus");
    }
    return DPFHE_OK;
}

// the launches of a checked compaction of n ciphertexts at level l: the level-1 pairs into compact_work, the inverse transform, the pack
static int compact_run(dpfhe_ctx *ctx, unsigned l, const CompactArgs &A, const uint64_t *d_ct, uint64_t *d_out, size_t n, cudaStream_t st) {
    const size_t N = ctx->N(), polys = 2 * n;
    const bool chain = A.t && l >= 2;
    const size_t words_a = polys * N * (chain ? l - 1 : 1), words_b = chain && l >= 3 ? polys * N * (l - 2) : 0;
    int rc = ctx->compact_work.reserve(ctx, (words_a + words_b) * 8);
    if (!rc && chain) rc = ctx->ms_tau.reserve(ctx, polys * N * 8);
    if (rc) return rc;
    u64 *bufs[2] = {ctx->compact_work.get(), ctx->compact_work.get() + words_a};
    u64 *x = bufs[0];
    uint64_t launches = 2;
    if (chain) {
        // BGV: l - 1 modulus switches, alternating between the two buffers
        const u64 *src = d_ct;
        for (unsigned k = l, i = 0; k >= 2; --k, ++i) {
            const HostParams *hp = prefix_params(ctx, k);
            if (!hp) return fail(DPFHE_ERR_NOMEM, "out of host memory");
            MsConsts K;
            build_ms_consts(*hp, A.t, K);
            x = bufs[i & 1];
            CU_TRY(VCALL(launch_mod_switch, level_view(ctx, k), src, ctx->ms_tau.get(), x, K, polys, st));
            src = x;
            launches += 2;
        }
    } else {
        // CKKS (or level 1): limb 0 of every polynomial
        CU_TRY(cudaMemcpy2DAsync(x, N * 8, d_ct, l * N * 8, N * 8, polys, cudaMemcpyDeviceToDevice, st));
    }
    const LaunchCtx lc1 = level_view(ctx, 1);
    CU_TRY(VCALL(launch_ntt, lc1, x, polys, true, st));
    CU_TRY(VCALL(launch_compact_pack, lc1, A, x, d_out, polys, st));
    note_launch(ctx, launches);
    return DPFHE_OK;
}

static int compact_at(dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, const uint64_t *d_ct, uint64_t *d_out, size_t n,
                      void *stream) {
    CompactArgs A;
    int rc = check_compact(ctx, level, bits, t_plain, A);
    if (rc) return rc;
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_ct); CHECK_PTR(d_out);
    if (overlaps(d_out, n * 2 * A.tiles * bits * 8, d_ct, n * 2 * level * ctx->N() * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the input");
    return compact_run(ctx, level, A, d_ct, d_out, n, pick(ctx, stream));
}

int dpfhe_compact_ciphertexts(dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, const uint64_t *d_ct, uint64_t *d_out,
                              size_t n, void *stream) {
    return prefix_call(ctx, level, [&] { return compact_at(ctx, level, bits, t_plain, d_ct, d_out, n, stream); });
}

// device ciphertexts read in place chunk by chunk (DeviceIn), each chunk compacted into its staging slot, the packed words downloaded
int dpfhe_download_compact_ciphertexts(dpfhe_ctx *ctx, unsigned level, unsigned bits, uint64_t t_plain, const uint64_t *d_ct,
                                       uint64_t *h_out, size_t n) {
    return prefix_call(ctx, level, [&]() -> int {
        CompactArgs A;
        int rc = check_compact(ctx, level, bits, t_plain, A);
        if (rc) return rc;
        if (n == 0) return DPFHE_OK;
        CHECK_PTR(d_ct);
        const size_t in_words = 2 * level * ctx->N(), out_words = 2 * (size_t)A.tiles * bits;
        return host_call(ctx, {h_out}, nullptr, 0, nullptr, nullptr, h_out, n, in_words, out_words,
                         [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) { return compact_run(ctx, level, A, din, dout, cnt, pick(ctx, st)); },
                         no_check, DeviceOut{}, DeviceIn{d_ct});
    });
}

// c1' lifted, forward transform, times s_0, inverse transform, c0' added and mapped, forward transform.  The product by s_0 is
// ct_mul_plain's, whose plaintext is shared by every row: the rows are taken two by two as level-1 ciphertexts, an odd count padded
// with a zero row.
static int decrypt_compact_at(dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, const uint64_t *d_sk, const uint64_t *d_cct, uint64_t *d_pt,
                              size_t n, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CompactArgs A;
    rc = compact_args(ctx, bits, t_plain, A);
    if (rc) return rc;
    if (n == 0) return DPFHE_OK;
    CHECK_PTR(d_sk); CHECK_PTR(d_cct); CHECK_PTR(d_pt);
    const size_t N = ctx->N();
    if (overlaps(d_pt, n * N * 8, d_sk, N * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the secret");
    if (overlaps(d_pt, n * N * 8, d_cct, n * 2 * A.tiles * bits * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap an input");
    const size_t pairs = (n + 1) / 2;
    rc = ctx->compact_work.reserve(ctx, 2 * pairs * N * 8);
    if (rc) return rc;
    u64 *rows = ctx->compact_work.get();
    cudaStream_t st = pick(ctx, stream);
    const LaunchCtx lc1 = level_view(ctx, 1);
    if (n & 1) CU_TRY(cudaMemsetAsync(rows + n * N, 0, N * 8, st));
    CU_TRY(VCALL(launch_compact_unpack, lc1, false, A, d_cct, nullptr, rows, n, st));
    CU_TRY(VCALL(launch_ntt, lc1, rows, n, false, st));
    CU_TRY(VCALL(launch_ct_mul_plain, lc1, rows, d_sk, rows, pairs, st));
    CU_TRY(VCALL(launch_ntt, lc1, rows, n, true, st));
    CU_TRY(VCALL(launch_compact_unpack, lc1, true, A, d_cct, rows, d_pt, n, st));
    CU_TRY(VCALL(launch_ntt, lc1, d_pt, n, false, st));
    note_launch(ctx, 6);
    return DPFHE_OK;
}

int dpfhe_decrypt_compact(dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, const uint64_t *d_sk, const uint64_t *d_cct, uint64_t *d_pt,
                          size_t n, void *stream) {
    return decrypt_compact_at(ctx, bits, t_plain, d_sk, d_cct, d_pt, n, stream);
}

// row 0 of the secret is the staged shared operand
int dpfhe_decrypt_compact_host(dpfhe_ctx *ctx, unsigned bits, uint64_t t_plain, const uint64_t *h_sk, const uint64_t *h_cct,
                               uint64_t *h_pt, size_t n) {
    int rc = enter(ctx);
    if (rc) return rc;
    CompactArgs A;
    rc = compact_args(ctx, bits, t_plain, A);
    if (rc || n == 0) return rc;
    const size_t N = ctx->N();
    return host_call(ctx, {h_sk, h_cct, h_pt}, h_sk, N, h_cct, nullptr, h_pt, n, 2 * (size_t)A.tiles * bits, N,
                     [&](u64 *din, u64 *, u64 *dout, size_t cnt, cudaStream_t st) {
                         return decrypt_compact_at(ctx, bits, t_plain, ctx->stage_key.get(), din, dout, cnt, st);
                     });
}

#undef CHECK_SEED

// waits for everything this context has in flight, whatever stream it was issued on
int dpfhe_synchronize(dpfhe_ctx *ctx) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (ctx->have_last) CU_TRY(cudaEventSynchronize(ctx->ev_last));
    CU_TRY(cudaStreamSynchronize(ctx->stream));
    CU_TRY(cudaStreamSynchronize(ctx->s_h2d));
    CU_TRY(cudaStreamSynchronize(ctx->s_d2h));
    return DPFHE_OK;
}

int dpfhe_device_count(int *out) {
    if (!out) return fail(DPFHE_ERR_INVALID, "null argument");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    *out = e == cudaSuccess ? n : 0;
    if (e != cudaSuccess) return fail(DPFHE_ERR_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    return DPFHE_OK;
}

int dpfhe_context_device(const dpfhe_ctx *ctx) { return ctx ? ctx->lc.device : -1; }

// rotation by k slots (k may be negative): the Galois element is 5^k mod 2N (DESIGN.md 2.8)
int dpfhe_galois_element(const dpfhe_ctx *ctx, int k, uint64_t *galois_elt) {
    if (!ctx || !galois_elt) return fail(DPFHE_ERR_INVALID, "null argument");
    const uint64_t two_n = (uint64_t)2 << ctx->hp.log_n, order = two_n / 4;   // 5 has order N/2 in Z_2N^*
    uint64_t e = (uint64_t)(((long long)k % (long long)order + (long long)order) % (long long)order), g = 1, b = 5;
    for (; e; e >>= 1) {
        if (e & 1) g = g * b % two_n;
        b = b * b % two_n;
    }
    *galois_elt = g;
    return DPFHE_OK;
}
int dpfhe_rotate_steps(dpfhe_ctx *ctx, const uint64_t *d_ct, int k, const uint64_t *d_gk, uint64_t *d_out, size_t batch, void *stream) {
    uint64_t g = 0;
    int rc = dpfhe_galois_element(ctx, k, &g);
    if (rc) return rc;
    return dpfhe_rotate(ctx, d_ct, g, d_gk, d_out, batch, stream);
}

// ---------------------------------------------------------------- device memory that other processes / devices can map
int dpfhe_device_alloc(dpfhe_ctx *ctx, void **d_out, size_t bytes) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!d_out) return fail(DPFHE_ERR_INVALID, "null argument");
    *d_out = nullptr;
    CU_TRY(cudaMalloc(d_out, bytes));   // a whole allocation of its own, so that an IPC handle maps exactly this buffer
    return DPFHE_OK;
}
int dpfhe_device_free(dpfhe_ctx *ctx, void *d_ptr) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (d_ptr) CU_TRY(cudaFree(d_ptr));
    return DPFHE_OK;
}
int dpfhe_ipc_export(dpfhe_ctx *ctx, const void *d_ptr, unsigned char handle[DPFHE_IPC_HANDLE_BYTES]) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!d_ptr || !handle) return fail(DPFHE_ERR_INVALID, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == DPFHE_IPC_HANDLE_BYTES, "handle size");
    cudaIpcMemHandle_t h;
    CU_TRY(cudaIpcGetMemHandle(&h, const_cast<void *>(d_ptr)));
    memcpy(handle, &h, sizeof(h));
    return DPFHE_OK;
}
int dpfhe_ipc_open(dpfhe_ctx *ctx, const unsigned char handle[DPFHE_IPC_HANDLE_BYTES], void **d_out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!handle || !d_out) return fail(DPFHE_ERR_INVALID, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    *d_out = nullptr;
    CU_TRY(cudaIpcOpenMemHandle(d_out, h, cudaIpcMemLazyEnablePeerAccess));   // maps the peer's buffer into this context's device
    return DPFHE_OK;
}
int dpfhe_ipc_close(dpfhe_ctx *ctx, void *d_ptr) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (d_ptr) CU_TRY(cudaIpcCloseMemHandle(d_ptr));
    return DPFHE_OK;
}

// Diagnostics (not part of the drop-in surface): sums the fused kernel's per-phase clock64 counters over
// all CTAs into out[16] and clears them.  Only available when the context was created with DPFHE_KS_PROF set.
int dpfhe_debug_phase_cycles(dpfhe_ctx *ctx, uint64_t *out16) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out16 || !ctx->lc.ks_prof) return fail(DPFHE_ERR_INVALID, "phase profiling is not enabled (DPFHE_KS_PROF)");
    std::vector<unsigned long long> h(ctx->lc.ks_slots * 16);
    CU_TRY(cudaDeviceSynchronize());
    CU_TRY(cudaMemcpy(h.data(), ctx->lc.ks_prof, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CU_TRY(cudaMemset(ctx->lc.ks_prof, 0, h.size() * sizeof(unsigned long long)));
    for (int k = 0; k < 16; ++k) out16[k] = 0;
    for (size_t s = 0; s < ctx->lc.ks_slots; ++s)
        for (int k = 0; k < 16; ++k) out16[k] += h[s * 16 + k];
    out16[11] = out16[12] = out16[13] = 0;   // [11] = CTAs that ran (the launched grid); [12] = min, [13] = max CTA lifetime (ns)
    for (size_t s = 0; s < ctx->lc.ks_slots; ++s) {
        const uint64_t ns = h[s * 16 + 14];
        if (!ns) continue;
        ++out16[11];
        if (ns > out16[13]) out16[13] = ns;
        if (!out16[12] || ns < out16[12]) out16[12] = ns;
    }
    return DPFHE_OK;
}

// ---------------------------------------------------------------- encrypted linear layer (SURVEY.md §8 row f-4, BASELINE config 4)
// y = sum_g rot_{g*baby}( sum_b D[g*baby + b] o rot_b(x) ): baby-step/giant-step diagonals on top of the hot-path ops.
// The weights (diagonal plaintexts) and Galois keys are uploaded ONCE when the layer is created; an application is
//   baby-1 hoisted rotations of the input (one shared digit decomposition)  -> dpfhe_rotate_hoisted
//   all giant-step inner sums in one pass over the baby steps               -> dpfhe_ct_mul_plain_inner
//   Horner over the giant steps: acc = rot_baby(acc) + inner[g]              -> dpfhe_rotate + dpfhe_poly_add
// and the host-buffer form pipelines chunks of the batch through it (upload / compute / download overlapped).
// With grouped special-prime keys (dpfhe_linear_create_grouped, ciphertexts of Lq = L - K limbs) the baby steps are hoisted
// grouped rotations with companions prepared at creation, the inner sums run on an Lq-limb view of the context, and every
// Horner step is ONE launch: the grouped rotation adds inner[g] in its final store (ks_grouped_kernel<..., ADD>).
struct dpfhe_linear {
    static constexpr const char *what = "null layer";
    dpfhe_ctx *const ctx;
    size_t baby = 0, giant = 0;
    unsigned n_special = 0;                 // 0: per-limb-digit keys; K > 0: grouped keys with K special primes
    size_t Lq = 0;                          // limbs of a ciphertext polynomial: L, or L - K with grouped keys, or the level
    unsigned level = 0;                     // grouped keys below the top level (DESIGN.md §2.21): Lq = level < L - K; 0 at the top
    u64 *d_diags = nullptr;                 // [n][Lq][N]
    std::vector<uint64_t> g_baby;           // Galois elements 5^b, b = 1 .. baby-1
    uint64_t g_giant = 0;
    // per-limb-digit keys
    u64 *d_keys = nullptr;                  // [baby-1 + 1][L][2][L][N]: baby-step keys, then the giant-step key
    std::vector<const uint64_t *> k_baby;   // device pointers of the baby-step keys
    u64 *d_prep = nullptr;                  // per baby step: Shoup companions of its key [L][2][L][N] + kprime [2][L][N], built once
    std::vector<const uint64_t *> prep;     // {companions, kprime} pointers per baby step (rotate_hoisted_impl)
    // grouped keys
    PreparedKeys gk;                        // baby-step keys, then the giant-step key when there are giant steps to rotate (giant > 1)
    uint64_t t_plain = 0;                   // plaintext modulus of the divisions by P (0: plain rounding)
    MsConsts K;                             // constants of the division by P
    GroupConsts G;
    DeviceScratch scratch;                  // [baby + giant + 1][batch][2][Lq][N] for the largest batch applied so far; like the rest of
                                            //   the layer, not counted in the context's device bytes

    explicit dpfhe_linear(dpfhe_ctx *c) : ctx(c) {}
    ~dpfhe_linear() {
        cudaFree(d_diags);
        cudaFree(d_keys);
        cudaFree(d_prep);
        gk.release();
    }
    size_t in_words() const { return 2 * Lq * ctx->N(); }
    size_t out_words() const { return in_words(); }
    int reserve(size_t batch) { return scratch.reserve(ctx, (baby + giant + 1) * batch * in_words() * 8); }
    size_t host_chunk(size_t batch) const { return grid_round_chunk(ctx, batch, "DPFHE_LINEAR_CHUNK_ROUNDS"); }
    int apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
    int apply_grouped_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
};

static int linear_check_shape(size_t n_diags, size_t baby, const uint64_t *h_gk_baby, const uint64_t *h_gk_giant) {
    if (baby == 0 || baby > 128 || n_diags == 0 || n_diags % baby) return fail(DPFHE_ERR_INVALID, "need 1 <= baby <= 128 and a multiple of baby diagonals");
    const size_t giant = n_diags / baby;
    if (giant > 65535) return fail(DPFHE_ERR_INVALID, "too many giant steps");
    if ((baby > 1 && !h_gk_baby) || (giant > 1 && !h_gk_giant)) return fail(DPFHE_ERR_INVALID, "missing Galois keys");
    return DPFHE_OK;
}

// The start of both constructors: a layer with its diagonals on the device, and the Galois elements of its rotations.
// level: the layer's level below the top (its diagonals have `level` rows), 0 at the top.
static int linear_new(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const uint64_t *h_diags, size_t n_diags, size_t baby, dpfhe_linear **out,
                      unsigned level = 0) {
    dpfhe_linear *lin = new (std::nothrow) dpfhe_linear(ctx);
    if (!lin) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    lin->baby = baby; lin->giant = n_diags / baby; lin->n_special = n_special; lin->Lq = level ? level : ctx->hp.L - n_special; lin->t_plain = t_plain;
    lin->level = level;
    const size_t diag_bytes = n_diags * lin->Lq * ctx->N() * 8;
    cudaError_t e = cudaMalloc(&lin->d_diags, diag_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(lin->d_diags, h_diags, diag_bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        delete lin;
        return fail(DPFHE_ERR_CUDA, "linear layer upload: %s", cudaGetErrorString(e));
    }
    for (size_t b = 1; b < baby; ++b) {
        uint64_t g = 0;
        dpfhe_galois_element(ctx, (int)b, &g);
        lin->g_baby.push_back(g);
    }
    dpfhe_galois_element(ctx, (int)baby, &lin->g_giant);
    *out = lin;
    return DPFHE_OK;
}

// copies a layer's keys of key_words words each to d_keys: the baby-step keys, then the giant-step key if the layer rotates by it
static cudaError_t linear_upload_keys(const dpfhe_linear *lin, u64 *d_keys, size_t key_words, const uint64_t *h_gk_baby, const uint64_t *h_gk_giant) {
    cudaError_t e = cudaSuccess;
    if (lin->baby > 1) e = cudaMemcpy(d_keys, h_gk_baby, (lin->baby - 1) * key_words * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && lin->giant > 1) e = cudaMemcpy(d_keys + (lin->baby - 1) * key_words, h_gk_giant, key_words * 8, cudaMemcpyHostToDevice);
    return e;
}

int dpfhe_linear_create(dpfhe_ctx *ctx, const uint64_t *h_diags, size_t n_diags, size_t baby, const uint64_t *h_gk_baby, const uint64_t *h_gk_giant,
                        dpfhe_linear **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !h_diags) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    rc = linear_check_shape(n_diags, baby, h_gk_baby, h_gk_giant);
    if (rc) return rc;
    dpfhe_linear *lin = nullptr;
    rc = linear_new(ctx, 0, 0, h_diags, n_diags, baby, &lin);
    if (rc) return rc;
    cudaStream_t st = pick(ctx, nullptr);
    const size_t key_words = 2 * ctx->hp.L * ctx->P(), kp_words = 2 * ctx->P();
    cudaError_t e = cudaMalloc(&lin->d_keys, baby * key_words * 8);
    if (e == cudaSuccess) e = linear_upload_keys(lin, lin->d_keys, key_words, h_gk_baby, h_gk_giant);
    if (e != cudaSuccess) return object_finish(lin, fail(DPFHE_ERR_CUDA, "linear layer upload: %s", cudaGetErrorString(e)), st, nullptr, out);
    // the constants of the baby-step rotations do not depend on the data: prepare them once (four small launches per rotation
    // that every hoisted call would otherwise repeat — a tenth of a 31-rotation call at batch 512, more for smaller chunks)
    if (baby > 1) {
        e = ensure_hoist_consts(ctx) == DPFHE_OK ? cudaMalloc(&lin->d_prep, (baby - 1) * (key_words + kp_words) * 8) : cudaErrorMemoryAllocation;
        for (size_t b = 1; b < baby && e == cudaSuccess; ++b) {
            u64 *ks = lin->d_prep + (b - 1) * (key_words + kp_words), *kp = ks + key_words;
            lin->k_baby.push_back(lin->d_keys + (b - 1) * key_words);
            e = VCALL(launch_rot_prepare, ctx->lc, lin->k_baby[b - 1], (u32)lin->g_baby[b - 1], ctx->hoist_delta.get(), ctx->hoist_M.get(), kp, st, ks);
            note_launch(ctx, 4);
            lin->prep.push_back(ks);
            lin->prep.push_back(kp);
        }
    }
    rc = e == cudaSuccess ? DPFHE_OK : fail(DPFHE_ERR_CUDA, "linear layer constants: %s", cudaGetErrorString(e));
    return object_finish(lin, rc, st, "linear layer constants", out);
}

// the grouped layer once its arguments are checked; level: below the top level (DESIGN.md §2.21), 0 at the top.  A level layer builds
// the level's state here, so that its first application allocates no level tables; its keys and their companions are the top-level
// ones, which serve every level.
static int linear_grouped_new(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *h_diags, size_t n_diags, size_t baby,
                              const uint64_t *h_gk_baby, const uint64_t *h_gk_giant, uint64_t t_plain, dpfhe_linear **out) {
    const KsLevel *lv = nullptr;
    int rc = level ? level_state(ctx, n_special, level, lv) : DPFHE_OK;
    if (rc) return rc;
    dpfhe_linear *lin = nullptr;
    rc = linear_new(ctx, n_special, t_plain, h_diags, n_diags, baby, &lin, level);
    if (rc) return rc;
    build_group_consts(lv ? lv->hp : ctx->hp, n_special, t_plain, lin->G, lin->K);
    rc = lin->giant > 1 ? ensure_hyb(ctx) : DPFHE_OK;   // the special-prime rows of the giant steps' kernel
    cudaStream_t st = pick(ctx, nullptr);
    // the Shoup companions of every key, once: each application would otherwise rebuild them for every rotation
    const size_t dnum = key_digits(ctx, n_special);
    if (rc == DPFHE_OK)
        rc = prepare_keys(ctx, ctx->lc, baby - 1 + (lin->giant > 1), dnum, st, "linear layer keys",
                          [&](u64 *d_keys) { return linear_upload_keys(lin, d_keys, dnum * 2 * ctx->P(), h_gk_baby, h_gk_giant); }, lin->gk);
    return object_finish(lin, rc, st, "linear layer constants", out);
}

int dpfhe_linear_create_grouped(dpfhe_ctx *ctx, unsigned n_special, const uint64_t *h_diags, size_t n_diags, size_t baby,
                                const uint64_t *h_gk_baby, const uint64_t *h_gk_giant, uint64_t t_plain, dpfhe_linear **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !h_diags) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    rc = linear_check_shape(n_diags, baby, h_gk_baby, h_gk_giant);
    if (rc) return rc;
    return linear_grouped_new(ctx, n_special, 0, h_diags, n_diags, baby, h_gk_baby, h_gk_giant, t_plain, out);
}

// the grouped layer at level l (DESIGN.md §2.21): the checks of dpfhe_linear_create_grouped, then the level's; l = Lq is that call
int dpfhe_linear_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const uint64_t *h_diags, size_t n_diags, size_t baby,
                                      const uint64_t *h_gk_baby, const uint64_t *h_gk_giant, uint64_t t_plain, dpfhe_linear **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !h_diags) return fail(DPFHE_ERR_INVALID, "level %u: null argument", level);
    *out = nullptr;
    rc = check_grouped(ctx, n_special, t_plain);
    if (!rc) rc = check_level(ctx, n_special, level, false, t_plain);
    if (!rc) rc = linear_check_shape(n_diags, baby, h_gk_baby, h_gk_giant);
    if (rc) return rc;
    return linear_grouped_new(ctx, n_special, level == ctx->hp.L - n_special ? 0 : level, h_diags, n_diags, baby, h_gk_baby, h_gk_giant, t_plain, out);
}

void dpfhe_linear_destroy(dpfhe_linear *lin) { object_destroy(lin); }

// grouped keys: hoisted baby steps, the inner sums on the ciphertext moduli, giant - 1 fused Horner steps.  Launches per application
// (a batch within one chunk of the hoisted-rotation scratch): [baby > 1] * (1 + 3 (baby-1)) + ceil(giant / gmax(baby)) + (giant - 1),
// gmax = the giant steps one inner-product launch holds; the same at a level.  A level layer looks its level's state up at every
// application rather than keeping it: dpfhe_context_trim frees it (the lookup then builds it again).
int dpfhe_linear::apply_grouped_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    const KsLevel *lv = nullptr;
    int rc = level ? level_state(ctx, n_special, level, lv) : DPFHE_OK;
    if (rc) return rc;
    const size_t ctb = batch * in_words();                      // words of one ciphertext batch
    u64 *steps = scratch.get(), *inner = steps + baby * ctb, *tmp = inner + giant * ctb;
    cudaStream_t st = pick(ctx, stream);
    CU_TRY(cudaMemcpyAsync(steps, d_ct, ctb * 8, cudaMemcpyDeviceToDevice, st));
    if (baby > 1)
        rc = rotate_hoisted_grouped_impl(ctx, n_special, steps, baby - 1, g_baby.data(), gk.keys.data(), gk.key_s.data(), steps + ctb, batch, t_plain,
                                         stream, lv);
    if (rc) return rc;
    // every inner sum in one pass, on the ciphertext moduli
    st = pick(ctx, stream);
    const LaunchCtx lcq = level_view(ctx, (unsigned)Lq);
    unsigned launches = 0;
    CU_TRY(VCALL(launch_pt_inner, lcq, steps, (u32)baby, d_diags, (u32)giant, inner, batch, st, &launches));
    note_launch(ctx, launches);
    if (giant == 1) {
        CU_TRY(cudaMemcpyAsync(d_out, inner, ctb * 8, cudaMemcpyDeviceToDevice, st));
        return DPFHE_OK;
    }
    // Horner: acc = rot_baby(acc) + inner[g], one launch per step.  The output may not alias the rotated input or the addend: the
    // steps alternate between tmp and d_out so that the last one (g = 0) writes d_out.
    const u64 *acc = inner + (giant - 1) * ctb;
    for (size_t g = giant - 1; g-- > 0;) {
        u64 *dst = g % 2 == 0 ? d_out : tmp;
        if (lv)
            CU_TRY(on_level_view(ctx, *lv, [&](LaunchCtx &lc) {
                return VCALL(launch_ks_grouped_level, lc, KS_ROTATE, &acc, nullptr, 1, gk.keys[baby - 1], gk.key_s[baby - 1], (u32)ctx->hp.L, dst, batch,
                             (u32)g_giant, K, G, nullptr, st, inner + g * ctb);
            }));
        else
            CU_TRY(VCALL(launch_ks_grouped, ctx->lc, KS_ROTATE, acc, nullptr, gk.keys[baby - 1], dst, batch, (u32)g_giant, K, G, st, inner + g * ctb,
                         gk.key_s[baby - 1]));
        note_launch(ctx, 1);
        acc = dst;
    }
    return DPFHE_OK;
}

int dpfhe_linear::apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    if (n_special) return apply_grouped_on(d_ct, d_out, batch, stream);
    const size_t ctb = batch * in_words();                      // words of one ciphertext batch
    u64 *steps = scratch.get(), *inner = steps + baby * ctb, *tmp = inner + giant * ctb;
    cudaStream_t st = pick(ctx, stream);
    CU_TRY(cudaMemcpyAsync(steps, d_ct, ctb * 8, cudaMemcpyDeviceToDevice, st));
    int rc = DPFHE_OK;
    if (baby > 1) rc = rotate_hoisted_impl(ctx, steps, baby - 1, g_baby.data(), k_baby.data(), prep.data(), steps + ctb, batch, stream);
    if (rc) return rc;
    rc = dpfhe_ct_mul_plain_inner(ctx, steps, baby, d_diags, giant, inner, batch, stream);
    if (rc) return rc;
    st = pick(ctx, stream);
    CU_TRY(cudaMemcpyAsync(d_out, inner + (giant - 1) * ctb, ctb * 8, cudaMemcpyDeviceToDevice, st));
    const u64 *gk_giant = d_keys + (baby - 1) * 2 * ctx->hp.L * ctx->P();
    for (size_t g = giant - 1; g-- > 0;) {
        rc = dpfhe_rotate(ctx, d_out, g_giant, gk_giant, tmp, batch, stream);           // Horner step: acc = rot_baby(acc) + inner[g]
        if (rc) return rc;
        rc = dpfhe_poly_add(ctx, tmp, inner + g * ctb, d_out, 2 * batch, stream);
        if (rc) return rc;
    }
    return DPFHE_OK;
}

int dpfhe_linear_apply(dpfhe_linear *lin, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    return object_apply(lin, d_ct, d_out, batch, stream);
}

int dpfhe_linear_apply_host(dpfhe_linear *lin, const uint64_t *h_ct, uint64_t *h_out, size_t batch) { return object_apply_host(lin, h_ct, h_out, batch); }

// ---------------------------------------------------------------- scalar linear combinations, BGV polynomial evaluation (DESIGN.md §2.15)
// on the prefix of L limbs (DESIGN.md §2.22); L = hp.L is dpfhe_ct_lincomb
static int ct_lincomb_at(dpfhe_ctx *ctx, unsigned L, size_t n_terms, const uint64_t *const *d_cts, const int64_t *coeffs, int64_t constant,
                         uint64_t *d_out, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (n_terms < 1 || n_terms > (size_t)LINCOMB_MAX_TERMS) return fail(DPFHE_ERR_INVALID, "n_terms must be in [1, %d]", LINCOMB_MAX_TERMS);
    if (!d_cts || !coeffs) return fail(DPFHE_ERR_INVALID, "null argument");
    for (size_t i = 0; i < n_terms; ++i)
        if (!d_cts[i] || !aligned16(d_cts[i])) return fail(DPFHE_ERR_INVALID, "null or misaligned input ciphertext %zu", i);
    CHECK_PTR(d_out);
    if (batch == 0) return DPFHE_OK;
    // the output may BE an input (a thread reads chunk c of every input, then writes chunk c), but not overlap one at another offset
    const size_t ct_bytes = batch * 2 * L * ctx->N() * 8;
    for (size_t i = 0; i < n_terms; ++i)
        if (d_out != d_cts[i] && overlaps(d_out, ct_bytes, d_cts[i], ct_bytes))
            return fail(DPFHE_ERR_INVALID, "output must be an input or not overlap it (input %zu)", i);
    CU_TRY(VCALL(launch_lincomb, level_view(ctx, L), d_cts, coeffs, (u32)n_terms, constant, nullptr, d_out, batch, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_ct_lincomb(dpfhe_ctx *ctx, size_t n_terms, const uint64_t *const *d_cts, const int64_t *coeffs, int64_t constant, uint64_t *d_out,
                     size_t batch, void *stream) {
    return ct_lincomb_at(ctx, ctx ? ctx->hp.L : 0, n_terms, d_cts, coeffs, constant, d_out, batch, stream);
}

// the linear-combination body with one term of coefficient 1 and the plaintext as the c0 addend; on the prefix of L limbs
// (DESIGN.md §2.22), L = hp.L is dpfhe_ct_add_plain
static int ct_add_plain_at(dpfhe_ctx *ctx, unsigned L, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch, void *stream) {
    int rc = enter(ctx);
    if (rc) return rc;
    CHECK_PTR(d_ct); CHECK_PTR(d_pt); CHECK_PTR(d_out);
    if (batch == 0) return DPFHE_OK;
    const size_t P = L * ctx->N();
    if (overlaps(d_out, batch * 2 * P * 8, d_pt, P * 8)) return fail(DPFHE_ERR_INVALID, "output must not overlap the plaintext");
    if (overlaps_shifted(d_out, d_ct, batch * 2 * P * 8)) return fail(DPFHE_ERR_INVALID, "output must be the input or not overlap it");
    const int64_t one = 1;
    CU_TRY(VCALL(launch_lincomb, level_view(ctx, L), &d_ct, &one, 1u, (int64_t)0, d_pt, d_out, batch, pick(ctx, stream)));
    note_launch(ctx, 1);
    return DPFHE_OK;
}
int dpfhe_ct_add_plain(dpfhe_ctx *ctx, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch, void *stream) {
    return ct_add_plain_at(ctx, ctx ? ctx->hp.L : 0, d_ct, d_pt, d_out, batch, stream);
}

// at level l (DESIGN.md §2.22), as the keyless level calls above
int dpfhe_ct_lincomb_level(dpfhe_ctx *ctx, unsigned level, size_t n_terms, const uint64_t *const *d_cts, const int64_t *coeffs, int64_t constant,
                           uint64_t *d_out, size_t batch, void *stream) {
    return prefix_call(ctx, level, [&] { return ct_lincomb_at(ctx, level, n_terms, d_cts, coeffs, constant, d_out, batch, stream); });
}
int dpfhe_ct_add_plain_level(dpfhe_ctx *ctx, unsigned level, const uint64_t *d_ct, const uint64_t *d_pt, uint64_t *d_out, size_t batch,
                             void *stream) {
    return prefix_call(ctx, level, [&] { return ct_add_plain_at(ctx, level, d_ct, d_pt, d_out, batch, stream); });
}

// host buffers: the plaintext uploaded once, the batch pipelined in chunks (as dpfhe_ct_mul_plain_host)
int dpfhe_ct_add_plain_host(dpfhe_ctx *ctx, const uint64_t *h_ct, const uint64_t *h_pt, uint64_t *h_out, size_t batch) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (batch == 0) return DPFHE_OK;
    const size_t P = ctx->P();
    const int64_t one = 1;
    return host_call(ctx, {h_ct, h_pt, h_out}, h_pt, P, h_ct, nullptr, h_out, batch, 2 * P, 2 * P,
                     [&](u64 *dc, u64 *, u64 *dout, size_t cnt, cudaStream_t st) -> int {
                         const u64 *in = dc;
                         CU_TRY(VCALL(launch_lincomb, ctx->lc, &in, &one, 1u, (int64_t)0, ctx->stage_key.get(), dout, cnt, st));
                         note_launch(ctx, 1);
                         return DPFHE_OK;
                     });
}

namespace {

// x^-1 mod m for gcd(x, m) = 1 (m < 2^31)
uint64_t inv_mod(uint64_t x, uint64_t m) {
    int64_t a = (int64_t)(x % m), b = (int64_t)m, u = 1, v = 0;
    while (b) {
        const int64_t q = a / b;
        a -= q * b; std::swap(a, b);
        u -= q * v; std::swap(u, v);
    }
    return (uint64_t)((u % (int64_t)m + (int64_t)m) % (int64_t)m);
}
int64_t centred(uint64_t x, uint64_t t) { return x <= t / 2 ? (int64_t)x : (int64_t)x - (int64_t)t; }
unsigned ceil_log2(size_t k) {
    unsigned j = 0;
    while (((size_t)1 << j) < k) ++j;
    return j;
}

// key switching at level l: the basis {q_0 .. q_{l-1}, p_0 .. p_{K-1}}, its device tables (the context's own at the top level), the
// level's key restricted from the top-level key and its Shoup companions
struct PeLevel {
    unsigned l = 0;
    HostParams hp;
    LimbParams *d_lp = nullptr;
    Twiddle *d_tw = nullptr, *d_itw = nullptr;
    LimbTable lt;
    bool lift_reduce = true;
    MsConsts K;
    GroupConsts G;
    PreparedKeys key;   // one key: key.keys[0], key.key_s[0]
};

// one step of an application.  Buffers: >= 0 an entry of bufs, IN the input, OUT the output
enum PeOpKind { PE_MUL = 0, PE_SWITCH = 1, PE_LINCOMB = 2, PE_CUT = 3, PE_CKKS_COMB = 4 };
constexpr int PE_IN = -1, PE_OUT = -2;
struct PeOp {
    int kind;
    unsigned level;           // PE_MUL: level of the product; PE_SWITCH: level of the input (drops q_{level-1}); PE_LINCOMB: its level;
                              // PE_CUT: level of the copy (the first `level` rows of each polynomial of a); PE_CKKS_COMB: Lc
    int a, b, out;            // PE_CUT: b is the level of a
    std::vector<int> terms;   // PE_LINCOMB, PE_CKKS_COMB
    std::vector<int64_t> coeffs;
    int64_t constant = 0;
    std::vector<unsigned> levels;   // PE_CKKS_COMB: the level of every term (>= Lc; rows below Lc are read)
    std::vector<double> dcoeffs;    // PE_CKKS_COMB: the integer-valued doubles c_k and c_0
    double dconstant = 0;
};

}  // namespace

struct dpfhe_polyeval {
    static constexpr const char *what = "null evaluator";
    dpfhe_ctx *const ctx;
    unsigned K = 0, Lq = 0, Lf = 0;      // Lq: the level the evaluator starts from (its input's limbs; DESIGN.md §2.22), Lf: the result's
    unsigned Lk = 0;                     // the context's L - K: the row of the first special prime in the top-level key, and the level
                                         //   whose tables are the context's own
    uint64_t t = 0;
    std::vector<PeLevel> lev;            // by level: lev[l - lev_lo]
    unsigned lev_lo = 0;
    std::vector<MsConsts> ms;            // modulus switch dropping q_{l-1} (BGV; CKKS: t = 0): ms[l]
    bool ckks = false;                   // DESIGN.md §2.16: Lf is then the result's level Lc - 1
    double scale_out = 0;                // CKKS: the scale S of the result
    std::vector<PeOp> ops;
    std::vector<unsigned> bufs;          // level of every scratch buffer
    CountedScratch mem;                  // counts the level tables and keys; its scratch: the buffers back to back, then the switch's
                                         //   tau rows [2 batch][N], for the largest batch so far

    explicit dpfhe_polyeval(dpfhe_ctx *c) : ctx(c), mem(c) {}
    ~dpfhe_polyeval() {
        for (auto &v : lev) {
            if (v.l != Lk) {   // the top level's tables are the context's
                cudaFree(v.d_lp);
                cudaFree(v.d_tw);
                cudaFree(v.d_itw);
            }
            v.key.release();
        }
    }
    size_t in_words() const { return 2 * Lq * ctx->N(); }
    size_t out_words() const { return 2 * Lf * ctx->N(); }
    int reserve(size_t batch) {
        size_t w = bufs.empty() && !ckks ? 0 : 2 * batch * ctx->N();
        for (unsigned l : bufs) w += batch * 2 * l * ctx->N();
        return mem.reserve(w * 8);
    }
    size_t host_chunk(size_t batch) const { return item_chunk(ctx, batch, "DPFHE_POLYEVAL_CHUNK"); }
    int apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
};

namespace {

// the schedule of DESIGN.md §2.15: powers in increasing order, each operand brought to the product's level by single-limb switches
// (each copy made once, from the copy one level above), the combination one level above the last switch
int pe_plan(dpfhe_polyeval *pe, const int64_t *coeffs, size_t d) {
    const unsigned Lq = pe->Lq, D = ceil_log2(d);
    const uint64_t t = pe->t;
    std::vector<uint64_t> a(d + 1), qinv(Lq);
    for (size_t k = 0; k <= d; ++k) a[k] = floor_mod(coeffs[k], t);
    for (unsigned i = 0; i < Lq; ++i) qinv[i] = inv_mod(pe->ctx->hp.limbs[i].lp.q % t, t);
    if (D == 0) {
        PeOp op{PE_LINCOMB, Lq, 0, 0, PE_OUT};
        op.terms = {PE_IN};
        op.coeffs = {centred(a[1], t)};
        op.constant = centred(a[0], t);
        pe->ops.push_back(op);
        return DPFHE_OK;
    }
    const unsigned Lf = Lq - D;
    // powers needed: every k with a_k != 0 and, recursively, the operands of their products (x alone if every a_k, k >= 1, is 0)
    std::vector<char> need(d + 1, 0);
    bool any = false;
    for (size_t k = 1; k <= d; ++k) any |= (need[k] = a[k] != 0);
    if (!any) need[1] = 1;
    auto split = [](size_t k, size_t &u, size_t &v) {
        size_t p = 1;
        while (2 * p < k) p *= 2;
        u = p;
        v = k - p;   // = p when k is a power of two
    };
    for (size_t k = d; k >= 2; --k)
        if (need[k]) {
            size_t u, v;
            split(k, u, v);
            need[u] = need[v] = 1;
        }
    // copies of the powers by level, with their factors
    std::vector<std::vector<int>> at(d + 1, std::vector<int>(Lq + 1, -3));
    std::vector<std::vector<uint64_t>> fac(d + 1, std::vector<uint64_t>(Lq + 1, 0));
    std::vector<int> ybuf(d + 1, -3);
    std::vector<uint64_t> yfac(d + 1, 0);
    at[1][Lq] = PE_IN;
    fac[1][Lq] = 1;
    auto new_buf = [&](unsigned l) {
        pe->bufs.push_back(l);
        return (int)pe->bufs.size() - 1;
    };
    int tmp = -3;   // the product of a power that is switched right away: one buffer at the top level, reused
    std::function<void(size_t, unsigned)> get = [&](size_t k, unsigned l) {
        if (at[k][l] != -3) return;
        get(k, l + 1);
        const int b = new_buf(l);
        pe->ops.push_back(PeOp{PE_SWITCH, l + 1, at[k][l + 1], 0, b});
        at[k][l] = b;
        fac[k][l] = fac[k][l + 1] * qinv[l] % t;
    };
    for (size_t k = 2; k <= d; ++k) {
        if (!need[k]) continue;
        size_t u, v;
        split(k, u, v);
        const unsigned ck = ceil_log2(k), l = Lq - ck + 1;
        get(u, l);
        get(v, l);
        const uint64_t f = fac[u][l] * fac[v][l] % t;
        if (ck == D) {
            ybuf[k] = new_buf(l);
            yfac[k] = f;
            pe->ops.push_back(PeOp{PE_MUL, l, at[u][l], at[v][l], ybuf[k]});
        } else {
            if (tmp == -3) tmp = new_buf(Lq);
            pe->ops.push_back(PeOp{PE_MUL, l, at[u][l], at[v][l], tmp});
            const int b = new_buf(l - 1);
            pe->ops.push_back(PeOp{PE_SWITCH, l, tmp, 0, b});
            at[k][l - 1] = b;
            fac[k][l - 1] = f * qinv[l - 1] % t;
        }
    }
    const uint64_t G = pe->ctx->hp.limbs[Lf].lp.q % t;
    if (tmp == -3) tmp = new_buf(Lf + 1);
    PeOp lc{PE_LINCOMB, Lf + 1, 0, 0, tmp};
    for (size_t k = 1; k <= d; ++k) {
        if (any ? a[k] == 0 : k != 1) continue;
        uint64_t g;
        if (ceil_log2(k) == D) {   // the pre-switch product, at Lf + 1 already
            lc.terms.push_back(ybuf[k]);
            g = yfac[k];
        } else {
            get(k, Lf + 1);
            lc.terms.push_back(at[k][Lf + 1]);
            g = fac[k][Lf + 1];
        }
        lc.coeffs.push_back(centred(a[k] * inv_mod(g, t) % t * G % t, t));
    }
    lc.constant = centred(a[0] * G % t, t);
    pe->ops.push_back(lc);
    pe->ops.push_back(PeOp{PE_SWITCH, Lf + 1, tmp, 0, PE_OUT});
    return DPFHE_OK;
}

// the schedule of DESIGN.md §2.16: the powers of §2.15, each product rescaled right away (x^k at level Lq - ceil(log2 k)), an operand
// above a product's level cut to its first rows (each cut made once per power and level), the scales tracked in doubles, and the
// combination over the prefixes at Lc = Lq - D fused into the final rescale
int pe_plan_ckks(dpfhe_polyeval *pe, const double *a, size_t d, double scale_in) {
    const unsigned Lq = pe->Lq, D = ceil_log2(d), Lc = Lq - D;
    const HostParams &hp = pe->ctx->hp;
    std::vector<char> need(d + 1, 0);
    bool any = false;
    for (size_t k = 1; k <= d; ++k) any |= (need[k] = a[k] != 0.0);
    if (!any) need[1] = 1;
    auto split = [](size_t k, size_t &u, size_t &v) {
        size_t p = 1;
        while (2 * p < k) p *= 2;
        u = p;
        v = k - p;
    };
    for (size_t k = d; k >= 2; --k)
        if (need[k]) {
            size_t u, v;
            split(k, u, v);
            need[u] = need[v] = 1;
        }
    std::vector<std::vector<int>> at(d + 1, std::vector<int>(Lq + 1, -3));
    std::vector<unsigned> home(d + 1, 0);
    std::vector<double> s(d + 1, 0.0);
    at[1][Lq] = PE_IN;
    home[1] = Lq;
    s[1] = scale_in;
    auto new_buf = [&](unsigned l) {
        pe->bufs.push_back(l);
        return (int)pe->bufs.size() - 1;
    };
    auto get = [&](size_t k, unsigned l) {
        if (at[k][l] != -3) return;
        const int b = new_buf(l);
        pe->ops.push_back(PeOp{PE_CUT, l, at[k][home[k]], (int)home[k], b});
        at[k][l] = b;
    };
    int tmp = -3;   // the product before its rescale: one buffer at the top level, reused
    for (size_t k = 2; k <= d; ++k) {
        if (!need[k]) continue;
        size_t u, v;
        split(k, u, v);
        const unsigned l = Lq - ceil_log2(k) + 1;
        get(u, l);
        get(v, l);
        if (tmp == -3) tmp = new_buf(Lq);
        pe->ops.push_back(PeOp{PE_MUL, l, at[u][l], at[v][l], tmp});
        const int b = new_buf(l - 1);
        pe->ops.push_back(PeOp{PE_SWITCH, l, tmp, 0, b});
        at[k][l - 1] = b;
        home[k] = l - 1;
        s[k] = (s[u] * s[v]) / (double)hp.limbs[l - 1].lp.q;
    }
    const double m = pe->scale_out * (double)hp.limbs[Lc - 1].lp.q;
    PeOp c{PE_CKKS_COMB, Lc, 0, 0, PE_OUT};
    for (size_t k = 1; k <= d; ++k) {
        if (any ? a[k] == 0.0 : k != 1) continue;
        c.terms.push_back(at[k][home[k]]);
        c.levels.push_back(home[k]);
        c.dcoeffs.push_back(ckks_comb_coeff(a[k], m, s[k]));
    }
    c.dconstant = ckks_comb_coeff(a[0], m, 1.0);
    pe->ops.push_back(c);
    return DPFHE_OK;
}

// the launch state of key switching at level l: unlike level_view, not a prefix of the context's basis but the l + K limbs
// {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the level's own tables (DESIGN.md §4.11)
LaunchCtx pe_view(const dpfhe_polyeval *pe, const PeLevel &v) {
    LaunchCtx lc = pe->ctx->lc;
    lc.L = v.l + pe->K;
    lc.lp = v.d_lp;
    lc.lt = v.lt;
    lc.tw = v.d_tw;
    lc.itw = v.d_itw;
    lc.lift_reduce = v.lift_reduce;
    return lc;
}

// builds level l's tables, key and companions (st: the context's stream)
int pe_level(dpfhe_polyeval *pe, PeLevel &v, unsigned l, const uint64_t *h_key, cudaStream_t st) {
    dpfhe_ctx *ctx = pe->ctx;
    const unsigned K = pe->K, Lk = pe->Lk, L = ctx->hp.L, Ll = l + K;
    const size_t N = ctx->N(), dl = (l + K - 1) / K;
    v.l = l;
    std::vector<uint64_t> mod(Ll);
    for (unsigned i = 0; i < l; ++i) mod[i] = ctx->hp.limbs[i].lp.q;
    for (unsigned k = 0; k < K; ++k) mod[l + k] = ctx->hp.limbs[Lk + k].lp.q;
    std::string msg = build_host_params(ctx->hp.log_n, Ll, mod.data(), v.hp);
    if (!msg.empty()) return fail(DPFHE_ERR_INVALID, "%s", msg.c_str());
    build_group_consts(v.hp, K, pe->t, v.G, v.K);
    if (l == Lk) {   // the context's own basis
        v.d_lp = ctx->d_lp;
        v.d_tw = ctx->d_tw;
        v.d_itw = ctx->d_itw;
        v.lt = ctx->lc.lt;
        v.lift_reduce = ctx->lc.lift_reduce;
    } else {
        size_t bytes = 0;
        const int rc = upload_basis(v.hp, v.d_lp, v.d_tw, v.d_itw, v.lt, v.lift_reduce, bytes);
        if (rc) return rc;
        pe->mem.count_fixed(bytes);
    }
    // the key of level l: digits g < ceil(l / K), limb rows 0 .. l-1 and the special rows Lk .. Lk+K-1 of the top-level key
    const int rc = prepare_keys(ctx, pe_view(pe, v), 1, dl, st, "polynomial evaluator keys", [&](u64 *d_key) {
        cudaError_t e = cudaSuccess;
        for (size_t gc = 0; gc < 2 * dl && e == cudaSuccess; ++gc) {   // (digit, component) rows
            const uint64_t *src = h_key + gc * L * N;
            u64 *dst = d_key + gc * Ll * N;
            e = cudaMemcpy(dst, src, l * N * 8, cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(dst + l * N, src + Lk * N, K * N * 8, cudaMemcpyHostToDevice);
        }
        return e;
    }, v.key);
    if (rc == DPFHE_OK) pe->mem.count_fixed(v.key.bytes);
    return rc;
}

// The rest of an evaluator's creation after its plan (rc: the planner's result): the switch constants of every level from ms_lo to
// Lq, the level views, keys and companions of the products' levels.
int pe_finish(dpfhe_polyeval *pe, int rc, unsigned ms_lo, const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    dpfhe_ctx *ctx = pe->ctx;
    const unsigned Lq = pe->Lq;
    // the levels of the products, and the switch constants of every level a switch starts from
    unsigned lo = Lq + 1;
    for (const PeOp &op : pe->ops)
        if (op.kind == PE_MUL) lo = std::min(lo, op.level);
    pe->ms.resize(Lq + 1);
    for (unsigned l = ms_lo; l <= Lq && rc == DPFHE_OK; ++l) {
        HostParams hp;
        std::vector<uint64_t> mod(l);
        for (unsigned i = 0; i < l; ++i) mod[i] = ctx->hp.limbs[i].lp.q;
        std::string msg = build_host_params(ctx->hp.log_n, l, mod.data(), hp);
        if (!msg.empty()) rc = fail(DPFHE_ERR_INVALID, "%s", msg.c_str());
        else build_ms_consts(hp, pe->t, pe->ms[l]);
    }
    if (rc == DPFHE_OK && lo <= Lq) rc = ensure_hyb(ctx);
    cudaStream_t st = pick(ctx, nullptr);
    if (rc == DPFHE_OK && lo <= Lq) {
        pe->lev_lo = lo;
        pe->lev.resize(Lq - lo + 1);
        for (unsigned l = lo; l <= Lq && rc == DPFHE_OK; ++l) rc = pe_level(pe, pe->lev[l - lo], l, h_relin_key, st);
    }
    return object_finish(pe, rc, st, "polynomial evaluator keys", out);
}

}  // namespace

// launches per application: one per product, two per modulus switch, one for the combination (DESIGN.md §2.15)
int dpfhe_polyeval::apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    const size_t N = ctx->N();
    std::vector<u64 *> ptr(bufs.size());
    u64 *p = mem.get();
    for (size_t i = 0; i < bufs.size(); ++i) {
        ptr[i] = p;
        p += batch * 2 * bufs[i] * N;
    }
    u64 *tau = p;
    auto buf = [&](int b) -> u64 * { return b == PE_IN ? const_cast<u64 *>(d_ct) : b == PE_OUT ? d_out : ptr[b]; };
    cudaStream_t st = pick(ctx, stream);
    for (const PeOp &op : ops) {
        if (op.kind == PE_MUL) {
            const PeLevel &v = lev[op.level - lev_lo];
            LaunchCtx lc = pe_view(this, v);
            lc.ks_epoch = ctx->lc.ks_epoch;
            const cudaError_t e = VCALL(launch_ks_grouped, lc, KS_MUL_RELIN, buf(op.a), buf(op.b), v.key.keys[0], buf(op.out), batch, 0u, v.K, v.G, st,
                                        nullptr, v.key.key_s[0]);
            // the round numbering is the context's: the next key switch on any view must continue from here
            ctx->lc.ks_epoch = lc.ks_epoch;
            ctx->lc.ks_epoch_restarts = lc.ks_epoch_restarts;
            CU_TRY(e);
            note_launch(ctx, 1);
        } else if (op.kind == PE_SWITCH) {
            const LaunchCtx lc = level_view(ctx, op.level);
            CU_TRY(VCALL(launch_mod_switch, lc, buf(op.a), tau, buf(op.out), ms[op.level], 2 * batch, st));
            note_launch(ctx, 2);
        } else if (op.kind == PE_LINCOMB) {
            const LaunchCtx lc = level_view(ctx, op.level);
            std::vector<const u64 *> in;
            for (int b : op.terms) in.push_back(buf(b));
            CU_TRY(VCALL(launch_lincomb, lc, in.data(), op.coeffs.data(), (u32)in.size(), op.constant, nullptr, buf(op.out), batch, st));
            note_launch(ctx, 1);
        } else if (op.kind == PE_CUT) {   // a strided device copy, not a kernel
            const size_t row = (size_t)op.level * N * 8;
            CU_TRY(cudaMemcpy2DAsync(buf(op.out), row, buf(op.a), (size_t)op.b * N * 8, row, 2 * batch, cudaMemcpyDeviceToDevice, st));
        } else {   // PE_CKKS_COMB
            const LaunchCtx lc = level_view(ctx, op.level);
            std::vector<const u64 *> in;
            for (int b : op.terms) in.push_back(buf(b));
            CU_TRY(VCALL(launch_ckks_comb, lc, in.data(), op.levels.data(), op.dcoeffs.data(), (u32)in.size(), op.dconstant, ms[op.level], tau,
                         buf(op.out), batch, st));
            note_launch(ctx, 2);
        }
    }
    return DPFHE_OK;
}

// level: the start level (DESIGN.md §2.22), nullptr for the top level Lq = L - K
static int polyeval_grouped_new(dpfhe_ctx *ctx, unsigned n_special, const unsigned *level, uint64_t t_plain, const int64_t *coeffs, size_t degree,
                                const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !coeffs || !h_relin_key) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    rc = check_special(ctx, n_special);
    if (!rc && level) rc = check_level(ctx, n_special, *level, false, 0);
    if (rc) return rc;
    if (t_plain < 2 || t_plain >= ((uint64_t)1 << 31)) return fail(DPFHE_ERR_INVALID, "the plaintext modulus must be in [2, 2^31)");
    if (degree < 1 || degree > 64) return fail(DPFHE_ERR_INVALID, "the degree must be in [1, 64]");
    const unsigned L = ctx->hp.L, K = n_special, Lk = L - K, Lq = level ? *level : Lk, D = ceil_log2(degree);
    if (D > Lq - 1 || D > Lq - K + 1)
        return fail(DPFHE_ERR_INVALID, "degree %zu needs %u levels: at most min(Lq - 1, Lq - K + 1) = %u with Lq = %u, K = %u", degree, D,
                    std::min(Lq - 1, Lq - K + 1), Lq, K);
    dpfhe_polyeval *pe = new (std::nothrow) dpfhe_polyeval(ctx);
    if (!pe) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    pe->K = K; pe->Lq = Lq; pe->Lk = Lk; pe->Lf = Lq - D; pe->t = t_plain;
    rc = pe_plan(pe, coeffs, degree);
    return pe_finish(pe, rc, D > 0 ? pe->Lf + 1 : Lq + 1, h_relin_key, out);
}

static int polyeval_ckks_new(dpfhe_ctx *ctx, unsigned n_special, const unsigned *level, const double *coeffs, size_t degree, double scale_in,
                             double scale_out, const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !coeffs || !h_relin_key) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    rc = check_special(ctx, n_special);
    if (!rc && level) rc = check_level(ctx, n_special, *level, false, 0);
    if (rc) return rc;
    if (degree < 1 || degree > 64) return fail(DPFHE_ERR_INVALID, "the degree must be in [1, 64]");
    for (size_t k = 0; k <= degree; ++k)
        if (!std::isfinite(coeffs[k])) return fail(DPFHE_ERR_INVALID, "coefficient %zu is not finite", k);
    if (!(std::isfinite(scale_in) && scale_in > 0) || !(std::isfinite(scale_out) && scale_out > 0))
        return fail(DPFHE_ERR_INVALID, "the scales must be finite and positive");
    const unsigned L = ctx->hp.L, K = n_special, Lk = L - K, Lq = level ? *level : Lk, D = ceil_log2(degree);
    if (D + 2 > Lq || D > Lq - K + 1)
        return fail(DPFHE_ERR_INVALID, "degree %zu needs %u levels: at most min(Lq - 2, Lq - K + 1) with Lq = %u, K = %u", degree, D, Lq, K);
    dpfhe_polyeval *pe = new (std::nothrow) dpfhe_polyeval(ctx);
    if (!pe) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    pe->K = K; pe->Lq = Lq; pe->Lk = Lk; pe->Lf = Lq - D - 1; pe->t = 0;
    pe->ckks = true;
    pe->scale_out = scale_out;
    rc = pe_plan_ckks(pe, coeffs, degree, scale_in);
    return pe_finish(pe, rc, Lq - D, h_relin_key, out);
}

int dpfhe_polyeval_create_grouped(dpfhe_ctx *ctx, unsigned n_special, uint64_t t_plain, const int64_t *coeffs, size_t degree,
                                  const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    return polyeval_grouped_new(ctx, n_special, nullptr, t_plain, coeffs, degree, h_relin_key, out);
}

int dpfhe_polyeval_create_ckks(dpfhe_ctx *ctx, unsigned n_special, const double *coeffs, size_t degree, double scale_in, double scale_out,
                               const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    return polyeval_ckks_new(ctx, n_special, nullptr, coeffs, degree, scale_in, scale_out, h_relin_key, out);
}

// the evaluators at level l (DESIGN.md §2.22): the top-level objects of a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the top-level
// key restricted to it; a failure names the level
int dpfhe_polyeval_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, uint64_t t_plain, const int64_t *coeffs, size_t degree,
                                        const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    const int rc = polyeval_grouped_new(ctx, n_special, &level, t_plain, coeffs, degree, h_relin_key, out);
    return level_failure(level, rc);
}

int dpfhe_polyeval_create_ckks_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, const double *coeffs, size_t degree, double scale_in,
                                     double scale_out, const uint64_t *h_relin_key, dpfhe_polyeval **out) {
    const int rc = polyeval_ckks_new(ctx, n_special, &level, coeffs, degree, scale_in, scale_out, h_relin_key, out);
    return level_failure(level, rc);
}

unsigned dpfhe_polyeval_result_limbs(const dpfhe_polyeval *pe) { return pe ? pe->Lf : 0; }

double dpfhe_polyeval_result_scale(const dpfhe_polyeval *pe) { return pe && pe->ckks ? pe->scale_out : 0.0; }

void dpfhe_polyeval_destroy(dpfhe_polyeval *pe) { object_destroy(pe); }

int dpfhe_polyeval_apply(dpfhe_polyeval *pe, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    return object_apply(pe, d_ct, d_out, batch, stream);
}

int dpfhe_polyeval_apply_host(dpfhe_polyeval *pe, const uint64_t *h_ct, uint64_t *h_out, size_t batch) { return object_apply_host(pe, h_ct, h_out, batch); }

// ---------------------------------------------------------------- slot sums (DESIGN.md §2.17)
int dpfhe_slotsum_steps(size_t stride, const unsigned *radices, size_t n_stages, int *steps, size_t *n_steps) {
    if (!radices || !n_steps) return fail(DPFHE_ERR_INVALID, "null argument");
    if (stride < 1) return fail(DPFHE_ERR_INVALID, "the stride must be at least 1");
    if (n_stages < 1 || n_stages > 16) return fail(DPFHE_ERR_INVALID, "a slot sum has 1 to 16 stages");
    constexpr size_t max_half = (size_t)1 << 13;   // N/2 at the largest ring, N = 16384
    size_t count = 1, n = 0;
    for (size_t t = 0; t < n_stages; ++t) {
        if (radices[t] < 2 || radices[t] > 16) return fail(DPFHE_ERR_INVALID, "radix %u of stage %zu is outside [2, 16]", radices[t], t);
        count *= radices[t];
        if (stride > max_half / count) return fail(DPFHE_ERR_INVALID, "stride * prod(radices) must be at most N/2 <= %zu", max_half);
        n += radices[t] - 1;
    }
    if (steps) {
        size_t k = 0, span = stride;
        for (size_t t = 0; t < n_stages; ++t) {
            for (unsigned m = 1; m < radices[t]; ++m) steps[k++] = (int)(m * span);
            span *= radices[t];
        }
    }
    *n_steps = n;
    return DPFHE_OK;
}

struct dpfhe_slotsum {
    static constexpr const char *what = "null slot sum";
    dpfhe_ctx *const ctx;
    unsigned K = 0;
    size_t Lq = 0;
    unsigned level = 0;                  // below the top level (DESIGN.md §2.21): Lq = level < L - K, its state looked up at each use; 0 at the top
    std::vector<u32> n_rot;              // rotations of each stage
    std::vector<u32> galois;             // Galois elements of every step, stage by stage
    PreparedKeys gk;                     // the keys of every step, in the same order
    MsConsts Kc;
    GroupConsts G;
    CountedScratch mem;                  // counts the keys; its scratch: one intermediate batch [batch][2][Lq][N] (two or more stages), for
                                         //   the largest batch so far

    explicit dpfhe_slotsum(dpfhe_ctx *c) : ctx(c), mem(c) {}
    ~dpfhe_slotsum() { gk.release(); }
    size_t in_words() const { return 2 * Lq * ctx->N(); }
    size_t out_words() const { return in_words(); }
    // the level's state (nullptr at the top): never kept, dpfhe_context_trim frees it
    int level_of(const KsLevel *&lv) const {
        lv = nullptr;
        return level ? level_state(ctx, K, level, lv) : DPFHE_OK;
    }
    // the object's intermediate batch and the context's hoisted-rotation scratch
    int reserve(size_t batch) {
        const KsLevel *lv = nullptr;
        int rc = n_rot.size() > 1 ? mem.reserve(batch * in_words() * 8) : DPFHE_OK;
        if (!rc) rc = level_of(lv);
        return rc ? rc : rotate_sum_reserve(ctx, K, 0, batch, lv);
    }
    size_t host_chunk(size_t batch) const { return item_chunk(ctx, batch, "DPFHE_SLOTSUM_CHUNK"); }
    int apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream);
};

// S stages, alternating between the scratch batch and d_out so that the last one writes d_out; 4 launches per stage and chunk
int dpfhe_slotsum::apply_on(const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    const KsLevel *lv = nullptr;
    const int rc = level_of(lv);
    if (rc) return rc;
    cudaStream_t st = pick(ctx, stream);
    const size_t S = n_rot.size();
    const u64 *in = d_ct;
    size_t first = 0;
    for (size_t t = 0; t < S; ++t) {
        u64 *dst = (S - 1 - t) % 2 == 0 ? d_out : mem.get();
        const int rc = rotate_sum_stage(ctx, K, 0, in, n_rot[t], galois.data() + first, gk.keys.data() + first, gk.key_s.data() + first, dst, batch, Kc, G, st,
                                        lv);
        if (rc) return rc;
        first += n_rot[t];
        in = dst;
    }
    return DPFHE_OK;
}

// the slot sum at `level` (0: the top level) once the context, the pointers, n_special and t_plain are checked; a level slot sum builds
// its level's state here, so that its first application allocates no level tables; its keys are the top-level keys
static int slotsum_new(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t stride, const unsigned *radices, size_t n_stages,
                       const uint64_t *h_gks, uint64_t t_plain, dpfhe_slotsum **out) {
    int rc = DPFHE_OK;
    int steps[16 * 15];   // the most dpfhe_slotsum_steps accepts: 16 stages of radix 16
    size_t n_steps = 0;
    rc = dpfhe_slotsum_steps(stride, radices, n_stages, steps, &n_steps);
    if (rc) return rc;
    // stride * prod(radices) is the last stage's span, its first step, times its radix
    const unsigned r_last = radices[n_stages - 1];
    const size_t total = (size_t)steps[n_steps - (r_last - 1)] * r_last;
    if (total > ctx->N() / 2) return fail(DPFHE_ERR_INVALID, "stride * prod(radices) = %zu exceeds N/2 = %zu", total, ctx->N() / 2);
    const KsLevel *lv = nullptr;
    rc = level ? level_state(ctx, n_special, level, lv) : DPFHE_OK;
    if (rc) return rc;
    dpfhe_slotsum *ss = new (std::nothrow) dpfhe_slotsum(ctx);
    if (!ss) return fail(DPFHE_ERR_NOMEM, "out of host memory");
    ss->K = n_special; ss->Lq = level ? level : ctx->hp.L - n_special; ss->level = level;
    for (size_t t = 0; t < n_stages; ++t) ss->n_rot.push_back(radices[t] - 1);
    for (size_t k = 0; k < n_steps; ++k) {
        uint64_t g = 0;
        dpfhe_galois_element(ctx, steps[k], &g);
        ss->galois.push_back((u32)g);
    }
    build_group_consts(lv ? lv->hp : ctx->hp, n_special, t_plain, ss->G, ss->Kc);
    const size_t dnum = key_digits(ctx, n_special);
    cudaStream_t st = pick(ctx, nullptr);
    rc = prepare_keys(ctx, ctx->lc, n_steps, dnum, st, "slot sum keys",
                      [&](u64 *d_keys) { return cudaMemcpyAsync(d_keys, h_gks, n_steps * dnum * 2 * ctx->P() * 8, cudaMemcpyHostToDevice, st); }, ss->gk);
    if (rc == DPFHE_OK) ss->mem.count_fixed(ss->gk.bytes);
    return object_finish(ss, rc, st, "slot sum keys", out);
}

int dpfhe_slotsum_create_grouped(dpfhe_ctx *ctx, unsigned n_special, size_t stride, const unsigned *radices, size_t n_stages,
                                 const uint64_t *h_gks, uint64_t t_plain, dpfhe_slotsum **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !h_gks) return fail(DPFHE_ERR_INVALID, "null argument");
    *out = nullptr;
    rc = check_grouped(ctx, n_special, t_plain);
    if (rc) return rc;
    return slotsum_new(ctx, n_special, 0, stride, radices, n_stages, h_gks, t_plain, out);
}

// the slot sum at level l (DESIGN.md §2.21): the checks of dpfhe_slotsum_create_grouped, then the level's; l = Lq is that call
int dpfhe_slotsum_create_grouped_level(dpfhe_ctx *ctx, unsigned n_special, unsigned level, size_t stride, const unsigned *radices, size_t n_stages,
                                       const uint64_t *h_gks, uint64_t t_plain, dpfhe_slotsum **out) {
    int rc = enter(ctx);
    if (rc) return rc;
    if (!out || !h_gks) return fail(DPFHE_ERR_INVALID, "level %u: null argument", level);
    *out = nullptr;
    rc = check_grouped(ctx, n_special, t_plain);
    if (!rc) rc = check_level(ctx, n_special, level, false, t_plain);
    if (rc) return rc;
    return slotsum_new(ctx, n_special, level == ctx->hp.L - n_special ? 0 : level, stride, radices, n_stages, h_gks, t_plain, out);
}

void dpfhe_slotsum_destroy(dpfhe_slotsum *ss) { object_destroy(ss); }

int dpfhe_slotsum_apply(dpfhe_slotsum *ss, const uint64_t *d_ct, uint64_t *d_out, size_t batch, void *stream) {
    return object_apply(ss, d_ct, d_out, batch, stream);
}

int dpfhe_slotsum_apply_host(dpfhe_slotsum *ss, const uint64_t *h_ct, uint64_t *h_out, size_t batch) { return object_apply_host(ss, h_ct, h_out, batch); }

int dpfhe_describe(const dpfhe_ctx *ctx, char *buf, size_t buf_len) {
    if (!ctx || !buf || !buf_len) return fail(DPFHE_ERR_INVALID, "bad argument");
    const unsigned nt = ctx->hp.log_n == 12 ? 256 : 512;
    int n = snprintf(buf, buf_len,
                     "{\"log_n\": %u, \"n_limbs\": %u, \"num_sms\": %d, \"ntt_kernel\": {\"threads\": %u, \"smem_bytes\": %zu, "
                     "\"grid\": \"one CTA per limb\"}, \"ks_fused_kernel\": {\"threads\": %u, \"smem_bytes\": %zu, "
                     "\"grid\": \"persistent cooperative, multiple of %s, <= %zu slots\"}}",
                     ctx->hp.log_n, ctx->hp.L, ctx->lc.num_sms, nt, ctx->N() * 8, 256u, ctx->hp.log_n <= 13 ? (size_t)3 * 4096 * 8 : ctx->N() * 4,
                     ctx->hp.log_n == 13 ? "2L (a cluster of two CTAs per limb)" : "L", ctx->lc.ks_slots);
    return n;
}

}  // extern "C"
