"""The encrypted linear layer of BASELINE.json config 4 (768 x 768, baby 32 x giant 24, N = 8192, 4 ciphertext limbs) with grouped
special-prime keys (2 special primes) as the library object (LinearLayer.grouped: companions prepared once, fused Horner steps), against
the Python composition linear_bsgs_grouped and against the per-limb-digit layer (LinearLayer on 4 limbs).  Synthetic data from
fill_uniform; the three are timed with CUDA events, alternated in one run after warm-up; the first two outputs must be identical.
Prints one JSON line with the GPU's name and power limit (DESIGN.md section 6).

    python tools/bench_linear_grouped.py [--batch 512] [--iters 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402

LOG_N, LQ, K, DIM, BABY = 13, 4, 2, 768, 32
N = 1 << LOG_N


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def uniform(ctx, seed, shape):
    t = torch.empty(shape, dtype=torch.int64, device="cuda")
    ctx.fill_uniform(seed, t, t.numel() // ctx.P)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    B, L = args.batch, LQ + K
    giant = DIM // BABY
    ctx, ctx_q = dp.Context(LOG_N, L), dp.Context(LOG_N, LQ)
    assert ctx_q.moduli == ctx.moduli[:LQ]
    lq_ctx_bytes = ctx_q.device_bytes()   # what a context over the ciphertext moduli costs before any call: the layer uses a view instead
    dnum = ctx.grouped_digits(K)
    x = uniform(ctx_q, 1, (B, 2, LQ, N))
    diags = uniform(ctx_q, 2, (DIM, LQ, N))
    gkeys = [uniform(ctx, 100 + r, (dnum, 2, L, N)) for r in range(BABY)]        # 31 baby-step keys, then the giant-step key
    bkeys = [uniform(ctx_q, 200 + r, (LQ, 2, LQ, N)) for r in range(BABY)]       # per-limb-digit keys on the ciphertext moduli
    h = lambda t: t.cpu().numpy().view("uint64")
    h_diags = h(diags)
    layer = dp.LinearLayer.grouped(ctx, K, h_diags, BABY, h(torch.stack(gkeys[:BABY - 1])), h(gkeys[BABY - 1]), 65537)
    layer_q = dp.LinearLayer(ctx_q, h_diags, BABY, h(torch.stack(bkeys[:BABY - 1])), h(bkeys[BABY - 1]))
    out_lib, out_py, out_pl = (torch.empty_like(x) for _ in range(3))
    scratch = torch.empty((BABY + giant + 1, B, 2, LQ, N), dtype=torch.int64, device="cuda")
    runs = {
        "library_object": lambda: layer.apply(x, out_lib, B),
        "linear_bsgs_grouped": lambda: dp.linear_bsgs_grouped(ctx, ctx_q, K, x, diags, gkeys[:BABY - 1], gkeys[BABY - 1], BABY, out_py, B, 65537,
                                                              scratch),
        "per_limb_layer": lambda: layer_q.apply(x, out_pl, B),
    }
    n0 = ctx.launch_count()
    runs["library_object"]()
    torch.cuda.synchronize()
    launches_lib = ctx.launch_count() - n0
    n0, m0 = ctx.launch_count(), ctx_q.launch_count()
    runs["linear_bsgs_grouped"]()
    torch.cuda.synchronize()
    launches_py = ctx.launch_count() - n0 + ctx_q.launch_count() - m0
    for _ in range(args.warmup):
        for fn in runs.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(args.iters):
        for name, fn in runs.items():      # alternated: clocks and thermals drift across the run, not between the three
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    identical = bool(torch.equal(out_lib, out_py))
    name, power = gpu_info()
    res = {k: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v), "ciphertexts_per_s": B / statistics.median(v) * 1e3}
           for k, v in times.items()}
    lib_ms, py_ms = res["library_object"]["ms_median"], res["linear_bsgs_grouped"]["ms_median"]
    print(json.dumps({"gpu": name, "power_limit": power, "workload": "768x768 layer, N=%d, %d+%d limbs, baby %d x giant %d, batch %d, t=65537"
                      % (N, LQ, K, BABY, giant, B), "iters": args.iters, "results": res, "speedup_vs_composition": py_ms / lib_ms,
                      "library_equals_composition": identical, "launches_per_apply": {"library_object": launches_lib, "linear_bsgs_grouped": launches_py},
                      "device_bytes_of_an_Lq_context": lq_ctx_bytes}))
    layer.close()
    layer_q.close()
    ctx.close()
    ctx_q.close()
    if not identical:
        sys.exit(1)


if __name__ == "__main__":
    main()
