"""BGV polynomial evaluation (PolyEval, DESIGN.md section 2.15) at N = 8192, Lq = 4 ciphertext limbs + K = 2 special primes, t = 65537:
ciphertexts per second for d = 2 and d = 8 at batch 512 (CUDA events around whole applications after warm-up), the split of one
application's kernel time between the grouped key switches (ks_grouped_kernel) and everything else (torch.profiler, a run of its own
after the timed one), and the achieved HBM bandwidth of ct_lincomb (CUDA events over many launches; bytes = every input row read once
plus the output written once) against the 3.35 TB/s data-sheet peak.  Synthetic data from fill_uniform.  Prints one JSON line with the
GPU's name and power limit (DESIGN.md section 6).

    python tools/bench_polyeval.py [--batch 512] [--iters 10]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402
from bench_linear_grouped import gpu_info, uniform  # noqa: E402

LOG_N, LQ, K, T = 13, 4, 2, 65537
N = 1 << LOG_N
PEAK = 3.35e12
POLYS = {2: [1, 2, 3], 8: [1, 2, 3, 4, 5, 6, 7, 8, 9]}


def time_events(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters / 1e3   # seconds per call


def kernel_split(fn):
    """device time of one call: (key-switch kernels, everything else), in seconds"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = other = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "ks_grouped_kernel" in e.name:
            ks += us
        elif "kernel" in e.name.lower():
            other += us
    return ks / 1e6, other / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    B, L = args.batch, LQ + K
    name, power = gpu_info()
    ctx, ctx_q = dp.Context(LOG_N, L), dp.Context(LOG_N, LQ)
    key = uniform(ctx, 1, (ctx.grouped_digits(K), 2, L, N)).cpu().numpy().view("uint64")
    x = uniform(ctx_q, 2, (B, 2, LQ, N))
    res = {"gpu": name, "power_limit": power, "N": N, "Lq": LQ, "K": K, "t": T, "batch": B}
    for d, coeffs in POLYS.items():
        pe = dp.PolyEval(ctx, K, T, coeffs, key)
        out = torch.empty((B, 2, pe.result_limbs, N), dtype=torch.int64, device="cuda")
        run = lambda: pe.apply(x, out, B)
        for _ in range(args.warmup):
            run()
        n0 = ctx.launch_count()
        reps = [time_events(run, args.iters) for _ in range(3)]
        launches = (ctx.launch_count() - n0) // (3 * args.iters)
        ks, other = kernel_split(run)
        res["d%d" % d] = {"ct_per_s": B / statistics.median(reps), "ms_per_apply": [round(r * 1e3, 3) for r in reps], "launches": launches,
                          "ks_ms": round(ks * 1e3, 3), "other_ms": round(other * 1e3, 3), "ks_share": round(ks / (ks + other), 3)}
        pe.close()
    # ct_lincomb on the ciphertext moduli, 8 terms and 1 term (+ the output)
    for m in (8, 1):
        cts = [uniform(ctx_q, 10 + i, (B, 2, LQ, N)) for i in range(m)]
        out = torch.empty((B, 2, LQ, N), dtype=torch.int64, device="cuda")
        run = lambda: ctx_q.ct_lincomb(cts, list(range(3, 3 + m)), 5, out, B)
        for _ in range(args.warmup):
            run()
        reps = [time_events(run, 20) for _ in range(3)]
        nbytes = (m + 1) * B * 2 * LQ * N * 8
        s = statistics.median(reps)
        res["lincomb_%d" % m] = {"ms": round(s * 1e3, 3), "GBps": round(nbytes / s / 1e9, 1), "frac_of_peak": round(nbytes / s / PEAK, 3)}
        del cts
    print(json.dumps(res))


if __name__ == "__main__":
    main()
