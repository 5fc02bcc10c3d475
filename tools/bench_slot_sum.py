"""Summed rotations and slot sums (DESIGN.md section 2.17) at N = 8192, Lq = 4 ciphertext limbs + K = 2 special primes, batch 512,
synthetic data from fill_uniform:
  - seconds per stage of r = 2, 4, 8, 16 (r - 1 rotations): dpfhe_rotate_sum_grouped against the composition it replaces,
    dpfhe_rotate_hoisted_grouped + dpfhe_ct_lincomb on the same inputs, the two alternated in one run (CUDA events after warm-up);
  - ciphertexts per second of a 64-slot SlotSum under radices {2,2,2,2,2,2}, {4,4,4}, {8,8} and {16,4};
  - the split of one r = 8 stage's kernel time between the mod-up (ks_hoistg_kernel), the summed multiply-accumulate
    (rot_sum_grouped_kernel) and the division by P (md_tau_kernel, md_limb_kernel), from torch.profiler.
Prints one JSON line with the GPU's name and power limit (DESIGN.md section 6).

    python tools/bench_slot_sum.py [--batch 512] [--iters 10]
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
RADICES = {"2x6": [2] * 6, "4x3": [4, 4, 4], "8x2": [8, 8], "16x4": [16, 4]}


def time_events(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters / 1e3   # seconds per call


def kernel_split(fn):
    """device time of one call by kernel family, in seconds"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"mod_up": 0.0, "sum_mac": 0.0, "mod_down": 0.0, "other": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "ks_hoistg_kernel" in e.name:
            split["mod_up"] += us
        elif "rot_sum_grouped_kernel" in e.name:
            split["sum_mac"] += us
        elif "md_tau_kernel" in e.name or "md_limb_kernel" in e.name:
            split["mod_down"] += us
        elif "kernel" in e.name.lower():
            split["other"] += us
    return {k: round(v / 1e3, 3) for k, v in split.items()}   # ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    B, L = args.batch, LQ + K
    name, power = gpu_info()
    ctx, ctx_q = dp.Context(LOG_N, L), dp.Context(LOG_N, LQ)
    dnum = ctx.grouped_digits(K)
    x = uniform(ctx_q, 2, (B, 2, LQ, N))
    keys = uniform(ctx, 3, (15, dnum, 2, L, N))
    res = {"gpu": name, "power_limit": power, "N": N, "Lq": LQ, "K": K, "t": T, "batch": B, "stage": {}, "slot_sum_64": {}}
    out = torch.empty((B, 2, LQ, N), dtype=torch.int64, device="cuda")
    rots = torch.empty((15, B, 2, LQ, N), dtype=torch.int64, device="cuda")
    for r in (2, 4, 8, 16):
        g = [ctx.galois_elt(m) for m in range(1, r)]
        ks = [keys[m] for m in range(r - 1)]
        fused = lambda: ctx.rotate_sum_grouped(K, x, g, ks, out, B, T)

        def composed():
            ctx.rotate_hoisted_grouped(K, x, g, ks, rots[:r - 1], B, T)
            ctx_q.ct_lincomb([x] + [rots[m] for m in range(r - 1)], [1] * r, 0, out, B)
        for _ in range(args.warmup):
            fused()
            composed()
        tf, tc = [], []
        for _ in range(3):   # alternated
            tf.append(time_events(fused, args.iters))
            tc.append(time_events(composed, args.iters))
        res["stage"]["r%d" % r] = {"summed_ms": round(statistics.median(tf) * 1e3, 3), "composition_ms": round(statistics.median(tc) * 1e3, 3),
                                   "speedup": round(statistics.median(tc) / statistics.median(tf), 3)}
        if r == 8:
            res["stage"]["r8"]["split_ms"] = kernel_split(fused)
    for label, radices in RADICES.items():
        steps = dp.slotsum_steps(1, radices)
        gks = keys[:len(steps)] if len(steps) <= 15 else torch.cat([keys, keys[:len(steps) - 15]])
        ss = dp.SlotSum.grouped(ctx, K, 1, radices, gks.contiguous().cpu().numpy().view("uint64"), T)
        run = lambda: ss.apply(x, out, B)
        for _ in range(args.warmup):
            run()
        reps = [time_events(run, args.iters) for _ in range(3)]
        res["slot_sum_64"][label] = {"keys": len(steps), "ct_per_s": round(B / statistics.median(reps), 1),
                                     "ms_per_apply": [round(t * 1e3, 3) for t in reps]}
        ss.close()
    ctx_q.close()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
