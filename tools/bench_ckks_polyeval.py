"""CKKS polynomial evaluation (PolyEval.ckks, DESIGN.md section 2.16) at N = 8192 on the CKKS chain of the tests (q_0 a 60-bit
k 2^32 + 1 prime, q_1 .. q_4 such primes just above 2^45, K = 2 special 60-bit primes), batch 512, d = 3, 7 and 8: milliseconds per
application (CUDA events around whole applications after warm-up); the split of one application's device time between the products
(ks_grouped_kernel), the rescales (ms_tau/ms_limb), the fused combination (ckks_comb_*) and the operand cuts (device copies), from
torch.profiler in a run of its own; and the fused combination against the composition it replaces (the cut copies, ct_lincomb and
mod_switch_down) on the same shapes.  Synthetic data from fill_uniform.  Prints one JSON line with the GPU's name and power limit.

    python tools/bench_ckks_polyeval.py [--batch 512] [--iters 10]
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
from bench_polyeval import time_events  # noqa: E402

LOG_N, LQ, K = 13, 5, 2
N = 1 << LOG_N
DELTA = 2.0**45
POLYS = {3: [0.1, 0.5, 0.0, -0.2], 7: [0.0, 0.5, 0.39894228, 0.0, -0.06649038, 0.0, 0.00997356, 0.0], 8: [1.0] * 9}


def is_prime(n):
    """deterministic Miller-Rabin for n < 3.3e24"""
    if n < 2:
        return False
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41):
        if n % p == 0:
            return n == p
    d, r = n - 1, 0
    while d % 2 == 0:
        d, r = d // 2, r + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(r - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def scan(start, step, count):
    """`count` primes start, start + step, ... that are 1 mod 2^15 (start is, step a multiple of 2^32)"""
    out, c = [], start
    while len(out) < count:
        if is_prime(c):
            out.append(c)
        c += step
    return out


def ckks_chain():
    top = scan((1 << 60) - (1 << 32) + 1, -(1 << 32), 1 + K)
    return [top[0]] + scan((1 << 45) + 1, 1 << 32, LQ - 1) + top[1:]


def kernel_split(fn):
    """device time of one call by part, in milliseconds"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    parts = {"products": 0.0, "rescales": 0.0, "combination": 0.0, "cuts": 0.0, "other": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "ks_grouped_kernel" in e.name:
            parts["products"] += us
        elif "ms_tau_kernel" in e.name or "ms_limb_kernel" in e.name:
            parts["rescales"] += us
        elif "ckks_comb" in e.name:
            parts["combination"] += us
        elif "memcpy" in e.name.lower():
            parts["cuts"] += us
        else:
            parts["other"] += us
    return {k: round(v / 1e3, 3) for k, v in parts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    B, L = args.batch, LQ + K
    moduli = ckks_chain()
    name, power = gpu_info()
    ctx, ctx_q = dp.Context(LOG_N, L, moduli), dp.Context(LOG_N, LQ, moduli[:LQ])
    key = uniform(ctx, 1, (ctx.grouped_digits(K), 2, L, N)).cpu().numpy().view("uint64")
    x = uniform(ctx_q, 2, (B, 2, LQ, N))
    res = {"gpu": name, "power_limit": power, "N": N, "Lq": LQ, "K": K, "batch": B}
    for d, coeffs in POLYS.items():
        pe = dp.PolyEval.ckks(ctx, K, coeffs, DELTA, key)
        out = torch.empty((B, 2, pe.result_limbs, N), dtype=torch.int64, device="cuda")
        run = lambda: pe.apply(x, out, B)
        for _ in range(args.warmup):
            run()
        n0 = ctx.launch_count()
        reps = [time_events(run, args.iters) for _ in range(3)]
        launches = (ctx.launch_count() - n0) // (3 * args.iters)
        res["d%d" % d] = {"ms_per_apply": [round(r * 1e3, 3) for r in reps], "ct_per_s": round(B / statistics.median(reps)), "launches": launches,
                          "split_ms": kernel_split(run)}
        pe.close()
    # the combination of d = 7: its terms x, x^2, x^4 and x^6 live at levels 5, 4, 3 and 2, the combination at Lc = 2.  The fused
    # pair against cut copies + ct_lincomb + mod_switch_down on the same shapes.
    Lc = 2
    levels = [5, 4, 3, 2]
    terms = [uniform(dp.Context(LOG_N, lv, moduli[:lv]), 20 + i, (B, 2, lv, N)) for i, lv in enumerate(levels)]
    ctx_c = dp.Context(LOG_N, Lc, moduli[:Lc])
    cuts = [torch.empty((B, 2, Lc, N), dtype=torch.int64, device="cuda") for _ in terms]
    comb = torch.empty((B, 2, Lc, N), dtype=torch.int64, device="cuda")
    res_c = torch.empty((B, 2, Lc - 1, N), dtype=torch.int64, device="cuda")

    def composed():
        for c, t in zip(cuts, terms):
            c.copy_(t[:, :, :Lc])
        ctx_c.ct_lincomb(cuts, [3, -5, 7, 11], 17, comb, B)
        ctx_c.mod_switch_down(comb, res_c, 2 * B)

    for _ in range(args.warmup):
        composed()
    t_comp = statistics.median([time_events(composed, 20) for _ in range(3)])
    # the fused pair of a d = 7 application, from the profiler split
    pe = dp.PolyEval.ckks(ctx, K, POLYS[7], DELTA, key)
    out = torch.empty((B, 2, pe.result_limbs, N), dtype=torch.int64, device="cuda")
    split = [kernel_split(lambda: pe.apply(x, out, B))["combination"] for _ in range(3)]
    res["combination_d7"] = {"fused_ms": statistics.median(split), "composed_ms": round(t_comp * 1e3, 3)}
    pe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
