"""Calls at level l on the top-level context (DESIGN.md sections 2.20 / 4.17) on one GPU: seconds per call of every *_level entry point
against the same call on a separate context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the key restricted to it (what a caller did
before), at N = 8192 and 16384.  Both arms are checked equal bit for bit at the timed size, warmed up, then alternated, with CUDA events
around at least --min-seconds of work per arm (medians of five).  Then the device memory of a full-depth chain both ways: one context
that has run a level call at every level l = Lq .. 2 with its one top-level key, against one context per level, each with its
restricted key.  The card's name and power limit are printed with the numbers.

    python tools/bench_levels.py [--log-n 13,14] [--limbs 6] [--special 2] [--level 4] [--batch 256] [--terms 4] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="13,14")
    ap.add_argument("--limbs", type=int, default=6, help="ciphertext moduli Lq at the top level")
    ap.add_argument("--special", type=int, default=2)
    ap.add_argument("--level", type=int, default=4)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--terms", type=int, default=4, help="pairs of the inner products and rotations of the rotation sum")
    ap.add_argument("--t", type=int, default=65537)
    ap.add_argument("--min-seconds", type=float, default=0.3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import deeppowers_b200 as dp
    from polyeval_ref import restrict_key
    if not torch.cuda.is_available():
        sys.exit("bench_levels.py needs a CUDA device; there is no CPU fallback and no number without one")
    Lq, K, l, n, t = args.limbs, args.special, args.level, args.terms, args.t
    L = Lq + K
    i64 = dict(dtype=torch.int64, device="cuda")
    gal = [pow(5, m + 1, 1 << 14) for m in range(n)]
    result = {"card": card(), "Lq": Lq, "K": K, "level": l, "batch": args.batch, "terms": n, "t": t, "rows": [], "memory": []}
    print("card: %s; Lq = %d, K = %d, level %d, batch %d, %d pairs / rotations, t = %d" % (result["card"], Lq, K, l, args.batch, n, t))

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    for log_n in [int(x) for x in args.log_n.split(",")]:
        c = dp.Context(log_n, L)
        mods = list(c.moduli)
        cl = dp.Context(log_n, l + K, mods[:l] + mods[Lq:])
        N, B = c.N, args.batch if log_n <= 13 else args.batch // 2
        dnum = c.grouped_digits(K)
        ops = torch.empty((2 * n, B, 2, l, N), **i64)
        # uniform operands over q_0 .. q_{l-1}: the level context's first l rows
        full = torch.empty((2 * n, B, 2, l + K, N), **i64)
        cl.fill_uniform(1, full, 2 * n * B * 2)
        ops.copy_(full[:, :, :, :l])
        del full
        keys = torch.empty((n, dnum, 2, L, N), **i64)
        c.fill_uniform(2, keys, n * dnum * 2)
        low = [torch.from_numpy(restrict_key(k.cpu().numpy().view(np.uint64), Lq, K, l).view(np.int64)).cuda() for k in keys]
        a, b = [ops[i] for i in range(n)], [ops[n + i] for i in range(n)]
        out, out_r = torch.empty((B, 2, l, N), **i64), torch.empty((B, 2, l - 1, N), **i64)
        calls = {
            "ct_mul_relin": (lambda: c.ct_mul_relin_grouped_level(K, l, a[0], b[0], keys[0], out, B, t),
                             lambda: cl.ct_mul_relin_grouped(K, a[0], b[0], low[0], out, B, t)),
            "ct_mul_relin_rescale": (lambda: c.ct_mul_relin_rescale_grouped_level(K, l, a[0], b[0], keys[0], out_r, B, t),
                                     lambda: cl.ct_mul_relin_rescale_grouped(K, a[0], b[0], low[0], out_r, B, t)),
            "ct_dot": (lambda: c.ct_dot_grouped_level(K, l, a, b, keys[0], out, B, t), lambda: cl.ct_dot_grouped(K, a, b, low[0], out, B, t)),
            "ct_dot_rescale": (lambda: c.ct_dot_rescale_grouped_level(K, l, a, b, keys[0], out_r, B, t),
                               lambda: cl.ct_dot_rescale_grouped(K, a, b, low[0], out_r, B, t)),
            "rotate": (lambda: c.rotate_grouped_level(K, l, a[0], gal[0], keys[0], out, B, t),
                       lambda: cl.rotate_grouped(K, a[0], gal[0], low[0], out, B, t)),
            "rotate_sum": (lambda: c.rotate_sum_grouped_level(K, l, a[0], gal, list(keys), out, B, t),
                           lambda: cl.rotate_sum_grouped(K, a[0], gal, low, out, B, t)),
        }
        print("N = %d" % N)
        print("%22s %12s %12s %8s" % ("call", "level s", "context s", "ratio"))
        for name, (lvl, ref) in calls.items():
            got = []
            for f in (lvl, ref):
                f()
                torch.cuda.synchronize()
                got.append((out_r if "rescale" in name else out).clone())
            if not torch.equal(got[0], got[1]):
                sys.exit("%s: the level call and the level context's call differ at N = %d" % (name, N))
            for f in (lvl, ref, lvl, ref):   # warm-up
                f()
            torch.cuda.synchronize()
            est = {f: timed(f, 1) for f in (lvl, ref)}
            ts = {f: [] for f in est}
            for _ in range(5):   # alternate the arms
                for f in (lvl, ref):
                    ts[f].append(timed(f, max(1, int(args.min_seconds / 5 / est[f]) + 1)))
            s = {f: sorted(v)[len(v) // 2] for f, v in ts.items()}
            row = {"log_n": log_n, "batch": B, "call": name, "level_s": s[lvl], "context_s": s[ref]}
            result["rows"].append(row)
            print("%22s %12.6f %12.6f %8.3f" % (name, s[lvl], s[ref], s[lvl] / s[ref]))
        cl.close()
        del ops, low, a, b, out, out_r

        # device memory of a full-depth multiply-and-rescale chain (levels Lq .. 2), one ciphertext per level
        key = keys[0].contiguous()
        torch.cuda.synchronize()
        for lv in range(Lq, 1, -1):
            x, y = torch.zeros((1, 2, lv, N), **i64), torch.empty((1, 2, lv - 1, N), **i64)
            c.ct_mul_relin_rescale_grouped_level(K, lv, x, x, key, y, 1, t)
        torch.cuda.synchronize()
        one = c.device_bytes() + key.numel() * 8
        per_level = 0
        for lv in range(Lq, 1, -1):
            cx = dp.Context(log_n, lv + K, mods[:lv] + mods[Lq:])
            k = torch.from_numpy(restrict_key(key.cpu().numpy().view(np.uint64), Lq, K, lv).view(np.int64)).cuda()
            x, y = torch.zeros((1, 2, lv, N), **i64), torch.empty((1, 2, lv - 1, N), **i64)
            cx.ct_mul_relin_rescale_grouped(K, x, x, k, y, 1, t)
            torch.cuda.synchronize()
            per_level += cx.device_bytes() + k.numel() * 8
            cx.close()
        result["memory"].append({"log_n": log_n, "one_context_bytes": one, "context_per_level_bytes": per_level})
        print("full-depth chain (levels %d .. 2), device bytes with the key(s): one context %d (%.1f MiB), a context per level %d (%.1f MiB)"
              % (Lq, one, one / 2**20, per_level, per_level / 2**20))
        c.close()
        del keys, key
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
