"""Polynomial evaluation at level l on the top-level context (DESIGN.md section 2.22) on one GPU: seconds per application of
PolyEval(..., level=l) and PolyEval.ckks(..., level=l) against the same objects on a separate context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}}
with the key restricted to it (what a caller did before), at N = 8192 and 16384.  Both arms launch the same kernels; they are checked
equal bit for bit at the timed size, warmed up, then alternated, with CUDA events around at least --min-seconds of work per arm (medians
of five).  Then dpfhe_context_device_bytes of the deep network of examples/encrypted_deep_mlp.cpp's shape (Lq = 5, K = 2, two
activations, batch --batch) built both ways: one context with level calls, against a context per level (prefix contexts for encoding,
the bias and decryption, and a context over {q_0 .. q_{Lf1-1}, p_0, p_1} for the second activation with its restricted key).  The card's
name and power limit are read in the same run and printed with the numbers.

    python tools/bench_level_polyeval.py [--log-n 13,14] [--limbs 6] [--special 2] [--level 4] [--batch 256] [--degree 7] [--json out.json]
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
    ap.add_argument("--level", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--degree", type=int, default=7)
    ap.add_argument("--t", type=int, default=65537)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import deeppowers_b200 as dp
    from polyeval_ref import restrict_key
    if not torch.cuda.is_available():
        sys.exit("bench_level_polyeval.py needs a CUDA device; there is no CPU fallback and no number without one")
    Lq, K, l, t, d = args.limbs, args.special, args.level, args.t, args.degree
    L = Lq + K
    i64 = dict(dtype=torch.int64, device="cuda")
    result = {"card": card(), "Lq": Lq, "K": K, "level": l, "batch": args.batch, "degree": d, "t": t, "rows": [], "memory": {}}
    print("card: %s; Lq = %d, K = %d, level %d, batch %d, degree %d" % (result["card"], Lq, K, l, args.batch, d))

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    rng = np.random.default_rng(1)
    for log_n in [int(x) for x in args.log_n.split(",")]:
        c = dp.Context(log_n, L)
        mods = list(c.moduli)
        cl = dp.Context(log_n, l + K, mods[:l] + mods[Lq:])
        N, B = c.N, args.batch if log_n <= 13 else args.batch // 2
        dnum = c.grouped_digits(K)
        kt = torch.empty((dnum, 2, L, N), **i64)
        c.fill_uniform(3, kt, dnum * 2)
        key = kt.cpu().numpy().view(np.uint64)
        key_low = np.ascontiguousarray(restrict_key(key, Lq, K, l))
        del kt
        full = torch.empty((B, 2, l + K, N), **i64)
        cl.fill_uniform(1, full, B * 2)
        ct = full[:, :, :l].contiguous()
        del full
        coeffs = [int(v) for v in rng.integers(-1000, 1000, d + 1)]
        dcoeffs = list(rng.uniform(-1, 1, d + 1) / (d + 1))
        scale = float(mods[1])
        objs = {
            "bgv": (dp.PolyEval(c, K, t, coeffs, key, level=l), dp.PolyEval(cl, K, t, coeffs, key_low)),
            "ckks": (dp.PolyEval.ckks(c, K, dcoeffs, scale, key, level=l), dp.PolyEval.ckks(cl, K, dcoeffs, scale, key_low)),
        }
        print("N = %d, batch %d" % (N, B))
        print("%6s %12s %12s %8s" % ("kind", "level s", "context s", "ratio"))
        for name, (lvl_o, ref_o) in objs.items():
            out = torch.empty((B, 2, lvl_o.result_limbs, N), **i64)
            lvl, ref = (lambda o=lvl_o: o.apply(ct, out, B)), (lambda o=ref_o: o.apply(ct, out, B))
            got = []
            for f in (lvl, ref):
                f()
                torch.cuda.synchronize()
                got.append(out.clone())
            if not torch.equal(got[0], got[1]):
                sys.exit("%s: the level evaluator and the level context's evaluator differ at N = %d" % (name, N))
            for f in (lvl, ref, lvl, ref):   # warm-up
                f()
            torch.cuda.synchronize()
            est = {f: timed(f, 1) for f in (lvl, ref)}
            ts = {f: [] for f in est}
            for _ in range(5):   # alternate the arms
                for f in (lvl, ref):
                    ts[f].append(timed(f, max(1, int(args.min_seconds / 5 / est[f]) + 1)))
            s = {f: sorted(v)[len(v) // 2] for f, v in ts.items()}
            spread = {f: (min(v), max(v)) for f, v in ts.items()}
            row = {"log_n": log_n, "batch": B, "kind": name, "level_s": s[lvl], "context_s": s[ref],
                   "level_range_s": spread[lvl], "context_range_s": spread[ref]}
            result["rows"].append(row)
            print("%6s %12.6f %12.6f %8.3f   (level %.6f .. %.6f, context %.6f .. %.6f)"
                  % (name, s[lvl], s[ref], s[lvl] / s[ref], *spread[lvl], *spread[ref]))
            del out
        for lvl_o, ref_o in objs.values():
            lvl_o.close()
            ref_o.close()
        cl.close()
        c.close()
        del ct
        torch.cuda.empty_cache()

    # device memory of the deep network's shape: Lq = 5, K = 2, two quadratic activations, one application of each at batch B, N = 8192
    log_n, Lq2, B = 13, 5, args.batch
    L2 = Lq2 + K

    def run_net(one_context):
        made = []
        c = dp.Context(log_n, L2)
        made.append(c)
        mods = list(c.moduli)
        N = c.N
        dnum = c.grouped_digits(K)
        kt = torch.empty((dnum, 2, L2, N), **i64)
        c.fill_uniform(3, kt, dnum * 2)
        key = kt.cpu().numpy().view(np.uint64)
        del kt
        pe1 = dp.PolyEval(c, K, t, [3, -2, 1], key)
        made.append(pe1)
        Lf1 = pe1.result_limbs
        x = torch.zeros((B, 2, Lq2, N), **i64)   # any words: the memory, not the values, is measured
        pt = torch.zeros((Lq2, N), **i64)
        if one_context:
            pe2 = dp.PolyEval(c, K, t, [3, -2, 1], key, level=Lf1)
            made.append(pe2)
            c.ct_add_plain_level(Lq2, x, pt, x, B)
            h1 = torch.empty((B, 2, Lf1, N), **i64)
            pe1.apply(x, h1, B)
            c.ct_add_plain_level(Lf1, h1, pt[:Lf1].contiguous(), h1, B)
            h2 = torch.empty((B, 2, pe2.result_limbs, N), **i64)
            pe2.apply(h1, h2, B)
            torch.cuda.synchronize()
            ctxs = [c]
        else:
            cq = dp.Context(log_n, Lq2, mods[:Lq2])                      # encoding, encryption, the first bias
            cf = dp.Context(log_n, Lf1, mods[:Lf1])                      # the second bias
            c2 = dp.Context(log_n, Lf1 + K, mods[:Lf1] + mods[Lq2:])    # the second activation, with its restricted key
            made += [cq, cf, c2]
            pe2 = dp.PolyEval(c2, K, t, [3, -2, 1], np.ascontiguousarray(restrict_key(key, Lq2, K, Lf1)))
            made.append(pe2)
            cq.ct_add_plain(x, pt, x, B)
            h1 = torch.empty((B, 2, Lf1, N), **i64)
            pe1.apply(x, h1, B)
            cf.ct_add_plain(h1, pt[:Lf1].contiguous(), h1, B)
            h2 = torch.empty((B, 2, pe2.result_limbs, N), **i64)
            pe2.apply(h1, h2, B)
            torch.cuda.synchronize()
            ctxs = [c, cq, cf, c2]
        total = sum(k.device_bytes() for k in ctxs)
        for o in reversed(made):
            o.close()
        torch.cuda.empty_cache()
        return total

    one, several = run_net(True), run_net(False)
    result["memory"] = {"log_n": log_n, "Lq": Lq2, "K": K, "batch": B, "one_context_bytes": one, "prefix_contexts_bytes": several}
    print("deep network, N = 8192, Lq = %d, K = %d, batch %d: dpfhe_context_device_bytes %.1f MiB on one context, %.1f MiB with prefix "
          "contexts" % (Lq2, K, B, one / 2 ** 20, several / 2 ** 20))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
