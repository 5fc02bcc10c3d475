"""The linear layer and the slot sum at level l on the top-level context (DESIGN.md sections 2.21 / 4.18) on one GPU: seconds per
application of LinearLayer.grouped(..., level=l) and SlotSum.grouped(..., level=l) against the same objects on a separate context over
{q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the keys restricted to it (what a caller did before), at N = 8192 and 16384.  Both arms are
checked equal bit for bit at the timed size, warmed up, then alternated, with CUDA events around at least --min-seconds of work per arm
(medians of five).  Then the device memory of a two-layer network both ways: one context holding a top-level layer and the level
layer with one set of top-level keys, against a second context for the level with its own restricted keys.  The card's name and power
limit are read in the same run and printed with the numbers.

    python tools/bench_level_layer.py [--log-n 13,14] [--limbs 6] [--special 2] [--level 4] [--batch 256] [--baby 8] [--giant 4]
                                      [--radices 4,4] [--json out.json]
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
    ap.add_argument("--baby", type=int, default=8)
    ap.add_argument("--giant", type=int, default=4)
    ap.add_argument("--radices", default="4,4")
    ap.add_argument("--t", type=int, default=65537)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import deeppowers_b200 as dp
    from polyeval_ref import restrict_key
    if not torch.cuda.is_available():
        sys.exit("bench_level_layer.py needs a CUDA device; there is no CPU fallback and no number without one")
    Lq, K, l, t, baby, giant = args.limbs, args.special, args.level, args.t, args.baby, args.giant
    radices = [int(r) for r in args.radices.split(",")]
    L = Lq + K
    i64 = dict(dtype=torch.int64, device="cuda")
    result = {"card": card(), "Lq": Lq, "K": K, "level": l, "batch": args.batch, "baby": baby, "giant": giant, "radices": radices, "t": t,
              "rows": [], "memory": []}
    print("card: %s; Lq = %d, K = %d, level %d, batch %d, baby %d, giant %d, radices %s, t = %d"
          % (result["card"], Lq, K, l, args.batch, baby, giant, radices, t))

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    def host_keys(c, n, seed):
        dnum = c.grouped_digits(K)
        k = torch.empty((n, dnum, 2, L, c.N), **i64)
        c.fill_uniform(seed, k, n * dnum * 2)
        return k.cpu().numpy().view(np.uint64)

    for log_n in [int(x) for x in args.log_n.split(",")]:
        c = dp.Context(log_n, L)
        mods = list(c.moduli)
        cl = dp.Context(log_n, l + K, mods[:l] + mods[Lq:])
        N, B = c.N, args.batch if log_n <= 13 else args.batch // 2
        full = torch.empty((B, 2, l + K, N), **i64)
        cl.fill_uniform(1, full, B * 2)
        ct = full[:, :, :l].contiguous()
        del full
        dfull = torch.empty((baby * giant, l + K, N), **i64)
        cl.fill_uniform(2, dfull, baby * giant)
        diags = np.ascontiguousarray(dfull[:, :l].cpu().numpy().view(np.uint64))
        del dfull
        lk = host_keys(c, baby, 3)   # baby-step keys, then the giant-step key
        lk_low = np.stack([restrict_key(k, Lq, K, l) for k in lk])
        n_steps = len(dp.slotsum_steps(1, radices))
        sk = host_keys(c, n_steps, 4)
        sk_low = np.ascontiguousarray(np.stack([restrict_key(k, Lq, K, l) for k in sk]))
        objs = {
            "linear layer": (dp.LinearLayer.grouped(c, K, diags, baby, np.ascontiguousarray(lk[:baby - 1]), lk[baby - 1], t, level=l),
                             dp.LinearLayer.grouped(cl, K, diags, baby, np.ascontiguousarray(lk_low[:baby - 1]), lk_low[baby - 1], t)),
            "slot sum": (dp.SlotSum.grouped(c, K, 1, radices, sk, t, level=l), dp.SlotSum.grouped(cl, K, 1, radices, sk_low, t)),
        }
        out = torch.empty_like(ct)
        print("N = %d, batch %d" % (N, B))
        print("%14s %12s %12s %8s" % ("object", "level s", "context s", "ratio"))
        for name, (lvl_o, ref_o) in objs.items():
            lvl, ref = (lambda o=lvl_o: o.apply(ct, out, B)), (lambda o=ref_o: o.apply(ct, out, B))
            got = []
            for f in (lvl, ref):
                f()
                torch.cuda.synchronize()
                got.append(out.clone())
            if not torch.equal(got[0], got[1]):
                sys.exit("%s: the level object and the level context's object differ at N = %d" % (name, N))
            for f in (lvl, ref, lvl, ref):   # warm-up
                f()
            torch.cuda.synchronize()
            est = {f: timed(f, 1) for f in (lvl, ref)}
            ts = {f: [] for f in est}
            for _ in range(5):   # alternate the arms
                for f in (lvl, ref):
                    ts[f].append(timed(f, max(1, int(args.min_seconds / 5 / est[f]) + 1)))
            s = {f: sorted(v)[len(v) // 2] for f, v in ts.items()}
            row = {"log_n": log_n, "batch": B, "object": name, "level_s": s[lvl], "context_s": s[ref]}
            result["rows"].append(row)
            print("%14s %12.6f %12.6f %8.3f" % (name, s[lvl], s[ref], s[lvl] / s[ref]))
        for lvl_o, ref_o in objs.values():
            lvl_o.close()
            ref_o.close()
        cl.close()
        del ct, out
        torch.cuda.empty_cache()

        # device memory of a two-layer network: a top-level layer and a layer at level l, batch B.  The layers' diagonals and keys with
        # their companions are not in dpfhe_context_device_bytes: they are added here, as the objects hold them.
        def layer_bytes(limbs, key_rows, dnum):
            return baby * giant * limbs * N * 8 + 2 * baby * dnum * 2 * key_rows * N * 8

        dnum_top, dnum_l = c.grouped_digits(K), -(-l // K)
        full = torch.empty((B, 2, L, N), **i64)
        c.fill_uniform(5, full, B * 2)
        x_top, x_l = full[:, :, :Lq].contiguous(), full[:, :, :l].contiguous()
        del full
        dtop = np.zeros((baby * giant, Lq, N), dtype=np.uint64)
        torch.cuda.synchronize()
        c2 = dp.Context(log_n, L)
        top = dp.LinearLayer.grouped(c2, K, dtop, baby, np.ascontiguousarray(lk[:baby - 1]), lk[baby - 1], t)
        lvl = dp.LinearLayer.grouped(c2, K, diags, baby, np.ascontiguousarray(lk[:baby - 1]), lk[baby - 1], t, level=l)
        top.apply(x_top, torch.empty_like(x_top), B)
        lvl.apply(x_l, torch.empty_like(x_l), B)
        torch.cuda.synchronize()
        one = c2.device_bytes() + layer_bytes(Lq, L, dnum_top) + layer_bytes(l, L, dnum_top)
        top.close(), lvl.close(), c2.close()
        torch.cuda.empty_cache()
        c3, c4 = dp.Context(log_n, L), dp.Context(log_n, l + K, mods[:l] + mods[Lq:])
        top = dp.LinearLayer.grouped(c3, K, dtop, baby, np.ascontiguousarray(lk[:baby - 1]), lk[baby - 1], t)
        lvl = dp.LinearLayer.grouped(c4, K, diags, baby, np.ascontiguousarray(lk_low[:baby - 1]), lk_low[baby - 1], t)
        top.apply(x_top, torch.empty_like(x_top), B)
        lvl.apply(x_l, torch.empty_like(x_l), B)
        torch.cuda.synchronize()
        two = c3.device_bytes() + c4.device_bytes() + layer_bytes(Lq, L, dnum_top) + layer_bytes(l, l + K, dnum_l)
        top.close(), lvl.close(), c3.close(), c4.close()
        result["memory"].append({"log_n": log_n, "batch": B, "one_context_bytes": one, "two_context_bytes": two})
        print("two layers (levels %d and %d), device bytes with the objects: one context %d (%.1f MiB), a context per level %d (%.1f MiB)"
              % (Lq, l, one, one / 2**20, two, two / 2**20))
        c.close()
        del x_top, x_l
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
