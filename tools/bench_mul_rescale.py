"""Multiply-and-rescale (DESIGN.md section 2.19) on one GPU: seconds per call of the fused calls against the composition they replace,
  ct x ct: dpfhe_ct_mul_relin_rescale_grouped   against dpfhe_ct_mul_relin_grouped + dpfhe_mod_switch_down
  n pairs: dpfhe_ct_dot_rescale_grouped         against dpfhe_ct_dot_grouped + dpfhe_mod_switch_down
(the modulus switch on a context over the ciphertext moduli).  The arms are warmed up, then alternated in one run, with CUDA events
around at least --min-seconds of work per arm.  Before timing, both arms' outputs at the timed size are decrypted and decoded (BGV,
t = 65537: the fused and the composed slots must be equal); the timed calls run with t = --t on uniform operands.
The card's name and power limit are printed with the numbers.

    python tools/bench_mul_rescale.py [--log-n 13] [--limbs 4] [--special 2] [--batches 512,4096] [--terms 4,64] [--t 0] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=13)
    ap.add_argument("--limbs", type=int, default=4)
    ap.add_argument("--special", type=int, default=2)
    ap.add_argument("--batches", default="512,4096")
    ap.add_argument("--terms", default="4,64")
    ap.add_argument("--t", type=int, default=0)
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import deeppowers_b200 as dp
    if not torch.cuda.is_available():
        sys.exit("bench_mul_rescale.py needs a CUDA device; there is no CPU fallback and no number without one")
    Lq, K = args.limbs, args.special
    L = Lq + K
    c = dp.Context(args.log_n, L)
    cq = dp.Context(args.log_n, Lq, c.moduli[:Lq])
    cl = dp.Context(args.log_n, Lq - 1, c.moduli[:Lq - 1])
    N, t = c.N, args.t
    i64 = dict(dtype=torch.int64, device="cuda")
    batches = [int(x) for x in args.batches.split(",")]
    terms = [int(x) for x in args.terms.split(",")]
    B_max, n_max = max(batches), max(terms)
    # distinct operands, so that a call reads what a real one does: two batches of the largest size for ct x ct, and 2 n_max of the
    # first batch size for the pairs (the inner products run at that size)
    ab = torch.empty((2, B_max, 2, Lq, N), **i64)
    cq.fill_uniform(1, ab, 2 * B_max * 2)
    ops = torch.empty((2 * n_max, batches[0], 2, Lq, N), **i64)
    cq.fill_uniform(3, ops, 2 * n_max * batches[0] * 2)
    key = torch.empty((c.grouped_digits(K), 2, L, N), **i64)
    c.fill_uniform(2, key, key.shape[0] * 2)

    # the decoded check: BGV, t = 65537, two encrypted batches at the timed size (the pairs repeat them), both arms
    def decoded_check(B, n):
        tc = 65537
        sk = torch.empty((L, N), **i64)
        c.generate_secret(bytes(range(32)), sk)
        evk = torch.empty_like(key)
        c.generate_relin_key(K, tc, sk, bytes(range(1, 33)), evk)
        rng = np.random.default_rng(3)
        m = torch.from_numpy(rng.integers(-8, 8, size=(2 * B, N), dtype=np.int64)).cuda()
        pt = torch.empty((2 * B, Lq, N), **i64)
        cq.bgv_encode(m, pt, 2 * B, tc)
        ct = torch.empty((2, B, 2, Lq, N), **i64)
        cq.encrypt(tc, sk[:Lq].contiguous(), bytes(range(2, 34)), 0, pt, ct.view(2 * B, 2, Lq, N), 2 * B)
        fused, mid, comp = torch.empty((B, 2, Lq - 1, N), **i64), torch.empty((B, 2, Lq, N), **i64), torch.empty((B, 2, Lq - 1, N), **i64)
        if n == 1:
            c.ct_mul_relin_rescale_grouped(K, ct[0], ct[1], evk, fused, B, tc)
            c.ct_mul_relin_grouped(K, ct[0], ct[1], evk, mid, B, tc)
        else:
            c.ct_dot_rescale_grouped(K, [ct[0]] * n, [ct[1]] * n, evk, fused, B, tc)
            c.ct_dot_grouped(K, [ct[0]] * n, [ct[1]] * n, evk, mid, B, tc)
        cq.mod_switch_down(mid, comp, 2 * B, tc)
        out = []
        for x in (fused, comp):
            ph = torch.empty((B, Lq - 1, N), **i64)
            cl.decrypt(sk[:Lq - 1].contiguous(), x, 2, ph, B)
            s = torch.empty((B, N), **i64)
            cl.bgv_decode(ph, s, B, tc)
            out.append(s)
        if not torch.equal(out[0], out[1]):
            sys.exit("the fused and the composed results decode differently (B = %d, n = %d)" % (B, n))
        del sk, evk, m, pt, ct, fused, mid, comp

    def timed(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    cases = [(B, 1) for B in batches] + [(batches[0], n) for n in terms]
    rows = []
    print("card: %s; N = %d, Lq = %d, K = %d, t = %d" % (card(), N, Lq, K, t))
    print("%6s %5s %12s %12s %8s %14s" % ("batch", "pairs", "fused s", "composed s", "speedup", "fused ct/s"))
    for B, n in cases:
        decoded_check(B, n)
        out, mid, low = torch.empty((B, 2, Lq - 1, N), **i64), torch.empty((B, 2, Lq, N), **i64), torch.empty((B, 2, Lq - 1, N), **i64)
        a_list, b_list = ([ab[0][:B]], [ab[1][:B]]) if n == 1 else ([ops[i][:B] for i in range(n)], [ops[n_max + i][:B] for i in range(n)])

        def fused():
            if n == 1:
                c.ct_mul_relin_rescale_grouped(K, a_list[0], b_list[0], key, out, B, t)
            else:
                c.ct_dot_rescale_grouped(K, a_list, b_list, key, out, B, t)

        def composed():
            if n == 1:
                c.ct_mul_relin_grouped(K, a_list[0], b_list[0], key, mid, B, t)
            else:
                c.ct_dot_grouped(K, a_list, b_list, key, mid, B, t)
            cq.mod_switch_down(mid, low, 2 * B, t)

        for f in (fused, composed, fused, composed):   # warm-up
            f()
        torch.cuda.synchronize()
        est = {f: timed(f, 1) for f in (fused, composed)}
        ts = {f: [] for f in est}
        for _ in range(5):   # alternate the arms
            for f in (fused, composed):
                ts[f].append(timed(f, max(1, int(args.min_seconds / 5 / est[f]) + 1)))
        s = {f: sorted(v)[len(v) // 2] for f, v in ts.items()}   # medians
        row = {"batch": B, "pairs": n, "fused_s": s[fused], "composed_s": s[composed], "fused_ct_per_s": B / s[fused]}
        rows.append(row)
        print("%6d %5d %12.6f %12.6f %7.2fx %14.0f" % (B, n, s[fused], s[composed], s[composed] / s[fused], row["fused_ct_per_s"]))
        del out, mid, low
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "log_n": args.log_n, "Lq": Lq, "K": K, "t": t, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
