"""Encrypted inner product (DESIGN.md section 2.18) on one GPU: seconds per call of dpfhe_ct_dot_grouped for n pairs against
  (a) n x dpfhe_ct_mul_relin_grouped + one dpfhe_ct_lincomb (what a caller had to do before; same plaintext, not the same bits), and
  (b) the bit-identical device composition (dpfhe_ct_tensor per pair summed with dpfhe_poly_add, dpfhe_keyswitch_grouped, dpfhe_poly_add),
the arms alternated in one run, CUDA events around at least --min-seconds of work per arm after a warm-up; the outputs of the call and
of (b) are compared before anything is timed.  Also printed: pairs per second, and the bytes the call must read (2 n operand
ciphertexts per output + the key once) over its time as a share of the HBM copy rate measured in the same run (a device-to-device
copy of 1 GiB: bytes read plus bytes written over time).  The card's name and power limit are printed with the numbers.

    python tools/bench_ct_dot.py [--log-n 13] [--limbs 4] [--special 2] [--batch 512] [--terms 1,2,4,8,16,32,64] [--json out.json]
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
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--terms", default="1,2,4,8,16,32,64")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    import deeppowers_b200 as dp
    if not torch.cuda.is_available():
        sys.exit("bench_ct_dot.py needs a CUDA device; there is no CPU fallback and no number without one")
    Lq, K, B = args.limbs, args.special, args.batch
    L = Lq + K
    c = dp.Context(args.log_n, L)
    cq = dp.Context(args.log_n, Lq, c.moduli[:Lq])
    N = c.N
    terms = [int(x) for x in args.terms.split(",")]
    n_max = max(terms)
    i64 = dict(dtype=torch.int64, device="cuda")
    # the operands: n_max distinct a_i and b_i (so that the call reads 2 n operands from memory, as a real inner product does)
    ops = torch.empty((2 * n_max, B, 2, Lq, N), **i64)
    cq.fill_uniform(1, ops, 2 * n_max * B * 2)
    key = torch.empty((c.grouped_digits(K), 2, L, N), **i64)
    c.fill_uniform(2, key, key.shape[0] * 2)
    out, ref = torch.empty((B, 2, Lq, N), **i64), torch.empty((B, 2, Lq, N), **i64)
    parts = torch.empty((n_max, B, 2, Lq, N), **i64)
    d, acc3 = torch.empty((B, 3, Lq, N), **i64), torch.empty((B, 3, Lq, N), **i64)
    d2, d01, ks = torch.empty((B, Lq, N), **i64), torch.empty((B, 2, Lq, N), **i64), torch.empty((B, 2, Lq, N), **i64)

    def dot(n):
        c.ct_dot_grouped(K, [ops[i] for i in range(n)], [ops[n_max + i] for i in range(n)], key, out, B, 65537)

    def separate(n):
        for i in range(n):
            c.ct_mul_relin_grouped(K, ops[i], ops[n_max + i], key, parts[i], B, 65537)
        cq.ct_lincomb([parts[i] for i in range(n)], [1] * n, 0, ref, B)

    def composition(n):
        cq.ct_tensor(ops[0], ops[n_max], acc3, B)
        for i in range(1, n):
            cq.ct_tensor(ops[i], ops[n_max + i], d, B)
            cq.poly_add(acc3, d, acc3, 3 * B)
        d2.copy_(acc3[:, 2])
        d01.copy_(acc3[:, :2])
        c.keyswitch_grouped(K, d2, key, ks, B, 65537)
        cq.poly_add(d01, ks, ref, 2 * B)

    def timed(fn, n, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn(n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e-3 / reps

    # HBM copy rate: bytes read + bytes written of a device-to-device copy over its time
    src, dst = torch.empty(1 << 27, **i64), torch.empty(1 << 27, **i64)
    dst.copy_(src)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        dst.copy_(src)
    e1.record()
    torch.cuda.synchronize()
    copy_rate = 20 * 2 * src.numel() * 8 / (e0.elapsed_time(e1) * 1e-3)
    del src, dst

    ct_bytes, key_bytes = 2 * Lq * N * 8, key.numel() * 8
    rows = []
    print("card: %s; N = %d, Lq = %d, K = %d, batch %d; HBM copy rate %.0f GB/s" % (card(), N, Lq, K, B, copy_rate / 1e9))
    print("%5s %12s %12s %12s %8s %8s %12s %10s" % ("n", "dot s", "separate s", "composed s", "vs sep", "vs comp", "pairs/s", "HBM share"))
    for n in terms:
        dot(n)
        composition(n)
        torch.cuda.synchronize()
        if not torch.equal(out, ref):
            sys.exit("the call and the device composition differ at n = %d" % n)
        separate(n)   # warm-up of the third arm
        torch.cuda.synchronize()
        est = {f: timed(f, n, 1) for f in (dot, separate, composition)}
        t = {f: [] for f in est}
        for _ in range(3):   # alternate the arms
            for f in (dot, separate, composition):
                t[f].append(timed(f, n, max(1, int(args.min_seconds / 3 / est[f]) + 1)))
        s = {f: sum(v) / len(v) for f, v in t.items()}
        must_read = B * 2 * n * ct_bytes + key_bytes
        row = {"n": n, "dot_s": s[dot], "separate_s": s[separate], "composition_s": s[composition], "pairs_per_s": n * B / s[dot],
               "hbm_share": must_read / s[dot] / copy_rate}
        rows.append(row)
        print("%5d %12.6f %12.6f %12.6f %7.2fx %7.2fx %12.0f %9.1f%%" % (n, s[dot], s[separate], s[composition], s[separate] / s[dot],
                                                                         s[composition] / s[dot], row["pairs_per_s"], 100 * row["hbm_share"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "log_n": args.log_n, "Lq": Lq, "K": K, "batch": B, "hbm_copy_bytes_per_s": copy_rate, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
