"""Seeded ciphertexts and keys (DESIGN.md section 2.23) against full ones, on pinned host memory: fresh ciphertexts landed on the
device per second (a full copy of [n][2][Lq][N] against dpfhe_upload_seeded_ciphertexts of [n][Lq][N]), the expansion kernel alone
(device to device), dpfhe_encrypt_seeded against dpfhe_encrypt, and 32 grouped Galois keys uploaded full and seeded.  N = 8192 with
4 + 2 limbs and N = 16384 with 8 + 4.  The two arms of each comparison alternate; each prints its median over the repetitions, the
bytes it moves over the bus, the card and its power limit.  One JSON line per comparison.

    python tools/bench_seeded.py [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = bytes(range(32))
CASES = [(13, 4, 2, 1024), (14, 8, 4, 256)]   # (log N, Lq, K, ciphertexts): 512 MiB of full ciphertexts each
N_KEYS = 32


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed_host(fn):
    """seconds of fn(), which ends in a device synchronise"""
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def timed_dev(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def compare(name, arms, reps, timer, extra):
    """arms: [(label, fn, bytes over the bus)]; alternated, one warm-up each"""
    for _, fn, _ in arms:
        timer(fn)
    t = {label: [] for label, _, _ in arms}
    for _ in range(reps):
        for label, fn, _ in arms:
            t[label].append(timer(fn))
    out = dict(extra, bench=name)
    for label, _, nbytes in arms:
        med = float(np.median(t[label]))
        out[label] = {"median_ms": round(med * 1e3, 3), "spread_ms": round((max(t[label]) - min(t[label])) * 1e3, 3), "bus_bytes": nbytes}
    labels = [a[0] for a in arms]
    out["speedup"] = round(out[labels[0]]["median_ms"] / out[labels[1]]["median_ms"], 3)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch

    import deeppowers_b200 as dp
    assert torch.cuda.is_available(), "bench_seeded needs a CUDA device; the library has no CPU fallback"
    gpu, limit = card()
    for log_n, Lq, K, n in CASES:
        L, N = Lq + K, 1 << log_n
        ctx = dp.Context(log_n, L)
        extra = {"gpu": gpu, "power_limit": limit, "N": N, "Lq": Lq, "K": K}
        sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
        ctx.generate_secret(SEED, sk)
        a_seed = dp.public_seed(SEED)
        pt = torch.empty((n, Lq, N), dtype=torch.int64, device="cuda")
        pt.zero_()   # the plaintext does not change what either encryption costs
        c0 = torch.empty((n, Lq, N), dtype=torch.int64, device="cuda")
        ctx.encrypt_seeded_level(Lq, 65537, sk, SEED, 0, pt, c0, n)
        ct = torch.empty((n, 2, Lq, N), dtype=torch.int64, device="cuda")
        ctx.expand_ciphertexts_level(Lq, a_seed, 0, c0, ct, n)
        h_ct = torch.empty((n, 2, Lq, N), dtype=torch.int64, pin_memory=True)
        h_ct.copy_(ct)
        h_c0 = torch.empty((n, Lq, N), dtype=torch.int64, pin_memory=True)
        h_c0.copy_(c0)
        h_c0_np = h_c0.numpy().view(np.uint64)
        dst = torch.empty_like(ct)
        torch.cuda.synchronize()

        def full_copy():
            dst.copy_(h_ct, non_blocking=True)
            torch.cuda.synchronize()

        def seeded_upload():
            ctx.upload_seeded_ciphertexts_level(Lq, a_seed, 0, h_c0_np, dst)

        seeded_upload()
        assert torch.equal(dst, ct), "the seeded upload differs from the expansion"
        compare("fresh ciphertexts to the device (%d)" % n, [("full_copy", full_copy, h_ct.numel() * 8), ("seeded_upload", seeded_upload, h_c0.numel() * 8)],
                args.reps, timed_host, dict(extra, ciphertexts=n))
        compare("expansion, device to device (%d)" % n,
                [("full_copy_d2d", lambda: dst.copy_(ct), 0), ("expand", lambda: ctx.expand_ciphertexts_level(Lq, a_seed, 0, c0, dst, n), 0)],
                args.reps, timed_dev, dict(extra, ciphertexts=n, expand_bytes_written=ct.numel() * 8, expand_bytes_read=c0.numel() * 8))
        compare("encryption (%d)" % n,
                [("encrypt", lambda: ctx.encrypt_level(Lq, 65537, sk, SEED, 0, pt, dst, n), 0),
                 ("encrypt_seeded", lambda: ctx.encrypt_seeded_level(Lq, 65537, sk, SEED, 0, pt, c0, n), 0)],
                args.reps, timed_dev, dict(extra, ciphertexts=n))
        del h_ct, h_c0, dst, ct
        torch.cuda.empty_cache()
        # 32 grouped Galois keys
        dnum = ctx.key_digits(K)
        elts = [ctx.galois_elt(k) for k in range(1, N_KEYS + 1)]
        b = torch.empty((N_KEYS, dnum, L, N), dtype=torch.int64, device="cuda")
        ctx.generate_galois_keys_seeded(K, 65537, sk, elts, SEED, b)
        keys = torch.empty((N_KEYS, dnum, 2, L, N), dtype=torch.int64, device="cuda")
        ctx.expand_switch_keys(K, a_seed, elts, b, keys)
        h_keys = torch.empty(keys.shape, dtype=torch.int64, pin_memory=True)
        h_keys.copy_(keys)
        h_b = torch.empty(b.shape, dtype=torch.int64, pin_memory=True)
        h_b.copy_(b)
        h_b_np = h_b.numpy().view(np.uint64)
        kdst = torch.empty_like(keys)
        torch.cuda.synchronize()

        def keys_full():
            kdst.copy_(h_keys, non_blocking=True)
            torch.cuda.synchronize()

        def keys_seeded():
            ctx.upload_seeded_switch_keys(K, a_seed, elts, h_b_np, kdst)

        keys_seeded()
        assert torch.equal(kdst, keys), "the seeded key upload differs from the expansion"
        compare("%d grouped Galois keys to the device" % N_KEYS,
                [("full_copy", keys_full, h_keys.numel() * 8), ("seeded_upload", keys_seeded, h_b.numel() * 8)], args.reps, timed_host,
                dict(extra, keys=N_KEYS, key_bytes=keys[0].numel() * 8))
        del h_keys, h_b, kdst, keys, b
        ctx.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
