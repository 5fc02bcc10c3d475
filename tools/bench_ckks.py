"""CKKS slot encoding rates (DESIGN.md section 6): encode and decode vectors per second next to the forward and inverse transforms
of the same [n][L][N] shape, CUDA-event timed, with the GPU's name and power limit.  Prints one JSON line per configuration.

    python tools/bench_ckks.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402

# config 4 of BASELINE.json encodes 768 diagonal plaintexts per level at N = 8192, L = 4
CONFIGS = [(13, 4, 768), (13, 4, 4096), (14, 8, 768)]


def time_ms(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these rates can only be measured on the GPU")
    name, power = gpu_info()
    for log_n, L, n in CONFIGS:
        N = 1 << log_n
        ctx = dp.Context(log_n, L)
        g = torch.Generator(device="cuda").manual_seed(1)
        z = torch.complex(torch.rand((n, N // 2), dtype=torch.float64, device="cuda", generator=g) * 2 - 1,
                          torch.rand((n, N // 2), dtype=torch.float64, device="cuda", generator=g) * 2 - 1)
        pt = torch.empty((n, L, N), dtype=torch.int64, device="cuda")
        out = torch.empty_like(z)
        scale = 2.0**40
        enc = time_ms(lambda: ctx.ckks_encode(z, pt, n, scale), args.iters)
        dec = time_ms(lambda: ctx.ckks_decode(pt, out, n, scale), args.iters)
        work = pt.clone()
        fwd = time_ms(lambda: ctx.ntt_fwd(work, n), args.iters)
        inv = time_ms(lambda: ctx.ntt_inv(work, n), args.iters)
        err = float((out - z).abs().max())
        print(json.dumps({"gpu": name, "power_limit": power, "log_n": log_n, "L": L, "vectors": n,
                          "encode_ms": round(enc, 4), "encode_vec_per_s": round(n / enc * 1e3),
                          "decode_ms": round(dec, 4), "decode_vec_per_s": round(n / dec * 1e3),
                          "ntt_fwd_ms": round(fwd, 4), "ntt_inv_ms": round(inv, 4), "round_trip_max_error": err}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
