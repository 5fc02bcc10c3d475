"""BGV slot encoding rates (DESIGN.md section 6): encode and decode vectors per second next to the forward and inverse transforms
of the same [n][L][N] shape, CUDA-event timed, with the GPU's name and power limit.  Prints one JSON line per configuration.

    python tools/bench_bgv.py [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402
from bench_ckks import gpu_info, time_ms  # noqa: E402

# config 4 of BASELINE.json encodes 768 diagonal plaintexts per level at N = 8192, L = 4, with t = 167772161
CONFIGS = [(13, 4, 768), (13, 4, 4096), (14, 8, 768)]
T_PLAIN = 167772161


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
        z = torch.randint(-128, 128, (n, 2, N // 2), dtype=torch.int64, device="cuda", generator=g)
        pt = torch.empty((n, L, N), dtype=torch.int64, device="cuda")
        out = torch.empty_like(z)
        enc = time_ms(lambda: ctx.bgv_encode(z, pt, n, T_PLAIN), args.iters)
        dec = time_ms(lambda: ctx.bgv_decode(pt, out, n, T_PLAIN), args.iters)
        work = pt.clone()
        fwd = time_ms(lambda: ctx.ntt_fwd(work, n), args.iters)
        inv = time_ms(lambda: ctx.ntt_inv(work, n), args.iters)
        exact = bool(torch.equal(out, z % T_PLAIN))
        print(json.dumps({"gpu": name, "power_limit": power, "log_n": log_n, "L": L, "vectors": n, "t_plain": T_PLAIN,
                          "encode_ms": round(enc, 4), "encode_vec_per_s": round(n / enc * 1e3),
                          "decode_ms": round(dec, 4), "decode_vec_per_s": round(n / dec * 1e3),
                          "ntt_fwd_ms": round(fwd, 4), "ntt_inv_ms": round(inv, 4), "round_trip_exact": exact}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
