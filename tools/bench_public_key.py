"""Public-key encryption rates (DESIGN.md section 6), CUDA-event timed, with the GPU's name and power limit: dpfhe_encrypt_public of a
batch alternated in one run with dpfhe_encrypt (symmetric) and ntt_fwd of the same [n][L][N] shape, at N = 8192, L = 4, 4096
ciphertexts and at N = 16384, L = 4, 1024 ciphertexts (the CTA-pair kernels).  Each is timed over --iters calls after warm-up, and
the three are alternated --reps times.  Prints one JSON line per shape.

    python tools/bench_public_key.py [--iters 10] [--reps 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402
from bench_ckks import gpu_info, time_ms  # noqa: E402

OWNER = bytes(range(32))
ENCRYPTOR = bytes(range(32, 64))
T_PLAIN = 65537


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these rates can only be measured on the GPU")
    name, power = gpu_info()
    for log_n, L, n in ((13, 4, 4096), (14, 4, 1024)):
        N = 1 << log_n
        ctx = dp.Context(log_n, L)
        sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
        ctx.generate_secret(OWNER, sk)
        pk = torch.empty((2, L, N), dtype=torch.int64, device="cuda")
        ctx.public_keygen(T_PLAIN, sk, OWNER, pk)
        pt = torch.empty((n, L, N), dtype=torch.int64, device="cuda")
        ctx.fill_uniform(3, pt, n)
        ct = torch.empty((n, 2, L, N), dtype=torch.int64, device="cuda")
        work = pt.clone()
        runs = {"public": [], "symmetric": [], "ntt_fwd": []}
        for _ in range(args.reps):
            runs["public"].append(time_ms(lambda: ctx.encrypt_public(T_PLAIN, pk, ENCRYPTOR, 0, pt, ct, n), args.iters))
            runs["symmetric"].append(time_ms(lambda: ctx.encrypt(T_PLAIN, sk, OWNER, 0, pt, ct, n), args.iters))
            runs["ntt_fwd"].append(time_ms(lambda: ctx.ntt_fwd(work, n), args.iters))
        pkg = time_ms(lambda: ctx.public_keygen(T_PLAIN, sk, OWNER, pk), args.iters)
        med = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}
        print(json.dumps(dict(gpu=name, power_limit=power, op="encrypt_public", log_n=log_n, L=L, batch=n,
                              encrypt_public_ms=[round(x, 3) for x in runs["public"]], encrypt_ms=[round(x, 3) for x in runs["symmetric"]],
                              ntt_fwd_ms=[round(x, 3) for x in runs["ntt_fwd"]],
                              encrypt_public_ct_per_s=round(n / med["public"] * 1e3), ratio_to_symmetric=round(med["public"] / med["symmetric"], 2),
                              ratio_to_ntt_fwd=round(med["public"] / med["ntt_fwd"], 2), public_keygen_ms=round(pkg, 4))), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
