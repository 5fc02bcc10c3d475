"""Key generation, encryption and decryption rates (DESIGN.md section 6), CUDA-event timed, with the GPU's name and power limit:
encryption and decryption of a batch next to the forward transform of the same [n][L][N] shape, the 26 Galois keys of config 3
(N = 16384, L = 8, per-limb digits, 16 MiB each), the 32 grouped Galois keys of config 4 (N = 8192, 4 + 2 limbs, K = 2), and
the oracle's single-threaded CPU key generation of the same keys as the baseline.  Prints one JSON line per measurement.

    python tools/bench_keys.py [--iters 10] [--oracle-keys 2]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import deeppowers_b200 as dp  # noqa: E402
from bench_ckks import gpu_info, time_ms  # noqa: E402

SEED = bytes(range(32))
T_PLAIN = 65537


def oracle_keys_s(log_n, L, K, elts, t):
    """seconds the oracle (one thread) takes for Galois keys of `elts`"""
    from oracle import Oracle
    o = Oracle(log_n, L)
    s = o.keygen_secret(1)
    t0 = time.perf_counter()
    for i, g in enumerate(elts):
        if K:
            o.keygen_galois_grouped(K, 10 + i, t, s, g)
        else:
            o.keygen_galois(10 + i, t, s, g)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--oracle-keys", type=int, default=2, help="config-3 keys the oracle generates (its time is per key)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these rates can only be measured on the GPU")
    name, power = gpu_info()
    base = {"gpu": name, "power_limit": power}

    # encryption / decryption at N = 8192, L = 4, batch 4096
    log_n, L, n = 13, 4, 4096
    N = 1 << log_n
    ctx = dp.Context(log_n, L)
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    ctx.generate_secret(SEED, sk)
    pt = torch.empty((n, L, N), dtype=torch.int64, device="cuda")
    ctx.fill_uniform(3, pt, n)
    ct = torch.empty((n, 2, L, N), dtype=torch.int64, device="cuda")
    enc = time_ms(lambda: ctx.encrypt(T_PLAIN, sk, SEED, 0, pt, ct, n), args.iters)
    dec = time_ms(lambda: ctx.decrypt(sk, ct, 2, pt, n), args.iters)
    work = pt.clone()
    fwd = time_ms(lambda: ctx.ntt_fwd(work, n), args.iters)
    print(json.dumps(dict(base, op="encrypt/decrypt", log_n=log_n, L=L, batch=n, encrypt_ms=round(enc, 3), encrypt_ct_per_s=round(n / enc * 1e3),
                          decrypt_ms=round(dec, 3), decrypt_ct_per_s=round(n / dec * 1e3), ntt_fwd_ms=round(fwd, 3))), flush=True)
    ctx.close()

    # config 3: 26 per-limb-digit Galois keys at N = 16384, L = 8; config 4: 32 grouped keys, N = 8192, 4 + 2 limbs, K = 2
    for cfg, log_n, L, K, n_keys in (("config3", 14, 8, 0, 26), ("config4", 13, 6, 2, 32)):
        N = 1 << log_n
        ctx = dp.Context(log_n, L)
        sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
        ctx.generate_secret(SEED, sk)
        elts = [ctx.galois_elt(k) for k in range(1, n_keys + 1)]
        nd = ctx.key_digits(K)
        keys = torch.empty((n_keys, nd, 2, L, N), dtype=torch.int64, device="cuda")
        gpu = time_ms(lambda: ctx.generate_galois_keys(K, T_PLAIN, sk, elts, SEED, keys), args.iters)
        work = torch.empty((n_keys * nd * 2, L, N), dtype=torch.int64, device="cuda")
        ctx.fill_uniform(4, work, n_keys * nd * 2)
        fwd = time_ms(lambda: ctx.ntt_fwd(work, n_keys * nd * 2), args.iters)
        n_oracle = n_keys if K else min(args.oracle_keys, n_keys)
        cpu_s = oracle_keys_s(log_n, L, K, elts[:n_oracle], T_PLAIN)
        print(json.dumps(dict(base, op="galois_keygen", config=cfg, log_n=log_n, L=L, n_special=K, keys=n_keys,
                              key_mib=round(nd * 2 * L * N * 8 / 2**20, 2), gpu_ms=round(gpu, 3), ntt_fwd_same_shape_ms=round(fwd, 3),
                              oracle_keys_timed=n_oracle, oracle_s_per_key=round(cpu_s / n_oracle, 3),
                              speedup_vs_oracle=round(cpu_s / n_oracle * n_keys * 1e3 / gpu))), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
