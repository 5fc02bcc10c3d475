"""Compact result ciphertexts (DESIGN.md section 2.24) against full ones, N = 8192 with 4 + 2 limbs and 4096 ciphertexts: the bytes of one
ciphertext in each form (from the shapes); the compaction on the device (dpfhe_compact_ciphertexts, device to device, beside a device
copy of the ciphertexts it reads); the download of the results to pinned host memory (a full device-to-host copy of [n][2][l][N]
against dpfhe_download_compact_ciphertexts); and the client's decryption (dpfhe_decrypt_compact against dpfhe_decrypt_level at level 1
of full level-1 ciphertexts).  BGV at level 1 and level 3, CKKS (limb 0) at level 3, bits = 32.  The two arms of each comparison
alternate; each prints its median over the repetitions, the card and its power limit.  One JSON line per comparison.

    python tools/bench_compact.py [--reps 7] [--n 4096]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_seeded import card, compare, timed_dev, timed_host  # noqa: E402

SEED = bytes(range(32))
LOG_N, LQ, K, BITS = 13, 4, 2, 32
CASES = [(1, 65537), (3, 65537), (3, 0)]   # (level, t_plain)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=4096)
    args = ap.parse_args()
    import torch

    import deeppowers_b200 as dp
    assert torch.cuda.is_available(), "bench_compact needs a CUDA device; the library has no CPU fallback"
    gpu, limit = card()
    n, L, N = args.n, LQ + K, 1 << LOG_N
    ctx = dp.Context(LOG_N, L)
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    ctx.generate_secret(SEED, sk)
    W = ctx.compact_words(BITS)
    out = torch.empty((n, W), dtype=torch.int64, device="cuda")
    h_out = torch.empty((n, W), dtype=torch.int64, pin_memory=True)
    h_out_np = h_out.numpy().view(np.uint64)
    for level, t in CASES:
        extra = {"gpu": gpu, "power_limit": limit, "N": N, "level": level, "t_plain": t, "bits": BITS, "ciphertexts": n,
                 "full_bytes_per_ct": 16 * level * N, "compact_bytes_per_ct": N * BITS // 4}
        pt = torch.zeros((n, level, N), dtype=torch.int64, device="cuda")
        ct = torch.empty((n, 2, level, N), dtype=torch.int64, device="cuda")
        ctx.encrypt_level(level, t, sk, SEED, 0, pt, ct, n)
        del pt
        h_ct = torch.empty(ct.shape, dtype=torch.int64, pin_memory=True)
        ctx.compact_ciphertexts(level, BITS, t, ct, out, n)
        ctx.download_compact_ciphertexts(level, BITS, t, ct, h_out_np, n)
        torch.cuda.synchronize()
        assert torch.equal(h_out, out.cpu()), "the download differs from the device compaction"

        def full_d2h():
            h_ct.copy_(ct, non_blocking=True)
            torch.cuda.synchronize()

        def compact_d2h():
            ctx.download_compact_ciphertexts(level, BITS, t, ct, h_out_np, n)

        d2d = torch.empty_like(ct)   # the yardstick of the compaction kernels: one device copy of the ciphertexts they read
        compare("compaction kernels, device to device (level %d, t %d)" % (level, t),
                [("full_copy_d2d", lambda: d2d.copy_(ct), 0), ("compact", lambda: ctx.compact_ciphertexts(level, BITS, t, ct, out, n), 0)],
                args.reps, timed_dev, extra)
        del d2d
        compare("results to the host (level %d, t %d)" % (level, t),
                [("full_d2h", full_d2h, ct.numel() * 8), ("download_compact", compact_d2h, out.numel() * 8)], args.reps, timed_host, extra)
        del h_ct
        if level == 1:
            pt1 = torch.empty((n, 1, N), dtype=torch.int64, device="cuda")
            compare("client decryption (t %d)" % t,
                    [("decrypt_level1", lambda: ctx.decrypt_level(1, sk, ct, 2, pt1, n), 0),
                     ("decrypt_compact", lambda: ctx.decrypt_compact(BITS, t, sk, out, pt1, n), 0)], args.reps, timed_dev, extra)
            del pt1
        del ct
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
