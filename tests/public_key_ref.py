"""Public keys and public-key encryption of DESIGN.md section 2.14, restated around the oracle's transforms and pointwise operations
(TEST INFRASTRUCTURE ONLY).  The samplers and the nonce word come from tests/keys_ref.c through tests/keys_ref.py, which share no code
with the product; what the GPU is compared with, bit for bit."""
import numpy as np

import keys_ref as kr

PK_A, PK_E, PENC_U, PENC_E0, PENC_E1 = 6, 7, 8, 9, 10


def _neg(o, x):
    q = np.array(o.moduli, dtype=np.uint64)[:, None]
    return (q - x) % q


def public_keygen(o, t_plain, s, seed):
    """the public key (b, a) [2][L][N] = (-a s + t NTT(e), a) under oracle context o and the first o.L rows of s, with a and e
    from domains 6 / 7 and item 0 of the key owner's seed"""
    s = np.ascontiguousarray(s[:o.L])
    a = np.stack([kr.uniform(seed, kr.nonce0(PK_A, 0, 0, l), 0, o.moduli[l], o.N) for l in range(o.L)])
    e = kr.small_eval(o, kr.cbd(seed, kr.nonce0(PK_E), 0, o.N), t_plain)
    return np.stack([o.poly_add(e, _neg(o, o.poly_mul_pointwise(a, s))), a])


def encrypt_public(o, t_plain, pk, seed, first_index, pt):
    """pt [n][L][N] -> ct [n][2][L][N] = (b NTT(u) + t NTT(e0) + pt, a NTT(u) + t NTT(e1)) under the first o.L rows of both
    components of pk; u, e0, e1 from domains 8 / 9 / 10 of the encryptor's seed, item first_index + k"""
    pt = np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, o.L, o.N)
    b, a = np.ascontiguousarray(pk[0][:o.L]), np.ascontiguousarray(pk[1][:o.L])
    ct = np.empty((pt.shape[0], 2, o.L, o.N), dtype=np.uint64)
    for k in range(pt.shape[0]):
        item = first_index + k
        u = kr.small_eval(o, kr.ternary(seed, kr.nonce0(PENC_U), item, o.N), 1)
        e0 = kr.small_eval(o, kr.cbd(seed, kr.nonce0(PENC_E0), item, o.N), t_plain)
        e1 = kr.small_eval(o, kr.cbd(seed, kr.nonce0(PENC_E1), item, o.N), t_plain)
        ct[k, 0] = o.poly_add(o.poly_add(o.poly_mul_pointwise(b, u), e0), pt[k])
        ct[k, 1] = o.poly_add(o.poly_mul_pointwise(a, u), e1)
    return ct
