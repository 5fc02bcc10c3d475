"""Seeded ciphertexts and switch keys of DESIGN.md section 2.23, restated by composing tests/keys_ref.py's samplers with an explicit
(a-key, a-domain, e-domain) (TEST INFRASTRUCTURE ONLY).  With the key owner's seed as a-key and the domains (4, 5) / (2, 3) the forms
below are keys_ref.encrypt / keys_ref.switch_key; with the public seed and (12, 13) / (14, 15) they are the seeded objects the GPU
is compared with, bit for bit."""
import numpy as np

import keys_ref as kr

PUBLIC_SEED, SENC_A, SENC_E, SKEY_A, SKEY_E = 11, 12, 13, 14, 15


def public_seed(seed):
    """words 0..7 (little-endian bytes) of the ChaCha20 block of the key owner's seed at counter 0, nonce (11, 0, 0)"""
    w = kr.chacha20_block(seed, 0, [kr.nonce0(PUBLIC_SEED), 0, 0])
    return w[:8].astype("<u4").tobytes()


def encrypt_with(o, t_plain, s, a_key, e_key, a_dom, e_dom, first_index, pt):
    """[n][2][L][N]: c0 = -a s + t NTT(e) + pt, c1 = a; a from (a_key, a_dom, limb), e from (e_key, e_dom), item first_index + k"""
    pt = np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, o.L, o.N)
    s = np.ascontiguousarray(s[:o.L])
    ct = np.empty((pt.shape[0], 2, o.L, o.N), dtype=np.uint64)
    for k in range(pt.shape[0]):
        item = first_index + k
        a = kr._uniform_rows(o, a_key, a_dom, 0, 0, item)
        e = kr.small_eval(o, kr.cbd(e_key, kr.nonce0(e_dom), item, o.N), t_plain)
        ct[k, 0] = o.poly_add(o.poly_add(e, kr._neg(o, o.poly_mul_pointwise(a, s))), pt[k])
        ct[k, 1] = a
    return ct


def switch_key_with(o, K, t_plain, s, a_key, e_key, a_dom, e_dom, target, item):
    """[digits][2][L][N]: b_j = -a_j s + t NTT(e_j) + gadget_j target, a_j from (a_key, a_dom, K, j, limb), e_j from (e_key, e_dom, K, j)"""
    L, N = o.L, o.N
    Lq = L - K
    P = 1
    for m in o.moduli[Lq:]:
        P *= m
    nd = kr.digits(o, K)
    key = np.empty((nd, 2, L, N), dtype=np.uint64)
    for j in range(nd):
        a = kr._uniform_rows(o, a_key, a_dom, K, j, item)
        e = kr.small_eval(o, kr.cbd(e_key, kr.nonce0(e_dom, K, j), item, N), t_plain)
        b = o.poly_add(e, kr._neg(o, o.poly_mul_pointwise(a, s)))
        limbs = [j] if K == 0 else [l for l in range(Lq) if l // K == j]
        fac = [(P % int(o.moduli[l])) if (K and l in limbs) else (1 if l in limbs else 0) for l in range(L)]
        b = o.poly_add(b, o.poly_mul_pointwise(target, kr._limb_const(o, fac)))
        key[j, 0], key[j, 1] = b, a
    return key


def encrypt_seeded(o, t_plain, s, seed, first_index, pt):
    """the expanded seeded ciphertexts [n][2][L][N]; c0 alone is [:, 0]"""
    return encrypt_with(o, t_plain, s, public_seed(seed), seed, SENC_A, SENC_E, first_index, pt)


def relin_key_seeded(o, K, t_plain, s, seed):
    """the expanded seeded relinearisation key [digits][2][L][N]; the b rows alone are [:, 0]"""
    return switch_key_with(o, K, t_plain, s, public_seed(seed), seed, SKEY_A, SKEY_E, o.poly_mul_pointwise(s, s), 0)


def galois_keys_seeded(o, K, t_plain, s, seed, elts):
    out = []
    for g in elts:
        perm = o.galois_perm(g)
        out.append(switch_key_with(o, K, t_plain, s, public_seed(seed), seed, SKEY_A, SKEY_E, np.ascontiguousarray(s[:, perm]), int(g)))
    return np.stack(out)


def expand_ciphertexts(o, a_seed, first_index, c0):
    """c0 [n][L][N] -> [n][2][L][N] with c1 regenerated from a_seed"""
    c0 = np.ascontiguousarray(c0, dtype=np.uint64).reshape(-1, o.L, o.N)
    out = np.empty((c0.shape[0], 2, o.L, o.N), dtype=np.uint64)
    for k in range(c0.shape[0]):
        out[k, 0] = c0[k]
        out[k, 1] = kr._uniform_rows(o, a_seed, SENC_A, 0, 0, first_index + k)
    return out


def expand_switch_keys(o, K, a_seed, items, b):
    """b [n_keys][digits][L][N] -> [n_keys][digits][2][L][N] with a_j regenerated from a_seed and each key's item number"""
    nd = kr.digits(o, K)
    b = np.ascontiguousarray(b, dtype=np.uint64).reshape(len(items), nd, o.L, o.N)
    out = np.empty((len(items), nd, 2, o.L, o.N), dtype=np.uint64)
    for e, item in enumerate(items):
        for j in range(nd):
            out[e, j, 0] = b[e, j]
            out[e, j, 1] = kr._uniform_rows(o, a_seed, SKEY_A, K, j, int(item))
    return out
