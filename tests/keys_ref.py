"""Key generation, encryption and decryption of DESIGN.md section 2.14, restated around the oracle's transforms and pointwise
operations (TEST INFRASTRUCTURE ONLY).  The ChaCha20 rows come from tests/keys_ref.c, which shares no code with the product;
what the GPU is compared with, bit for bit.

The library is built into tests/_emu/ on first use."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "keys_ref.c")
_SO = os.path.join(_HERE, "_emu", "libkeys_ref.so")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_lib = None

SECRET, KEY_A, KEY_E, ENC_A, ENC_E = 1, 2, 3, 4, 5


def lib():
    global _lib
    if _lib is not None:
        return _lib
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    if not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([gcc, "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", _SRC, "-o", _SO])
    L = C.CDLL(_SO)
    L.kr_chacha20_block.argtypes = [C.c_char_p, C.c_uint32, _u32p, _u32p]
    L.kr_nonce0.restype = C.c_uint32
    L.kr_nonce0.argtypes = [C.c_uint32] * 4
    L.kr_ternary.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_size_t, _i64p]
    L.kr_cbd.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_size_t, _i64p]
    L.kr_uniform.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_size_t, _u64p]
    L.kr_reduce128.restype = C.c_uint64
    L.kr_reduce128.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
    _lib = L
    return L


def chacha20_block(key, counter, nonce):
    out = np.empty(16, dtype=np.uint32)
    lib().kr_chacha20_block(bytes(key), counter, np.array(nonce, dtype=np.uint32), out)
    return out


def nonce0(domain, K=0, digit=0, limb=0):
    return int(lib().kr_nonce0(domain, K, digit, limb))


def ternary(seed, n0, item, n):
    out = np.empty(n, dtype=np.int64)
    lib().kr_ternary(bytes(seed), n0, item, n, out)
    return out


def cbd(seed, n0, item, n):
    out = np.empty(n, dtype=np.int64)
    lib().kr_cbd(bytes(seed), n0, item, n, out)
    return out


def uniform(seed, n0, item, q, n):
    out = np.empty(n, dtype=np.uint64)
    lib().kr_uniform(bytes(seed), n0, item, q, n, out)
    return out


def reduce128(lo, hi, q):
    return int(lib().kr_reduce128(lo, hi, q))


def _limb_const(o, values):
    """[L][N] array holding values[l] in every coefficient of limb l"""
    return np.repeat(np.array([int(v) for v in values], dtype=np.uint64)[:, None], o.N, axis=1)


def small_eval(o, v, t_plain):
    """t * v (t = 1 for t_plain = 0) for a small signed integer polynomial v, in evaluation form [L][N]"""
    q = np.array(o.moduli, dtype=np.uint64)[:, None]
    r = np.where(v[None, :] >= 0, v[None, :].astype(np.uint64), q - (-v[None, :]).astype(np.uint64)) % q
    t = t_plain if t_plain else 1
    r = o.poly_mul_pointwise(r, _limb_const(o, [t % int(m) for m in o.moduli]))
    return o.ntt_fwd(r).reshape(o.L, o.N)


def _neg(o, x):
    q = np.array(o.moduli, dtype=np.uint64)[:, None]
    return (q - x) % q


def secret(o, seed):
    """the secret over all limbs of oracle context o: [L][N]"""
    return small_eval(o, ternary(seed, nonce0(SECRET), 0, o.N), 1)


def _uniform_rows(o, seed, domain, K, digit, item):
    return np.stack([uniform(seed, nonce0(domain, K, digit, l), item, o.moduli[l], o.N) for l in range(o.L)])


def digits(o, K):
    return (o.L - K + K - 1) // K if K else o.L


def switch_key(o, K, t_plain, s, seed, target, item):
    """[digits][2][L][N]: b_j = -a_j s + t NTT(e_j) + gadget_j target, a_j (K = 0: per-limb digits, else grouped)"""
    L, N = o.L, o.N
    Lq = L - K
    P = 1
    for m in o.moduli[Lq:]:
        P *= m
    nd = digits(o, K)
    key = np.empty((nd, 2, L, N), dtype=np.uint64)
    for j in range(nd):
        a = _uniform_rows(o, seed, KEY_A, K, j, item)
        e = small_eval(o, cbd(seed, nonce0(KEY_E, K, j), item, N), t_plain)
        b = o.poly_add(e, _neg(o, o.poly_mul_pointwise(a, s)))
        limbs = [j] if K == 0 else [l for l in range(Lq) if l // K == j]
        fac = [(P % int(o.moduli[l])) if (K and l in limbs) else (1 if l in limbs else 0) for l in range(L)]
        b = o.poly_add(b, o.poly_mul_pointwise(target, _limb_const(o, fac)))
        key[j, 0], key[j, 1] = b, a
    return key


def relin_key(o, K, t_plain, s, seed):
    return switch_key(o, K, t_plain, s, seed, o.poly_mul_pointwise(s, s), 0)


def galois_keys(o, K, t_plain, s, seed, elts):
    out = []
    for g in elts:
        perm = o.galois_perm(g)
        out.append(switch_key(o, K, t_plain, s, seed, np.ascontiguousarray(s[:, perm]), int(g)))
    return np.stack(out)


def encrypt(o, t_plain, s, seed, first_index, pt):
    """pt [n][L][N] -> ct [n][2][L][N] under oracle context o (the ciphertext moduli) and the first o.L rows of s"""
    pt = np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, o.L, o.N)
    s = np.ascontiguousarray(s[:o.L])
    ct = np.empty((pt.shape[0], 2, o.L, o.N), dtype=np.uint64)
    for k in range(pt.shape[0]):
        item = first_index + k
        a = _uniform_rows(o, seed, ENC_A, 0, 0, item)
        e = small_eval(o, cbd(seed, nonce0(ENC_E), item, o.N), t_plain)
        ct[k, 0] = o.poly_add(o.poly_add(e, _neg(o, o.poly_mul_pointwise(a, s))), pt[k])
        ct[k, 1] = a
    return ct


def decrypt(o, s, ct):
    """ct [n][n_comp][L][N] -> c0 + c1 s (+ c2 s^2) [n][L][N] in evaluation form"""
    s = np.ascontiguousarray(s[:o.L])
    out = []
    for c in ct:
        v = o.poly_add(c[0], o.poly_mul_pointwise(c[1], s))
        if len(c) == 3:
            v = o.poly_add(v, o.poly_mul_pointwise(c[2], o.poly_mul_pointwise(s, s)))
        out.append(v)
    return np.stack(out)
