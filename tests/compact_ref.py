"""Compact ciphertexts of DESIGN.md section 2.24, restated in Python integers (TEST INFRASTRUCTURE ONLY).

The BGV chain down to q0 is the oracle's mod_switch_down, the transforms are the oracle's.  The switch to 2^bits and the map back to a
level-1 plaintext follow the definition in Python integers, with divisions rather than the kernels' exact-division trick; the phase
is an exact negacyclic product over the integers rather than the kernels' transform modulo q0.  pack / unpack index the bit stream
with numpy; pack_bigint is the definition they are checked against."""
import numpy as np


def lam(q0, bits, t):
    """lambda = 2^bits q0^-1 mod t, the factor a BGV compaction puts on the plaintext"""
    return (1 << bits) * pow(q0, -1, t) % t


def switch(x, q0, bits, t):
    """y in [0, 2^bits) of one coefficient x in [0, q0), and the unreduced value (before mod 2^bits)"""
    u = x << bits
    if t == 0:
        y = ((u << 1) + q0) // (2 * q0)
    else:
        z = u % q0
        j = -z * pow(q0, -1, t) % t
        if j > t // 2:
            j -= t
        y = u // q0 - j
    return y % (1 << bits), y


def pack(y, bits):
    """[..][N] coefficients below 2^bits -> [..][N bits / 64] little-endian bit streams (coefficient i at bits [i bits, (i+1) bits))"""
    y = np.asarray(y).astype(np.uint64)
    lead, N = y.shape[:-1], y.shape[-1]
    flat = y.reshape(-1, N)
    out = np.zeros((flat.shape[0], N * bits // 64), dtype=np.uint64)
    o = np.arange(N, dtype=np.int64) * bits
    k, sh = o >> 6, (o & 63).astype(np.uint64)
    spill = (o & 63) + bits > 64
    for r in range(flat.shape[0]):
        np.bitwise_or.at(out[r], k, flat[r] << sh)
        np.bitwise_or.at(out[r], k[spill] + 1, flat[r][spill] >> (np.uint64(64) - sh[spill]))
    return out.reshape(lead + (N * bits // 64,))


def unpack(words, bits, N):
    """[..][N bits / 64] -> [..][N] uint64"""
    words = np.asarray(words, dtype=np.uint64)
    lead = words.shape[:-1]
    flat = words.reshape(-1, words.shape[-1])
    o = np.arange(N, dtype=np.int64) * bits
    k, sh = o >> 6, (o & 63).astype(np.uint64)
    spill = (o & 63) + bits > 64
    out = np.empty((flat.shape[0], N), dtype=np.uint64)
    for r in range(flat.shape[0]):
        v = flat[r][k] >> sh
        v[spill] |= flat[r][k[spill] + 1] << (np.uint64(64) - sh[spill])
        out[r] = v & np.uint64((1 << bits) - 1)
    return out.reshape(lead + (N,))


def pack_bigint(y, bits):
    """pack() by the definition, one Python integer per polynomial (slow; the cross-check of pack and unpack)"""
    acc = 0
    for i, v in enumerate(y):
        acc |= int(v) << (i * bits)
    return np.array([(acc >> (64 * k)) & ((1 << 64) - 1) for k in range(len(y) * bits // 64)], dtype=np.uint64)


def level1(oracle_mod, o, level, t, ct):
    """[n][2][level][N] evaluation form (o: an oracle over the context's moduli) -> [n][2][N] coefficients in [0, q0) of the level-1
    pair: l - 1 modulus switches with t (BGV), or limb 0 (CKKS), then the inverse transform"""
    ct = np.ascontiguousarray(ct, dtype=np.uint64).reshape(-1, 2, level, o.N)
    n = ct.shape[0]
    x = ct.reshape(2 * n, level, o.N)
    if t:
        for k in range(level, 1, -1):
            x = oracle_mod.Oracle(o.logn, k, o.moduli[:k]).mod_switch_down(x, t)
    else:
        x = np.ascontiguousarray(x[:, :1])
    o1 = oracle_mod.Oracle(o.logn, 1, o.moduli[:1])
    return o1.ntt_inv(x).reshape(n, 2, o.N)


def compact(oracle_mod, o, level, bits, t, ct):
    """the compact ciphertexts [n][2][N bits / 64]"""
    x = level1(oracle_mod, o, level, t, ct)
    q0 = o.moduli[0]
    y = np.vectorize(lambda v: switch(int(v), q0, bits, t)[0], otypes=[object])(x)
    return pack(y, bits)


def phase(o, bits, s, cct):
    """[n][N] centred phases c0' + c1' s in Z_2^bits[X]/(X^N+1), exactly: c1' s is a negacyclic product over the integers, whose
    terms and partial sums stay below N 2^(bits-1) < 2^62"""
    N = o.N
    c = unpack(cct, bits, N).astype(np.int64)
    s_coef = _secret_coeffs(o, s)
    half, mod = 1 << (bits - 1), 1 << bits
    c1 = np.where(c[:, 1] >= half, c[:, 1] - mod, c[:, 1])
    prod = np.zeros_like(c1)
    for j, sj in enumerate(s_coef):
        if sj:
            r = np.concatenate([-c1[:, N - j:], c1[:, :N - j]], axis=1) if j else c1
            prod += r if sj == 1 else -r
    p = (c[:, 0] + prod) % mod
    return np.where(p >= half, p - mod, p)


def _secret_coeffs(o, s):
    """the ternary coefficients of the secret (row 0, evaluation form)"""
    q0 = o.moduli[0]
    v = _o1(o).ntt_inv(np.ascontiguousarray(np.asarray(s).reshape(-1, o.N)[:1]))[0]
    return [int(x) - q0 if int(x) > q0 // 2 else int(x) for x in v]


_O1 = {}


def _o1(o):
    import oracle as oracle_mod
    key = (o.logn, o.moduli[0])
    if key not in _O1:
        _O1[key] = oracle_mod.Oracle(o.logn, 1, o.moduli[:1])
    return _O1[key]


def plain_coeff(p, q0, bits, t):
    """the plaintext coefficient in [0, q0) of a centred phase p: BGV (p mod t) lambda^-1 mod t lifted centred, CKKS
    floor(p q0 / 2^bits + 1/2) mod q0"""
    if t:
        m = p % t * pow(lam(q0, bits, t), -1, t) % t
        v = m - t if m > t // 2 else m
    else:
        v = (2 * p * q0 + (1 << bits)) // (2 << bits)
    return v % q0


def plaintext(o, bits, t, phi):
    """[n][N] centred phases -> level-1 plaintexts [n][1][N] in evaluation form"""
    q0 = o.moduli[0]
    coef = np.array([[[plain_coeff(int(p), q0, bits, t) for p in row]] for row in phi], dtype=np.uint64).reshape(-1, 1, o.N)
    return _o1(o).ntt_fwd(coef)


def lift(c1, q0, bits):
    """c1' in [0, 2^bits) lifted centred into Z_q0"""
    return (c1 - (1 << bits)) % q0 if c1 >= 1 << (bits - 1) else c1


def decrypt(o, bits, t, s, cct):
    """the level-1 plaintexts [n][1][N] (evaluation form) of compact ciphertexts, through the exact phase"""
    return plaintext(o, bits, t, phase(o, bits, s, cct))


def max_bits(log_n, q0):
    """the largest bits with N 2^bits < q0"""
    b = 2
    while (1 << (b + 1 + log_n)) < q0:
        b += 1
    return b
