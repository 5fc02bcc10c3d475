"""BGV slot encoding (DESIGN.md section 2.13) composed from the suite's references: tests/slots.py's SlotEncoder, the oracle's
transforms and Python integers for the CRT (test infrastructure)."""
import numpy as np

from slots import SlotEncoder

T_VALUES = (65537, 167772161, 2147352577)   # 2147352577: the largest prime below 2^31 that is 1 mod 2^15
INT64_MIN, INT64_MAX = -(2**63), 2**63 - 1

_encoders = {}


def encoder(n, t):
    if (n, t) not in _encoders:
        _encoders[(n, t)] = SlotEncoder(n, t)
    return _encoders[(n, t)]


def lift(o, coeffs, t):
    """coefficients in [0, t) -> [L][N] residues of the centred lift (coefficient form)"""
    c = np.asarray(coeffs, dtype=np.int64)
    c = np.where(c > t // 2, c - t, c)
    return np.stack([(c % q).astype(np.uint64) for q in o.moduli])


def to_rns_eval(o, coeffs, t):
    return o.ntt_fwd(lift(o, coeffs, t)[None])[0]


def encode(o, slots, t):
    """slots [n_vec][2][N/2] int64 -> plaintexts [n_vec][L][N] in evaluation form"""
    enc = encoder(o.N, t)
    slots = np.asarray(slots, dtype=np.int64).reshape(-1, 2, o.N // 2)
    return o.ntt_fwd(np.stack([lift(o, enc.encode(s), t) for s in slots]))


def modulus_product(o):
    Q = 1
    for q in o.moduli:
        Q *= q
    return Q


def centred_values(o, res):
    """[L][N] residues (coefficient form) -> the N centred CRT values as Python integers"""
    Q = modulus_product(o)
    coef = [(Q // q) * pow(Q // q, -1, q) for q in o.moduli]
    X = sum(res[l].astype(object) * coef[l] for l in range(o.L)) % Q
    return [int(x) - Q if x > (Q - 1) // 2 else int(x) for x in X]


def decode(o, pts, t):
    """plaintexts [n_vec][L][N] in evaluation form -> slots [n_vec][2][N/2] in [0, t) (uint64)"""
    enc = encoder(o.N, t)
    res = o.ntt_inv(np.asarray(pts, dtype=np.uint64).reshape(-1, o.L, o.N))
    out = [enc.decode(np.array([x % t for x in centred_values(o, r)], dtype=np.uint64)) for r in res]
    return np.stack(out).astype(np.uint64)


def residues_of(o, values):
    """N Python integers -> [L][N] evaluation form"""
    return o.ntt_fwd(np.array([[v % q for v in values] for q in o.moduli], dtype=np.uint64)[None])[0]
