"""Restatement of DESIGN.md section 2.16 in Python integers, doubles and the oracle: CKKS polynomial evaluation down the rescaling
chain, composed from the oracle's ct_mul_relin_grouped(..., 0) and mod_switch_down(..., 0) on the per-level oracle contexts of
polyeval_ref.Chain, with keys restricted from the top-level key.  Cuts are slices; the combination is Python-integer arithmetic on
the exact integers int(c_k).  Shares no code with csrc/.

Python floats are IEEE doubles and every operation below rounds on its own (no FMA), round() on a float is round half to even, and
float(q) of an integer rounds to nearest: the scales and coefficients are those of the specification bit for bit."""
import math

import numpy as np

from polyeval_ref import ceil_log2, lincomb, restrict_key, split


def check(d, Lq, K, coeffs=None, scale_in=1.0, scale_out=1.0):
    """the argument rules of section 2.16; raises ValueError"""
    if not 1 <= d <= 64:
        raise ValueError("the degree must be in [1, 64]")
    D = ceil_log2(d)
    if D > Lq - 2 or D > Lq - K + 1:
        raise ValueError("degree %d needs %d levels" % (d, D))
    if coeffs is not None and not all(math.isfinite(a) for a in coeffs):
        raise ValueError("non-finite coefficient")
    for s in (scale_in, scale_out):
        if not (math.isfinite(s) and s > 0):
            raise ValueError("scales must be finite and positive")


def needed(a):
    """the powers made: every k >= 1 with a_k != 0 (x alone if there is none), and recursively the operands of their products"""
    d = len(a) - 1
    need = [False] + [a[k] != 0 for k in range(1, d + 1)]
    any_term = any(need)
    if not any_term:
        need[1] = True
    for k in range(d, 1, -1):
        if need[k]:
            u, v = split(k)
            need[u] = need[v] = True
    return need, any_term


def level_of(Lq, k):
    """the level x^k lives at"""
    return Lq - ceil_log2(k)


def scales(moduli, Lq, a, scale_in, mutate=None):
    """{k: s_k} for every power made"""
    need, _ = needed(a)
    s = {1: float(scale_in)}
    for k in range(2, len(a)):
        if need[k]:
            u, v = split(k)
            l = Lq - ceil_log2(k) + 1
            s[k] = float(scale_in) if mutate == "no_scales" else (s[u] * s[v]) / float(moduli[l - 1])
    return s


def coefficients(moduli, Lq, coeffs, scale_in, scale_out=None, mutate=None):
    """(Lc, terms [(k, c_k)], c_0): the powers of the combination in increasing k with their integer-valued doubles"""
    a = [float(c) for c in coeffs]
    S = float(scale_in if scale_out is None else scale_out)
    D = ceil_log2(len(a) - 1)
    Lc = Lq - D
    m = S * float(moduli[Lc - 1])
    s = scales(moduli, Lq, a, scale_in, mutate)
    _, any_term = needed(a)
    terms = []
    for k in range(1, len(a)):
        if (a[k] == 0) if any_term else (k != 1):
            continue
        terms.append((k, float(round((a[k] * m) / s[k]))))
    return Lc, terms, float(round(a[0] * m))


def residue(c, q):
    """an integer-valued double reduced exactly mod q"""
    return int(c) % int(q)


def polyeval(chain, coeffs, scale_in, ct, key, scale_out=None, mutate=None, stats=None):
    """p(x) for ct [batch][2][Lq][N] at the top level; returns [batch][2][Lc-1][N], Lc = Lq - ceil(log2 d).  `mutate` names a
    deliberate error of the schedule (tests show that each one moves the decoded slots far off): 'rescale_align' (operands
    aligned by rescaling instead of cutting), 'no_scales' (Delta_in for every scale), 'comb_after' (the combination after the last
    rescale), 'no_special_rows' (keys restricted without the special rows).  stats: mul, rescale, cut and the launch count."""
    Lq, K, moduli = chain.Lq, chain.K, chain.moduli
    d = len(coeffs) - 1
    check(d, Lq, K, [float(c) for c in coeffs], scale_in, scale_in if scale_out is None else scale_out)
    a = [float(c) for c in coeffs]
    B = ct.shape[0]
    stats = {} if stats is None else stats
    stats.update(mul=0, rescale=0, cut=0)

    def rescale(x, l):   # drops q_{l-1}
        stats["rescale"] += 1
        return chain.ct(l).mod_switch_down(x.reshape(2 * B, l, -1), 0).reshape(B, 2, l - 1, -1)

    need, _ = needed(a)
    home = {1: Lq}
    at = {(1, Lq): np.asarray(ct, dtype=np.uint64)}

    def get(k, l):
        if (k, l) not in at:
            if mutate == "rescale_align":
                get(k, l + 1)
                at[k, l] = rescale(at[k, l + 1], l + 1)
            else:
                stats["cut"] += 1
                at[k, l] = np.ascontiguousarray(at[k, home[k]][:, :, :l])
        return at[k, l]

    for k in range(2, d + 1):
        if not need[k]:
            continue
        u, v = split(k)
        l = Lq - ceil_log2(k) + 1
        kl = restrict_key(key, Lq, K, l)
        if mutate == "no_special_rows":
            kl = np.ascontiguousarray(np.concatenate([key[:kl.shape[0], :, :l], key[:kl.shape[0], :, l:l + K]], axis=2))
        stats["mul"] += 1
        prod = chain.ks(l).ct_mul_relin_grouped(K, get(u, l), get(v, l), kl, 0)
        at[k, l - 1] = rescale(prod, l)
        home[k] = l - 1
    Lc, terms, c0 = coefficients(moduli, Lq, coeffs, scale_in, scale_out, mutate)
    xs = [get(k, Lc) for k, _ in terms]
    cs = [int(c) for _, c in terms]
    stats["launches"] = stats["mul"] + 2 * stats["rescale"] + 2
    if mutate == "comb_after":
        xs = [rescale(x, Lc) for x in xs]
        return lincomb(moduli[:Lc - 1], xs, cs, int(c0))
    return rescale(lincomb(moduli[:Lc], xs, cs, int(c0)), Lc)


def poly_eval(coeffs, z):
    """p(z) in float64 by Horner"""
    acc = np.zeros(np.shape(z), dtype=np.complex128)
    for c in reversed(coeffs):
        acc = acc * z + float(c)
    return acc


def power_sum(coeffs, z):
    """sum_k |a_k| |z|^k: the cancellation factor of the power basis"""
    r = np.abs(z)
    return sum(abs(float(c)) * r ** k for k, c in enumerate(coeffs))


def ckks_chain(oracle_mod, Lq, K):
    """the CKKS chain of the tests: q_0 a 60-bit k 2^32 + 1 prime, q_1 .. q_{Lq-1} distinct k 2^32 + 1 primes just above 2^45, and K
    60-bit special primes (the next such primes below q_0)"""
    import bases
    lib = oracle_mod.lib()
    top = bases._scan(lib, (1 << 60) - bases.FAST_STEP + 1, -bases.FAST_STEP, True, 1 + K)
    mid = bases._scan(lib, (1 << 45) + 1, bases.FAST_STEP, True, Lq - 1)
    return [top[0]] + mid + top[1:]
