"""Restatement of DESIGN.md section 2.15 in Python integers and the oracle: the scalar linear combination of ciphertexts, and BGV
polynomial evaluation down the modulus chain composed from the oracle's ct_mul_relin_grouped and mod_switch_down on oracle contexts
over each level's own basis, with keys restricted from the top-level key."""
import numpy as np


def floor_mod(c, q):
    return int(c) % int(q)   # Python's % is floor-mod


def centred(x, t):
    return x if x <= t // 2 else x - t


def ceil_log2(k):
    return (k - 1).bit_length()


def lincomb(moduli, cts, coeffs, constant, pt=None):
    """sum_i (c_i mod q_l) ct_i + (constant mod q_l) on every c0 row (+ pt [L][N] on c0), canonical; cts [batch][2][L][N] each"""
    out = np.zeros_like(np.asarray(cts[0], dtype=np.uint64))
    for l, q in enumerate(moduli):
        q = int(q)
        acc = np.zeros(out[:, :, l].shape, dtype=object)
        for ct, c in zip(cts, coeffs):
            acc = acc + np.asarray(ct, dtype=np.uint64)[:, :, l].astype(object) * floor_mod(c, q)
        acc[:, 0] += floor_mod(constant, q)
        if pt is not None:
            acc[:, 0] += np.asarray(pt, dtype=np.uint64)[l].astype(object)
        out[:, :, l] = (acc % q).astype(np.uint64)
    return out


def restrict_key(key, Lq, K, l):
    """the level-l key from the top-level grouped key [dnum][2][Lq+K][N]: digits g < ceil(l/K), rows 0..l-1 and Lq..Lq+K-1"""
    dl = -(-l // K)
    return np.ascontiguousarray(np.concatenate([key[:dl, :, :l], key[:dl, :, Lq:Lq + K]], axis=2))


def split(k):
    p = 1
    while 2 * p < k:
        p *= 2
    return p, k - p


class Chain:
    """oracle contexts of every level of a top basis q_0 .. q_{Lq-1}, p_0 .. p_{K-1}"""

    def __init__(self, oracle_mod, logn, moduli, K):
        self.om, self.logn, self.K = oracle_mod, logn, K
        self.moduli = [int(q) for q in moduli]
        self.Lq = len(moduli) - K
        self._ks, self._ct = {}, {}

    def ks(self, l):   # key switching at level l
        if l not in self._ks:
            self._ks[l] = self.om.Oracle(self.logn, l + self.K, self.moduli[:l] + self.moduli[self.Lq:])
        return self._ks[l]

    def ct(self, l):   # the ciphertext moduli of level l
        if l not in self._ct:
            self._ct[l] = self.om.Oracle(self.logn, l, self.moduli[:l])
        return self._ct[l]


def polyeval(chain, t, coeffs, ct, key, mutate=None, stats=None):
    """p(x) for ct [batch][2][Lq][N] at the top level; returns [batch][2][Lf][N].  `mutate` names a deliberate error of the schedule
    (tests show that each one changes the decrypted slots): 'no_qinv', 'g_above', 'sum_after', 'no_special_rows'."""
    Lq, K = chain.Lq, chain.K
    d = len(coeffs) - 1
    D = ceil_log2(d)
    a = [floor_mod(c, t) for c in coeffs]
    qinv = [pow(chain.moduli[i] % t, -1, t) for i in range(Lq)]
    B = ct.shape[0]

    stats = {} if stats is None else stats
    stats.update(mul=0, switch=0, lincomb=1)

    def switch(x, l):   # drops q_{l-1}
        stats["switch"] += 1
        return chain.ct(l).mod_switch_down(x.reshape(2 * B, l, -1), t).reshape(B, 2, l - 1, -1)

    if D == 0:
        return lincomb(chain.moduli[:Lq], [ct], [centred(a[1], t)], centred(a[0], t))
    Lf = Lq - D
    need = [False] + [a[k] != 0 for k in range(1, d + 1)]
    any_term = any(need)
    if not any_term:
        need[1] = True
    for k in range(d, 1, -1):
        if need[k]:
            u, v = split(k)
            need[u] = need[v] = True
    at, fac, y, yfac = {(1, Lq): ct}, {(1, Lq): 1}, {}, {}

    def get(k, l):
        if (k, l) in at:
            return
        get(k, l + 1)
        at[k, l] = switch(at[k, l + 1], l + 1)
        fac[k, l] = fac[k, l + 1] * (1 if mutate == "no_qinv" else qinv[l]) % t

    for k in range(2, d + 1):
        if not need[k]:
            continue
        u, v = split(k)
        ck = ceil_log2(k)
        l = Lq - ck + 1
        get(u, l)
        get(v, l)
        kl = restrict_key(key, Lq, K, l)
        if mutate == "no_special_rows":
            kl = np.ascontiguousarray(np.concatenate([key[:kl.shape[0], :, :l], key[:kl.shape[0], :, l:l + K]], axis=2))
        stats["mul"] += 1
        prod = chain.ks(l).ct_mul_relin_grouped(K, at[u, l], at[v, l], kl, t)
        f = fac[u, l] * fac[v, l] % t
        if ck == D:
            y[k], yfac[k] = prod, f
        else:
            at[k, l - 1] = switch(prod, l)
            fac[k, l - 1] = f * (1 if mutate == "no_qinv" else qinv[l - 1]) % t
    G = chain.moduli[Lf + 1 if mutate == "g_above" else Lf] % t
    terms, cs = [], []
    for k in range(1, d + 1):
        if (a[k] == 0) if any_term else (k != 1):
            continue
        if ceil_log2(k) == D:
            x, g = y[k], yfac[k]
        else:
            get(k, Lf + 1)
            x, g = at[k, Lf + 1], fac[k, Lf + 1]
        if mutate == "sum_after":
            x = switch(x, Lf + 1)
        terms.append(x)
        cs.append(centred(a[k] * pow(g, -1, t) * G % t, t))
    c0 = centred(a[0] * G % t, t)
    if mutate == "sum_after":
        return lincomb(chain.moduli[:Lf], terms, cs, c0)
    return switch(lincomb(chain.moduli[:Lf + 1], terms, cs, c0), Lf + 1)


def poly_mod_t(coeffs, x, t):
    """p(x) mod t elementwise (x: integer array)"""
    acc = np.zeros(np.shape(x), dtype=object)
    xo = np.asarray(x).astype(object) % t
    for c in reversed(coeffs):
        acc = (acc * xo + int(c)) % t
    return acc.astype(np.uint64)
