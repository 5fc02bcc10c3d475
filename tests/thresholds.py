"""Inputs that put the kernels' data-dependent branches exactly on, just below and just above their thresholds, shared by the CPU
(oracle against exact integers, emulated bodies) and GPU tests.

Uniform residues land on such a threshold with probability about N L 2^-60 per call, so without these inputs a test cannot tell
`>` from `>=`.  Every value is built in the domain where the branch reads it (the coefficient form of the dropped limb, the inverse
transform of a digit, the CRT value) and mapped to evaluation form with the oracle's exact transforms.  Every crafting function
checks with Python integers that the values it promises occur, so that a construction error cannot leave a test vacuous.  The
targets are tiled over all N positions: every lane, both halves of a 16-byte pair and both CTA halves at N = 16384 see them.

The branches (DESIGN.md):
  - centred lift in the division by one modulus, tau' > q/2 (section 2.9: mod_switch_down, the hybrid key switch);
  - centred lift of every special residue in the division by P, y_k > p_k/2 (section 2.11);
  - a zero coefficient of a hoisted digit t_j, which sends the ciphertext to the ordinary rotation (section 2.8b);
  - CKKS decoding: the sign of X from its Garner digits, then the digits of Q - X (section 2.12);
  - CKKS encoding: rint ties to even and the sign of a zero residue (section 2.12).
"""
import random

import numpy as np


def targets(q):
    """the values either side of the centring threshold h = floor(q/2) (q odd: h stays, h + 1 is lifted to h + 1 - q), and the ends"""
    h = q >> 1
    return [0, 1, h - 1, h, h + 1, q - 2, q - 1]


def centred(v, q):
    """the representative of v mod q in (-q/2, q/2], stated without the kernels' `v > q >> 1`"""
    v %= q
    return v - q if 2 * v > q else v


def _odd(seq):
    """a period of odd length, so that every entry meets even and odd positions"""
    return seq if len(seq) % 2 else seq + seq[:1]


def _tile(period, n, shift=0):
    return [period[(k + shift) % len(period)] for k in range(n)]


def assert_spread(values, want, what):
    """every w in `want` occurs in `values` (one entry per coefficient position) at an even and an odd position, and in both halves"""
    n = len(values)
    for w in want:
        pos = [k for k, v in enumerate(values) if v == w]
        assert pos, "%s: %r never occurs" % (what, w)
        assert any(k % 2 == 0 for k in pos) and any(k % 2 for k in pos), "%s: %r not at both parities" % (what, w)
        assert any(k < n // 2 for k in pos) and any(k >= n // 2 for k in pos), "%s: %r not in both halves" % (what, w)


def _ints(a):
    return [int(v) for v in a]


def _pad(o, x, limbs):
    """[..., limbs][N] residues in a [..., L][N] array (the rest zero), for the oracle's L-limb transforms"""
    out = np.zeros(x.shape[:-2] + (o.L, o.N), dtype=np.uint64)
    out[..., :limbs, :] = x
    return out


def _coeff(o, x, limbs):
    """coefficient form of [..., limbs][N] evaluation-form residues under the first `limbs` moduli of o"""
    return o.ntt_inv(_pad(o, x, limbs))[..., :limbs, :]


def _eval(o, xc, limbs):
    return np.ascontiguousarray(o.ntt_fwd(_pad(o, xc, limbs))[..., :limbs, :])


def basis_moduli(oracle_mod, name, L):
    """the first L moduli of a basis: None for the default one; gen_mixed of tests/bases.py, extended by two generic primes (52 and
    47 bits) beyond its six limbs, so that four special primes (which need L >= 8) run on a generic basis too"""
    if name == "default":
        return None
    import bases
    mods = bases.catalogue(oracle_mod)[name]
    if L > len(mods):
        assert name == "gen_mixed" and L <= len(mods) + 2
        mods = mods + [bases._generic_prime(oracle_mod.lib(), b) for b in (52, 47)]
        assert len(set(mods)) == len(mods) and not any(bases.is_fast(q) for q in mods)
    return mods[:L]


def special_limbs(K):
    """the limbs of a context with K special primes: six, or eight for K = 4 (at most half the limbs may be special)"""
    return max(6, 2 * K)


def _prod(vals):
    r = 1
    for v in vals:
        r *= v
    return r


# ---------------------------------------------------------------- division by one modulus (DESIGN.md section 2.9)
def tau_prime(o, x, t):
    """tau' = INTT(last limb) * t^-1 mod q_last of every polynomial of x [n][L][N] (Python ints)"""
    ql = o.moduli[-1]
    tinv = pow(t, -1, ql) if t else 1
    return [[v * tinv % ql for v in _ints(row)] for row in o.ntt_inv(x)[:, -1]]


def mod_switch_input(o, n_polys, t, seed):
    """[n][L][N] evaluation form, uniform except the last limb, whose tau' runs through targets(q_last)"""
    ql = o.moduli[-1]
    x = o.fill_uniform(seed, n_polys)
    xc = o.ntt_inv(x)
    period = _odd(targets(ql))
    for p in range(n_polys):
        xc[p, -1] = [v * t % ql if t else v for v in _tile(period, o.N, p)]
    x = o.ntt_fwd(xc)
    for p, tp in enumerate(tau_prime(o, x, t)):
        assert_spread(tp, targets(ql), "tau' of polynomial %d" % p)
    return x


def exact_mod_switch(o, x, t):
    """coefficient form [n][L-1][N] of (X - s w) / q_last, w = centred(tau'), s = t (1 when t = 0), in Python integers"""
    ql, s = o.moduli[-1], t if t else 1
    xc = o.ntt_inv(x)
    taus = tau_prime(o, x, t)
    out = np.empty((x.shape[0], o.L - 1, o.N), dtype=np.uint64)
    for p in range(x.shape[0]):
        w = [centred(v, ql) for v in taus[p]]
        for i, q in enumerate(o.moduli[:-1]):
            inv = pow(ql, -1, q)
            out[p, i] = [(c - s * wn) * inv % q for c, wn in zip(_ints(xc[p, i]), w)]
    return out


def hybrid_key(o, seed):
    """a uniform hybrid key [L-1][2][L][N] whose special-prime column is 1 in digit 0 and 0 in every other digit: the special
    accumulator of a key switch is then the lift of digit 0 into p, so tau = INTT_{q_0}(d[0]) mod p"""
    Lq = o.L - 1
    key = o.fill_uniform(seed, 2 * Lq).reshape(Lq, 2, o.L, o.N)
    key[0, :, -1] = 1
    key[1:, :, -1] = 0
    one = o.ntt_inv(key[0])[:, -1]
    assert all(int(v) == (k == 0) for row in one for k, v in enumerate(row))   # all ones in evaluation form == the constant 1
    return key


def hybrid_digits(o, batch, t, seed):
    """d [batch][L-1][N]: uniform, except that tau' of the special accumulator (digit 0, under hybrid_key) runs through targets(p)"""
    Lq, p, q0 = o.L - 1, o.moduli[-1], o.moduli[0]
    rng = np.random.default_rng(seed)
    dc = np.stack([rng.integers(0, q, (batch, o.N), dtype=np.uint64) for q in o.moduli[:Lq]], axis=1)
    period = _odd(targets(p))
    for b in range(batch):
        tau = [v * t % p if t else v for v in _tile(period, o.N, b)]
        assert max(tau) < q0, "digit 0 cannot reach tau: q_0 < p"
        dc[b, 0] = tau
    d = _eval(o, dc, Lq)
    tinv = pow(t, -1, p) if t else 1
    for b, row in enumerate(_coeff(o, d, Lq)[:, 0]):
        assert_spread([v % p * tinv % p for v in _ints(row)], targets(p), "hybrid tau' of digit %d" % b)
    return d


# ---------------------------------------------------------------- division by P (DESIGN.md section 2.11)
def _special(o, K):
    Lq = o.L - K
    ps = o.moduli[Lq:]
    P = _prod(ps)
    return Lq, ps, P, [P // pk for pk in ps]


def md_factors(o, K, t):
    """f_k = t * Phat_k mod p_k (Phat_k when t = 0): y_k = INTT(special limb k) * f_k^-1"""
    _, ps, _, ph = _special(o, K)
    return [(t if t else 1) * h % pk for h, pk in zip(ph, ps)]


def y_values(o, K, x, t):
    """y_k of every polynomial of x [n][L][N]: [n][K] lists of N Python ints"""
    Lq, ps, _, _ = _special(o, K)
    finv = [pow(fk, -1, pk) for fk, pk in zip(md_factors(o, K, t), ps)]
    xc = o.ntt_inv(x)
    return [[[v * fi % pk for v in _ints(xc[p, Lq + k])] for k, (pk, fi) in enumerate(zip(ps, finv))] for p in range(x.shape[0])]


def check_y(o, K, ys, what):
    """every targets(p_k) for every k, and positions where every y_k is above its threshold at once (the largest lazy sum)"""
    _, ps, _, _ = _special(o, K)
    for k, pk in enumerate(ps):
        assert_spread(ys[k], targets(pk), "%s, y_%d" % (what, k))
    above = [int(all(2 * ys[k][n] > ps[k] for k in range(K))) for n in range(len(ys[0]))]
    assert_spread(above, [1], "%s, every y_k above p_k/2" % what)


def _y_combos(ps, rng):
    """K-tuples of y values: each target of each p_k with the others uniform, then every y_k at h_k, at h_k + 1, at p_k - 1"""
    K = len(ps)
    out = []
    for k, pk in enumerate(ps):
        for v in targets(pk):
            out.append(tuple(v if j == k else int(rng.integers(0, pj)) for j, pj in enumerate(ps)))
    out += [tuple(p >> 1 for p in ps), tuple((p >> 1) + 1 for p in ps), tuple(p - 1 for p in ps)]
    assert all(len(c) == K for c in out)
    return _odd(out)


def mod_down_input(o, K, n_polys, t, seed):
    """[n][L][N]: uniform, except that the special limbs' y_k run through targets(p_k), alone and all above at once"""
    Lq, ps, _, _ = _special(o, K)
    f = md_factors(o, K, t)
    x = o.fill_uniform(seed, n_polys)
    xc = o.ntt_inv(x)
    combos = _y_combos(ps, np.random.default_rng(seed))
    for p in range(n_polys):
        col = _tile(combos, o.N, p)
        for k in range(K):
            xc[p, Lq + k] = [c[k] * f[k] % ps[k] for c in col]
    x = o.ntt_fwd(xc)
    for p, ys in enumerate(y_values(o, K, x, t)):
        check_y(o, K, ys, "polynomial %d" % p)
    return x


def exact_mod_down(o, K, x, t):
    """coefficient form [n][L-K][N] of (X - s delta) / P, delta = sum_k centred(y_k) Phat_k, s = t (1 when t = 0), in Python integers"""
    Lq, ps, P, ph = _special(o, K)
    s = t if t else 1
    xc = o.ntt_inv(x)
    out = np.empty((x.shape[0], Lq, o.N), dtype=np.uint64)
    for p, ys in enumerate(y_values(o, K, x, t)):
        delta = [sum(centred(ys[k][n], ps[k]) * ph[k] for k in range(K)) for n in range(o.N)]
        for i, q in enumerate(o.moduli[:Lq]):
            inv = pow(P, -1, q)
            out[p, i] = [(c - s * dn) * inv % q for c, dn in zip(_ints(xc[p, i]), delta)]
    return out


def grouped_key(o, K, seed):
    """a uniform grouped key [dnum][2][L][N] whose special columns are 1 in digit 0 and 0 elsewhere: special accumulator k is then the
    lift of digit 0 into p_k"""
    Lq = o.L - K
    dnum = o.grouped_digits(K)
    key = o.fill_uniform(seed, 2 * dnum).reshape(dnum, 2, o.L, o.N)
    key[0, :, Lq:] = 1
    key[1:, :, Lq:] = 0
    return key


def _digit0(o, K):
    Lq = o.L - K
    qs = o.moduli[:min(K, Lq)]
    Qg = _prod(qs)
    return qs, [Qg // q for q in qs]


def grouped_y(o, K, d, t):
    """y_k of the division by P after a key switch of d [batch][Lq][N] under grouped_key: the lift of digit 0,
    sum_j y_j (Qhat_j mod p_k) with y_j = INTT_j(d[j]) Qhat_j^-1, times f_k^-1"""
    Lq, ps, _, _ = _special(o, K)
    qs, qh = _digit0(o, K)
    finv = [pow(fk, -1, pk) for fk, pk in zip(md_factors(o, K, t), ps)]
    hinv = [pow(h % q, -1, q) for q, h in zip(qs, qh)]
    dc = _coeff(o, d, Lq)
    out = []
    for b in range(d.shape[0]):
        yj = [[v * hi % q for v in _ints(dc[b, j])] for j, (q, hi) in enumerate(zip(qs, hinv))]
        lift = [sum(col[n] * h for col, h in zip(yj, qh)) for n in range(o.N)]
        out.append([[v % pk * fi % pk for v in lift] for pk, fi in zip(ps, finv)])
    return out


def grouped_digits_input(o, K, batch, t, seed):
    """d [batch][Lq][N]: uniform, except that at most positions the digit-0 values are solved so that one (k, target) pair of the
    division by P occurs; the remaining positions are uniform (where every y_k is above p_k/2 at once now and then)"""
    Lq, ps, _, _ = _special(o, K)
    qs, qh = _digit0(o, K)
    f = md_factors(o, K, t)
    rng = np.random.default_rng(seed)
    dc = np.stack([rng.integers(0, q, (batch, o.N), dtype=np.uint64) for q in o.moduli[:Lq]], axis=1)
    pairs = _odd([(k, v) for k, pk in enumerate(ps) for v in targets(pk)] + [None] * 5)
    for b in range(batch):
        for n, pair in enumerate(_tile(pairs, o.N, b)):
            if pair is None:
                continue
            k, v = pair
            pk, want = ps[k], v * f[k] % ps[k]                   # the lift into p_k must be `want`
            for _ in range(1000):                               # y_1.. uniform, y_0 solved mod p_k; retry until y_0 < q_0
                ys = [0] + [int(rng.integers(0, q)) for q in qs[1:]]
                rest = sum(y * h for y, h in zip(ys[1:], qh[1:])) % pk
                ys[0] = (want - rest) * pow(qh[0] % pk, -1, pk) % pk
                if ys[0] < qs[0]:
                    break
            else:
                raise AssertionError("digit 0 cannot reach the target")
            for j, (q, h) in enumerate(zip(qs, qh)):
                dc[b, j, n] = ys[j] * h % q                     # INTT_j(d[j]) = y_j Qhat_j
    d = _eval(o, dc, Lq)
    for b, ys in enumerate(grouped_y(o, K, d, t)):
        check_y(o, K, ys, "grouped digit %d" % b)
    return d


# ---------------------------------------------------------------- key-switch inputs from crafted digits
def ones(o, limbs):
    """the constant 1 in evaluation form: b1 = ones makes the ct x ct digit d2 = a1 * b1 equal a1"""
    return np.ones((limbs, o.N), dtype=np.uint64)


def mul_inputs(o, d, seed):
    """ciphertexts a, b [batch][2][limbs][N] with a1 = d and b1 = 1, so that the tensor's d2 is d"""
    batch, limbs = d.shape[0], d.shape[1]
    u = o.fill_uniform(seed, 2 * batch)[:, :limbs].reshape(batch, 2, limbs, o.N)
    a, b = u.copy(), u[::-1].copy()
    a[:, 1] = d
    b[:, 1] = ones(o, limbs)
    return a, b


def rotate_inputs(o, d, g, seed):
    """ciphertexts [batch][2][limbs][N] with sigma_g(c1) = d: the rotation key-switches d"""
    batch, limbs = d.shape[0], d.shape[1]
    ct = o.fill_uniform(seed, 2 * batch)[:, :limbs].reshape(batch, 2, limbs, o.N).copy()
    perm = o.galois_perm(g)
    c1 = np.empty_like(d)
    c1[..., perm] = d
    assert np.array_equal(c1[..., perm], d)          # the rotation reads c1[perm[n]] into position n
    ct[:, 1] = c1
    return ct


# ---------------------------------------------------------------- hoisted rotations (DESIGN.md section 2.8b)
def negated(o, g, pos):
    """whether sigma_g moves coefficient `pos` onto a negated coefficient (X^pos -> -X^(pos g - N))"""
    e = np.zeros(o.N, dtype=np.uint64)
    e[pos] = 1
    out = o.galois_coeff(0, g, e)
    return int(out.max()) == o.moduli[0] - 1


def hoist_zero_input(o, batch, zeros, seed):
    """ciphertexts [batch][2][L][N] whose digits t_j = INTT_j(c1[j]) have no zero coefficient, except exactly one zero at
    (digit, position) = zeros[k] in ciphertext k"""
    rng = np.random.default_rng(seed)
    ct = o.fill_uniform(seed, 2 * batch).reshape(batch, 2, o.L, o.N)
    c1 = np.stack([rng.integers(1, q, (batch, o.N), dtype=np.uint64) for q in o.moduli], axis=1)
    for k, (j, pos) in zeros.items():
        c1[k, j, pos] = 0
    ct[:, 1] = o.ntt_fwd(c1)
    back = o.ntt_inv(np.ascontiguousarray(ct[:, 1]))
    for k in range(batch):
        z = np.argwhere(back[k] == 0)
        assert [tuple(int(v) for v in r) for r in z] == ([zeros[k]] if k in zeros else []), k
    return ct


# ---------------------------------------------------------------- CKKS decoding (DESIGN.md section 2.12)
def decode_values(moduli):
    """coefficients X in [0, Q) either side of the sign threshold (Q - 1)/2, and with leading zero Garner digits (Q - q_0 ...)"""
    Q = _prod(moduli)
    h = (Q - 1) // 2
    q0 = moduli[0]
    vals = [0, 1, Q - 1, h, h + 1, h - 1, h + 2, h + q0, h - q0, Q - q0]
    if len(moduli) > 1:
        vals += [q0 * moduli[1], Q - q0 * moduli[1]]
    return sorted({v for v in vals if 0 <= v < Q})


def garner(moduli, X):
    """the mixed-radix digits of X: X = d_0 + d_1 q_0 + d_2 q_0 q_1 + ..."""
    out = []
    for q in moduli:
        out.append(X % q)
        X //= q
    return out


def decode_coeffs(moduli, n, seed):
    """N coefficients in [0, Q): decode_values at k and at k + N/2 (the real and imaginary parts of one slot pair), uniform elsewhere"""
    vals = decode_values(moduli)
    Q = _prod(moduli)
    rng = random.Random(seed)
    X = [rng.randrange(Q) for _ in range(n)]
    step = n // 2 // len(vals)
    for i, v in enumerate(vals):
        X[i * step + i % 2] = v                                     # both parities
        X[n // 2 + i * step + 1 - i % 2] = vals[(i + 1) % len(vals)]
    assert set(vals) <= set(X[:n // 2]) and set(vals) <= set(X[n // 2:])
    if len(moduli) > 1:                # negative values whose lowest Garner digits are zero: the lowest-non-zero-digit branch
        assert [v for v in vals if 2 * v > Q and garner(moduli, v)[:2] == [0, 0]]
    return X


def to_eval(o, X):
    """coefficients [N] (integers mod Q) -> [1][L][N] evaluation form"""
    res = np.array([[v % q for v in X] for q in o.moduli], dtype=np.uint64)
    return o.ntt_fwd(res[None])


# ---------------------------------------------------------------- CKKS encoding (DESIGN.md section 2.12)
TIE_K = [0, 1, 2, -1, -2, -3, 2**51 + 1]


def rint_even(num, den):
    """num / den rounded to the nearest integer, ties to even (Python integers)"""
    q, r = divmod(num, den)
    if 2 * r > den or (2 * r == den and q % 2):
        q += 1
    return q


def constant_slot_cases():
    """(slot value, scale, exact coefficient 0, exact coefficient N/2): constant slots c = a + ib encode to a scale at X^0 and
    b scale at X^(N/2) (every slot exponent is 1 mod 4, so X^(N/2) is i in every slot)"""
    from fractions import Fraction
    cases = []
    delta = 2.0**40
    halves = [Fraction(2 * k + 1, 2) for k in TIE_K] + [Fraction(-1, 4)]
    for i, v in enumerate(halves):
        w = halves[(i + 3) % len(halves)]
        cases.append((complex(float(v) / delta, float(w) / delta), delta,
                      rint_even(v.numerator, v.denominator), rint_even(w.numerator, w.denominator)))
    big = [2**53, 2**53 + 2, 2**63, 2**64]
    for i, m in enumerate(big):
        for sgn in (1, -1):
            w = -sgn * big[(i + 1) % len(big)]
            cases.append((complex(sgn * m / delta, w / delta), delta, sgn * m, w))
    s = 2.0**960                                            # near 2^1000 through the scale
    c = 2.0**40 + 3.0
    cases.append((complex(c, -c / 8), s, int(c) * 2**960, -int(c) * 2**957))
    for z, sc, a, b in cases:                               # the slot values carry the promised products exactly
        assert Fraction(z.real) * Fraction(sc) - a in (0, Fraction(1, 2), Fraction(-1, 2), Fraction(-1, 4))
        assert Fraction(z.imag) * Fraction(sc) - b in (0, Fraction(1, 2), Fraction(-1, 2), Fraction(-1, 4))
    return cases
