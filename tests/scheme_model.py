"""An exact model of decryption and of what the evaluator's calls mean on slots, independent of csrc/ (test infrastructure).

The bit-exactness tests compare every kernel with a restatement (the oracle, keys_ref.c, ckks_ref.c, mul_rescale_ref.c) written by
the same hands, so a mistake shared by a kernel and its restatement (a rotation the wrong way, a Galois key for the inverse element, a
gadget factor on the wrong limbs, a missing t^-1 in the BGV correction) passes them.  This model states what the calls *mean* instead:
a ciphertext decrypts to a phase, the phase to slots, and every call to a rule on slots with a noise bound.  From the oracle it uses
only the inverse transform, which tests/test_oracle_vs_sympy.py pins against sympy; everything else is Python integers, numpy and
tests/slots.py (pinned by Horner in tests/test_bgv_encoding_cpu.py).

Phase.  For a ciphertext (c0, c1 [, c2]) over q_0 .. q_{l-1} and a secret s in evaluation form, the phase is c0 + c1 s (+ c2 s^2)
per limb, brought to coefficients by the inverse transform and lifted by the CRT to the centred integer X in (-Q/2, Q/2].

BGV (plaintext modulus t).  X = m + t v with m = [X]_t centred; the message is m mod t read through SlotEncoder, the noise is
max |v| (`noise`).  A call on ciphertexts with noise v_i gives noise at most the bound below, and while that bound stays under
Q / (2t) - 1 the decrypted slots are exactly the rule's.

CKKS (t = 0).  X = Delta m + e; slots are m(zeta_j) with zeta_j = exp(i pi 5^j / N) (tests/ckks.py's convention), decoded from the
exact integers X_k (each divided by Delta once, in float64) by one FFT.  A phase error |e_k| <= E moves a slot by at most N E / Delta.
CKKS errors are tracked on the slots (`ckks_*_slot`): products are exact there, so a product of slots with errors e_a, e_b has error
|z_a| e_b + |z_b| e_a + e_a e_b, and each key switch or division adds N times its coefficient bound over the scale at that point.

Noise bounds (infinity norm of the coefficients, |a b| <= N |a| |b| in Z[X]/(X^N + 1); B_E = 21 is the centred binomial's largest
value; the secret is ternary; tf = t for BGV and 1 for CKKS; all in units of tf).  DESIGN.md section 2.14 gives the encryptions,
2.5 / 2.10 / 2.11 the key switches, 2.9 / 2.11 / 2.19 the divisions:

* fresh symmetric encryption: v <= B_E (the phase is pt + tf e);
* fresh public-key encryption: v <= B_E (2 N + 1) (the phase is pt + tf (e u + e0 + e1 s), u and s ternary);
* ct x ct before the key switch (BGV): X1 X2 = m1 m2 + t (m1 v2 + m2 v1 + t v1 v2) and m1 m2 = [m1 m2]_t + t r with
  |r| <= N t / 4 + 1/2, so v <= N t / 4 + 1 + N (t / 2)(v1 + v2) + N t v1 v2;  the same for a sum of n products, term by term;
* per-limb key switch (2.5): the accumulator adds tf sum_j u_j e_j with 0 <= u_j < q_j:  ks <= N B_E sum_j q_j;
* special-prime key switch (2.10, 2.11; K primes of product P, dnum digits of |g| <= K limbs and product Q_g): the lift of digit g is
  below |g| Q_g, so the accumulator adds tf E with |E| < N B_E sum_g |g| Q_g, and the division subtracts tf W with |W| <= K P (N + 1)/2:
  ks <= N B_E sum_g |g| Q_g / P + K (N + 1) / 2  (about dnum K N Q_g B_E / P plus the rounding term);
* a rotation keeps the norm of its input (sigma_g permutes coefficients up to sign) and adds one key switch; a sum of n_rot rotations
  summed before one division (2.17) adds n_rot accumulator terms and one rounding term; an inner product (2.18) one key switch;
* a division with k centred lifts (mod_switch_down: by q_last, k = 1; mod_down_special: by P, k = K; the fused rescale of 2.19: by
  P q_last, k = K + 1) of a phase with noise v, plus an accumulator term acc already divided by P, leaves
  v' <= (1/2 + v + acc) / D + k (N + 1) / 2 + 1/2 with D the divisor left after P (q_last, P or q_last); the message is multiplied
  by the divisor's inverse mod t (BGV) or divided by it (CKKS: the scale becomes Delta_a Delta_b / q_last).

The bounds are worst cases; measured noise sits far below them, which is why the tests print both.
"""
import math

import numpy as np

import slots as slots_mod

B_E = 21          # |e| of the centred binomial (eta = 21)


def prod(xs):
    p = 1
    for x in xs:
        p *= int(x)
    return p


def centred(x, m):
    r = x % m
    return r - m if r > m // 2 else r


def bits(v):
    return math.log2(v) if v > 0 else float("-inf")


# ---- phase and decryption -----------------------------------------------------------------------------------------------------------

class Model:
    """Decryption under one basis: `moduli` the context's moduli (ciphertexts over any prefix of them), `oracle_mod` for the oracle's
    inverse transform only."""

    def __init__(self, oracle_mod, log_n, moduli):
        self.om, self.log_n, self.N = oracle_mod, log_n, 1 << log_n
        self.moduli = [int(q) for q in moduli]
        self._o = {}
        self._enc = {}

    def _oracle(self, ell):
        if ell not in self._o:
            self._o[ell] = self.om.Oracle(self.log_n, ell, self.moduli[:ell])
        return self._o[ell]

    def phase(self, sk, ct):
        """centred integer coefficients (a list of N Python ints) of c0 + c1 s (+ c2 s^2) and Q; ct [n_comp][ell][N], sk [>= ell][N]
        in evaluation form (a top-level secret serves every prefix: its rows are per-limb transforms of one polynomial)"""
        ct = np.asarray(ct, dtype=np.uint64)
        n_comp, ell = ct.shape[0], ct.shape[1]
        assert 2 <= n_comp <= 3 and ell <= len(self.moduli)
        ev = np.empty((ell, self.N), dtype=np.uint64)
        for l in range(ell):
            q = self.moduli[l]
            s = np.asarray(sk[l], dtype=np.uint64).astype(object)
            acc = ct[0, l].astype(object) + ct[1, l].astype(object) * s
            if n_comp == 3:
                acc = acc + ct[2, l].astype(object) * (s * s % q)
            ev[l] = (acc % q).astype(np.uint64)
        co = self._oracle(ell).ntt_inv(ev[None])[0]
        Q = prod(self.moduli[:ell])
        x = np.zeros(self.N, dtype=object)
        for l in range(ell):
            q = self.moduli[l]
            Ql = Q // q
            x = x + co[l].astype(object) * (Ql * pow(Ql, -1, q))
        x = x % Q
        return [int(v) - Q if v > Q // 2 else int(v) for v in x], Q

    def encoder(self, t):
        if t not in self._enc:
            self._enc[t] = slots_mod.SlotEncoder(self.N, t)
        return self._enc[t]

    def bgv(self, sk, ct, t):
        """(slots [2][N/2] in [0, t), noise max |v| with X = [X]_t + t v, Q)"""
        X, Q = self.phase(sk, ct)
        m = [centred(x, t) for x in X]
        v = max(abs(x - mm) for x, mm in zip(X, m)) // t
        return self.encoder(t).decode(np.array([mm % t for mm in m], dtype=np.uint64)), v, Q

    def ckks(self, sk, ct, scale):
        """(slots [N/2] complex, the exact phase coefficients, Q)"""
        X, Q = self.phase(sk, ct)
        return ckks_decode(X, self.N, scale), X, Q


def ckks_decode(X, n, scale):
    """slot j = sum_k (X_k / scale) zeta_j^k, zeta_j = exp(i pi 5^j / n): the exact integers divided once, then one FFT"""
    c = np.array([x / scale for x in X], dtype=np.float64)
    k = np.arange(n)
    vals = n * np.fft.ifft(c * np.exp(1j * np.pi * k / n))         # vals[i] = m(exp(i pi (2i + 1) / n))
    e = np.array([pow(5, j, 2 * n) for j in range(n // 2)])
    return vals[(e - 1) // 2]


def ckks_decode_slack(n, z_max):
    """the float64 error of ckks_decode: each X_k / scale rounded once (relative 2^-53 of at most z_max) and the FFT"""
    return n * z_max * 2.0**-50 * max(1, int(math.log2(n)))


# ---- the meaning of the calls on slots ------------------------------------------------------------------------------------------------

def bgv_rotate(z, k):
    """BGV slots [2][N/2]: Galois element 5^k rolls each row left by k"""
    return np.roll(np.asarray(z), -k, axis=1)


def bgv_conjugate(z):
    """BGV slots: the element 2N - 1 swaps the rows"""
    return np.asarray(z)[::-1].copy()


def ckks_rotate(z, k):
    """CKKS slots [N/2]: slot j + k moves to slot j"""
    return np.roll(np.asarray(z), -k)


def ckks_conjugate(z):
    return np.conj(np.asarray(z))


def bgv_galois(z, g, n):
    """the slot rule of any Galois element 5^k or (2N - 1) 5^k"""
    two_n = 2 * n
    if g == two_n - 1:
        return bgv_conjugate(z)
    return bgv_rotate(z, dlog5(g, n))


def ckks_galois(z, g, n):
    if g == 2 * n - 1:
        return ckks_conjugate(z)
    return ckks_rotate(z, dlog5(g, n))


def dlog5(g, n):
    """k in [0, N/2) with 5^k = g mod 2N"""
    x = 1
    for k in range(n // 2):
        if x == g:
            return k
        x = x * 5 % (2 * n)
    raise ValueError("not a power of 5 mod 2N")


def bgv_mul(a, b, t):
    return np.asarray(a, dtype=object) * np.asarray(b, dtype=object) % t


def bgv_dot(xs, ys, t):
    acc = 0
    for x, y in zip(xs, ys):
        acc = acc + np.asarray(x, dtype=object) * np.asarray(y, dtype=object)
    return acc % t


def bgv_scale(z, f, t):
    """slots times the integer f (a factor such as q^-1 mod t)"""
    return np.asarray(z, dtype=object) * (int(f) % t) % t


def bgv_lincomb(zs, cs, t, constant=0):
    acc = int(constant)
    for z, c in zip(zs, cs):
        acc = acc + np.asarray(z, dtype=object) * int(c)
    return np.asarray(acc, dtype=object) % t


def ckks_lincomb(zs, cs):
    return sum(complex(c) * np.asarray(z) for z, c in zip(zs, cs))


def window_sums(z, stride, count, axis=-1):
    """slot i of the result is sum_{j < count} z[(i + j stride) mod N/2] (the slot sum of DESIGN.md 2.17)"""
    return sum(np.roll(np.asarray(z, dtype=object), -j * stride, axis=axis) for j in range(count))


# ---- noise bounds (module docstring), in units of tf = t (BGV) or 1 (CKKS) -----------------------------------------------------------

def fresh_bound(n, public=False):
    return B_E * (2 * n + 1) if public else B_E


def digits(moduli_q, K):
    """the digits of a special-prime key switch over the ciphertext moduli: K consecutive limbs each, the last one ragged"""
    return [moduli_q[i:i + K] for i in range(0, len(moduli_q), K)]


def ks_bound(n, moduli_q, K, special=()):
    """the noise a key switch adds: K = 0 per-limb digits without special primes, else the special primes `special` (K of them)"""
    if K == 0:
        return n * B_E * sum(moduli_q)
    P = prod(special)
    assert len(special) == K
    return n * B_E * sum(len(g) * prod(g) for g in digits(moduli_q, K)) / P + K * (n + 1) / 2


def ks_acc_bound(n, moduli_q, K, special):
    """the accumulator term of one special-prime key switch alone, already divided by P (the rounding term comes once per division)"""
    return n * B_E * sum(len(g) * prod(g) for g in digits(moduli_q, K)) / prod(special)


def tensor_bound(n, t, v1, v2):
    """BGV: the noise of the phase of a ct x ct before relinearisation, message [m1 m2]_t"""
    return n * t / 4 + 1 + n * (t / 2) * (v1 + v2) + n * t * v1 * v2


def mul_bound(n, t, v1, v2, ks):
    return tensor_bound(n, t, v1, v2) + ks


def dot_bound(n, t, pairs, ks):
    return sum(tensor_bound(n, t, a, b) for a, b in pairs) + ks


def rotate_bound(v, ks):
    return v + ks


def rotate_sum_bound(n, moduli_q, K, special, v, n_rot):
    """ct + sum of n_rot rotations with one division (DESIGN.md 2.17)"""
    return (1 + n_rot) * v + n_rot * ks_acc_bound(n, moduli_q, K, special) + K * (n + 1) / 2


def divide_bound(n, v, D, n_lifts, acc=0.0):
    """BGV: the noise after dividing a phase with noise v (plus an accumulator term acc already divided by P) by D with n_lifts
    centred lifts of the divided residues: X' = (m + t (v + acc) - t W) / D, |W| <= n_lifts D (N + 1) / 2, message m D^-1 mod t"""
    return (0.5 + v + acc) / D + n_lifts * (n + 1) / 2 + 0.5


def ckks_fresh_slot(n, scale, z_max, public=False):
    """CKKS slot error of a fresh encryption at `scale`: the noise plus the encoder's rounding (within 1 of rint of a value that is
    itself within log2(N) 2^-53 scale max|z| of the exact one, DESIGN.md 2.12), N coefficients per slot"""
    return n * (fresh_bound(n, public) + 1 + math.log2(n) * 2.0**-53 * scale * z_max) / scale


def ckks_mul_slot(za, ea, zb, eb):
    """CKKS slot error of a slot-wise product (z_a + d_a)(z_b + d_b) - z_a z_b, |d| <= e: products are exact on slots"""
    return za * eb + zb * ea + ea * eb


def ckks_ks_slot(n, ks, scale):
    """the slot error a phase error of at most ks per coefficient adds at `scale`"""
    return n * ks / scale


def ckks_div_slot(n, n_lifts, scale_out):
    """the slot error of a division's rounding (n_lifts centred lifts, |W| <= n_lifts D (N + 1) / 2) at the scale after it"""
    return n * n_lifts * (n + 1) / 2 / scale_out


def linear_bound(n, t, v, ks, n_diags, giant):
    """W x by baby-step/giant-step diagonals (plaintexts with coefficients |d| <= t/2): every diagonal product of a rotation of x,
    plus one key switch per Horner step"""
    return n_diags * (n * t / 4 + 1 + n * (t / 2) * (v + ks)) + giant * ks
