"""Pins tests/scheme_model.py without a GPU: its phase is the oracle's decryption (BGV) and tests/ckks.py's (CKKS), its slot rules are
what the automorphism X -> X^g does to the coefficients, and its noise bounds hold on the oracle's products, rotations and divisions."""
import numpy as np
import pytest

import ckks
import scheme_model as sm
from ckks_polyeval_ref import ckks_chain

T = 65537


def sigma(coeffs, g, n):
    """X -> X^g on integer coefficients: X^k goes to +-X^(k g mod N), negated when k g mod 2N >= N"""
    out = [0] * n
    for k, c in enumerate(coeffs):
        e = k * g % (2 * n)
        if e < n:
            out[e] += c
        else:
            out[e - n] -= c
    return out


def test_phase_is_the_oracle_decryption(oracle_mod):
    o = oracle_mod.Oracle(10, 3)
    m = sm.Model(oracle_mod, 10, o.moduli)
    s = o.keygen_secret(3)
    rng = np.random.default_rng(1)
    z = rng.integers(0, T, (2, o.N // 2))
    pt = m.encoder(T).encode(z)
    ct = o.encrypt(4, T, s, pt)
    X, Q = m.phase(s, ct)
    assert Q == sm.prod(o.moduli)
    assert np.array_equal(np.array([x % T for x in X], dtype=np.uint64), o.decrypt(s, ct, T))
    slots, v, _ = m.bgv(s, ct, T)
    assert np.array_equal(slots, z.astype(np.uint64))
    assert 0 < v <= sm.fresh_bound(o.N)
    # three components: the tensor product decrypts under (1, s, s^2) to the slot product
    d = o.ct_tensor(ct[None], o.encrypt(5, T, s, pt)[None])[0]
    assert np.array_equal(np.array([x % T for x in m.phase(s, d)[0]], dtype=np.uint64), o.decrypt(s, d, T))
    assert np.array_equal(m.bgv(s, d, T)[0], sm.bgv_mul(z, z, T).astype(np.uint64))


def test_ckks_phase_and_decode_agree_with_tests_ckks(oracle_mod):
    o = oracle_mod.Oracle(10, 3)
    m = sm.Model(oracle_mod, 10, o.moduli)
    s = o.keygen_secret(7)
    rng = np.random.default_rng(2)
    z = rng.uniform(-1, 1, o.N // 2) + 1j * rng.uniform(-1, 1, o.N // 2)
    scale = 2.0**40
    ct = ckks.encrypt(o, s, ckks.encode(z, range(o.N // 2), o.N, scale), 8)
    X, _ = m.phase(s, ct)
    assert X == ckks.decrypt_coeffs(o, s, ct)
    got = sm.ckks_decode(X, o.N, scale)
    assert np.abs(got - ckks.decode(X, range(o.N // 2), o.N, scale)).max() < 1e-9
    assert np.abs(got - z).max() <= sm.ckks_fresh_slot(o.N, scale, np.sqrt(2))


@pytest.mark.parametrize("log_n", [4, 5, 7])
def test_automorphism_agrees_with_the_slot_rules(oracle_mod, log_n):
    """g = 5^k for k = 1, -1, N/4 - 1 and the conjugation 2N - 1, on BGV coefficients mod t and on CKKS integer coefficients"""
    n = 1 << log_n
    m = sm.Model(oracle_mod, log_n, [])
    enc = m.encoder(T)
    rng = np.random.default_rng(log_n)
    zb = rng.integers(0, T, (2, n // 2))
    pb = [int(c) for c in enc.encode(zb)]
    zc = rng.uniform(-1, 1, n // 2) + 1j * rng.uniform(-1, 1, n // 2)
    scale = 2.0**40
    pc = ckks.encode(zc, range(n // 2), n, scale)
    for k in (1, -1, n // 4 - 1):
        g = pow(5, k % (n // 2), 2 * n)
        assert sm.dlog5(g, n) == k % (n // 2)
        assert np.array_equal(enc.decode(np.array([c % T for c in sigma(pb, g, n)], dtype=np.uint64)),
                              sm.bgv_rotate(zb, k).astype(np.uint64))
        assert np.abs(sm.ckks_decode(sigma(pc, g, n), n, scale) - sm.ckks_rotate(zc, k)).max() < 1e-9
        assert np.array_equal(sm.bgv_galois(zb, g, n), sm.bgv_rotate(zb, k))
    g = 2 * n - 1
    assert np.array_equal(enc.decode(np.array([c % T for c in sigma(pb, g, n)], dtype=np.uint64)), zb[::-1].astype(np.uint64))
    assert np.abs(sm.ckks_decode(sigma(pc, g, n), n, scale) - np.conj(zc)).max() < 1e-9
    # the inverse element is a different rule: a model that confused 5^k and 5^-k would fail here
    g = pow(5, n // 2 - 1, 2 * n)
    assert not np.array_equal(enc.decode(np.array([c % T for c in sigma(pb, g, n)], dtype=np.uint64)),
                              sm.bgv_rotate(zb, 1).astype(np.uint64))


def test_window_sums_and_lincomb():
    z = np.arange(16).reshape(2, 8)
    w = sm.window_sums(z, 2, 3)
    assert w[0][0] == 0 + 2 + 4 and w[1][7] == 15 + 9 + 11
    assert list(sm.bgv_lincomb([z[0], z[1]], [2, -1], 7, 3)) == [(2 * a - b + 3) % 7 for a, b in zip(z[0], z[1])]
    assert sm.digits([1, 2, 3, 4, 5], 2) == [[1, 2], [3, 4], [5]]


def test_bgv_bounds_hold_on_oracle_products_rotations_and_divisions(oracle_mod):
    """N = 1024: per-limb relinearisation and rotation, the grouped key switch with a ragged last digit (Lq = 5, K = 2), the modulus
    switch and the division by P; each result decrypts to the slot rule and its noise is below the model's bound"""
    log_n, Lq, K = 10, 5, 2
    o = oracle_mod.Oracle(log_n, Lq + K)
    n, qs, ps = o.N, o.moduli[:Lq], o.moduli[Lq:]
    oq = oracle_mod.Oracle(log_n, Lq, qs)
    m = sm.Model(oracle_mod, log_n, o.moduli)
    s = o.keygen_secret(11)
    sq = np.ascontiguousarray(s[:Lq])
    rng = np.random.default_rng(3)
    z1, z2 = rng.integers(0, T, (2, 2, n // 2))
    enc = m.encoder(T)
    c1, c2 = oq.encrypt(12, T, sq, enc.encode(z1)), oq.encrypt(13, T, sq, enc.encode(z2))
    v1, v2 = m.bgv(sq, c1, T)[1], m.bgv(sq, c2, T)[1]
    cases = []
    # per-limb digits over the ciphertext moduli
    ks0 = sm.ks_bound(n, qs, 0)
    cases.append(("mul per-limb", oq.ct_mul_relin(c1[None], c2[None], oq.keygen_relin(14, T, sq))[0], sm.bgv_mul(z1, z2, T),
                  sm.mul_bound(n, T, v1, v2, ks0)))
    g = o.galois_elt(-1)
    cases.append(("rotate per-limb", oq.rotate(c1[None], g, oq.keygen_galois(15, T, sq, g))[0], sm.bgv_rotate(z1, -1),
                  sm.rotate_bound(v1, ks0)))
    ksg = sm.ks_bound(n, qs, K, ps)
    cases.append(("mul grouped", o.ct_mul_relin_grouped(K, c1[None], c2[None], o.keygen_relin_grouped(K, 16, T, s), T)[0],
                  sm.bgv_mul(z1, z2, T), sm.mul_bound(n, T, v1, v2, ksg)))
    g = 2 * n - 1
    cases.append(("conjugate grouped", o.rotate_grouped(K, c1[None], g, o.keygen_galois_grouped(K, 17, T, s, g), T)[0], z1[::-1],
                  sm.rotate_bound(v1, ksg)))
    for what, ct, want, bound in cases:
        got, v, Q = m.bgv(s, ct, T)
        assert np.array_equal(got, np.asarray(want, dtype=np.uint64)), what
        assert v <= bound < Q / (2 * T) - 1, (what, v, bound)
    # the modulus switch: the message times q_last^-1 mod t
    prod_ct = cases[2][1]
    vp = m.bgv(s, prod_ct, T)[1]
    low = oq.mod_switch_down(prod_ct, T).reshape(2, Lq - 1, n)
    got, v, _ = m.bgv(s, low, T)
    assert np.array_equal(got, sm.bgv_scale(sm.bgv_mul(z1, z2, T), pow(qs[-1], -1, T), T).astype(np.uint64))
    assert v <= sm.divide_bound(n, vp, qs[-1], 1)
    # the division by P on a context whose special rows carry P times a ciphertext: exact, no factor
    up = np.concatenate([c1, np.zeros((2, K, n), dtype=np.uint64)], axis=1)
    Pq = [sm.prod(ps) % q for q in qs]
    up[:, :Lq] = (up[:, :Lq].astype(object) * np.array(Pq, dtype=object)[:, None] % np.array(qs, dtype=object)[:, None]).astype(np.uint64)
    got, v, _ = m.bgv(s, o.mod_down_special(K, up, T).reshape(2, Lq, n), T)
    assert np.array_equal(got, z1.astype(np.uint64)) and v <= sm.divide_bound(n, v1 * sm.prod(ps), sm.prod(ps), K)


def test_ckks_bounds_hold_on_an_oracle_product_and_rescale(oracle_mod):
    """the CKKS chain of the polynomial-evaluation tests (q_1 .. about 2^45), Delta = 2^40: ct x ct with the grouped key, then the
    division by q_last; the slots are within the model's error of z1 z2 at scale Delta^2 / q_last"""
    log_n, Lq, K = 10, 4, 2
    moduli = ckks_chain(oracle_mod, Lq, K)
    o = oracle_mod.Oracle(log_n, Lq + K, moduli)
    n, qs, ps = o.N, moduli[:Lq], moduli[Lq:]
    oq = oracle_mod.Oracle(log_n, Lq, qs)
    m = sm.Model(oracle_mod, log_n, moduli)
    s = o.keygen_secret(21)
    sq = np.ascontiguousarray(s[:Lq])
    rng = np.random.default_rng(4)
    z1, z2 = (rng.uniform(-1, 1, n // 2) + 1j * rng.uniform(-1, 1, n // 2) for _ in range(2))
    D = 2.0**40
    c1 = ckks.encrypt(oq, sq, ckks.encode(z1, range(n // 2), n, D), 22)
    c2 = ckks.encrypt(oq, sq, ckks.encode(z2, range(n // 2), n, D), 23)
    zmax = np.sqrt(2)
    e0 = sm.ckks_fresh_slot(n, D, zmax)
    pr = o.ct_mul_relin_grouped(K, c1[None], c2[None], o.keygen_relin_grouped(K, 24, 0, s), 0)[0]
    e_prod = sm.ckks_mul_slot(zmax, e0, zmax, e0) + sm.ckks_ks_slot(n, sm.ks_bound(n, qs, K, ps), D * D)
    got, _, _ = m.ckks(s, pr, D * D)
    assert np.abs(got - z1 * z2).max() <= e_prod + sm.ckks_decode_slack(n, 2)
    low = oq.mod_switch_down(pr, 0).reshape(2, Lq - 1, n)
    sc = D * D / qs[-1]
    got, _, _ = m.ckks(s, low, sc)
    err = np.abs(got - z1 * z2).max()
    bound = e_prod + sm.ckks_div_slot(n, 1, sc) + sm.ckks_decode_slack(n, 2)
    assert err <= bound, (err, bound)
    assert bound < 2.0**-8
