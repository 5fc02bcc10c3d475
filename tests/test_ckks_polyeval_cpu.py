"""CKKS polynomial evaluation of DESIGN.md section 2.16 without a GPU: the restatement (tests/ckks_polyeval_ref.py), composed on the
oracle, decrypts and decodes (tests/ckks_ref) to p(z) within the recorded bound; deliberate schedule errors move the slots far off;
the argument rules.  Encryption and keys (t = 0) are those of section 2.14 (tests/keys_ref.py)."""
import math

import numpy as np
import pytest

import ckks_polyeval_ref as cr
import ckks_ref
import keys_ref as kr
import polyeval_ref as pr

SEED = bytes(range(40, 72))
DELTA = 2.0**45

# the recorded bound (section 2.16): |decoded - p(z)| <= ERR_REL * (1 + sum_k |a_k| |z|^k) per slot.  The largest ratio measured
# below and on the device is recorded in DESIGN.md (2^-29.7 at most); ERR_REL leaves a margin of more than 32x over it.
ERR_REL = 2.0**-24


def setup(oracle_mod, logn, Lq, K, seed=SEED):
    moduli = cr.ckks_chain(oracle_mod, Lq, K)
    ch = pr.Chain(oracle_mod, logn, moduli, K)
    top = oracle_mod.Oracle(logn, Lq + K, moduli)
    s = kr.secret(top, seed)
    key = kr.relin_key(top, K, 0, s, seed)
    return ch, s, key


def encrypt(ch, s, z, scale, seed=SEED):
    o = ch.ct(ch.Lq)
    pt = ckks_ref.encode(o, z, scale)
    return kr.encrypt(o, 0, s, seed, 0, pt)


def decode(ch, s, ct, scale):
    o = ch.ct(ct.shape[2])
    return ckks_ref.decode(o, kr.decrypt(o, s, ct), scale)


def rel_error(coeffs, z, got):
    """the largest |got - p(z)| / (1 + sum |a_k| |z|^k) over the slots"""
    return float(np.max(np.abs(got - cr.poly_eval(coeffs, z)) / (1 + cr.power_sum(coeffs, z))))


def slots(rng, B, n):
    return rng.uniform(-1, 1, (B, n)) + 0j


CASES = [
    [0.25, 0.5],                                                   # d = 1
    [0.1, -0.3, 0.7],                                              # d = 2
    [0.0, 1.0, 0.0, -1.0 / 6],                                     # d = 3, zero coefficients
    [0.5, 0.25, 0.0, -0.02, 0.0, 0.001, 0.0, -1e-4],               # d = 7 (odd)
    [1.0, -2.0, 3.0, -4.0, 5.0, -6.0, 7.0, -8.0, 9.0],             # d = 8
    [0.0] * 8,                                                     # every coefficient 0 (x with coefficient 0)
    [-0.0, 0.0, -0.0, 3.0],                                        # -0.0 is skipped like 0.0
    [1000.0, -750.5, 2048.0, 3e3],                                 # large coefficients: c_k far beyond 2^53
]


@pytest.mark.parametrize("logn", [10, 12])
@pytest.mark.parametrize("coeffs", CASES, ids=lambda c: "d%d" % (len(c) - 1))
def test_restatement_decodes_to_p_of_z(oracle_mod, logn, coeffs, capsys):
    Lq, K, B = 5, 2, 2
    ch, s, key = setup(oracle_mod, logn, Lq, K)
    rng = np.random.default_rng(len(coeffs) * 7 + logn)
    z = slots(rng, B, ch.ct(Lq).N // 2)
    ct = encrypt(ch, s, z, DELTA)
    stats = {}
    out = cr.polyeval(ch, coeffs, DELTA, ct, key, stats=stats)
    D = pr.ceil_log2(len(coeffs) - 1)
    assert out.shape == (B, 2, Lq - D - 1, 1 << logn)
    got = decode(ch, s, out, DELTA)
    err = rel_error(coeffs, z, got)
    with capsys.disabled():
        print("\n[ckks polyeval] N = %d, d = %d: relative error %.3g (2^%.1f), launches %d" % (1 << logn, len(coeffs) - 1, err, math.log2(max(err, 2.0**-99)),
                                                                                              stats["launches"]))
    assert err <= ERR_REL


def test_sparse_degree_64(oracle_mod, capsys):
    """a sparse degree 64 on Lq = 8, K = 2 at N = 1024: six levels of products, the result on q_0 alone"""
    logn, Lq, K, B = 10, 8, 2, 1
    ch, s, key = setup(oracle_mod, logn, Lq, K)
    coeffs = [0.0] * 65
    coeffs[0], coeffs[1], coeffs[5], coeffs[33], coeffs[64] = 0.5, -1.0, 0.25, 0.125, 2.0
    z = slots(np.random.default_rng(64), B, ch.ct(Lq).N // 2)
    stats = {}
    out = cr.polyeval(ch, coeffs, DELTA, encrypt(ch, s, z, DELTA), key, stats=stats)
    assert out.shape[2] == 1
    err = rel_error(coeffs, z, decode(ch, s, out, DELTA))
    with capsys.disabled():
        print("\n[ckks polyeval] N = 1024, sparse d = 64: relative error %.3g (2^%.1f), %d products, %d cuts" % (err, math.log2(err), stats["mul"],
                                                                                                          stats["cut"]))
    assert err <= ERR_REL


def test_output_scale(oracle_mod):
    """scale_out = 2^40: the result decodes at 2^40"""
    logn, Lq, K = 10, 5, 2
    ch, s, key = setup(oracle_mod, logn, Lq, K)
    coeffs = [0.1, 0.2, 0.3]
    z = slots(np.random.default_rng(9), 1, ch.ct(Lq).N // 2)
    out = cr.polyeval(ch, coeffs, DELTA, encrypt(ch, s, z, DELTA), key, scale_out=2.0**40)
    assert rel_error(coeffs, z, decode(ch, s, out, 2.0**40)) <= ERR_REL


@pytest.mark.parametrize("mutant", ["rescale_align", "no_scales", "comb_after", "no_special_rows"])
def test_schedule_mutants_move_the_slots_far_off(oracle_mod, mutant):
    logn, Lq, K = 10, 5, 2
    ch, s, key = setup(oracle_mod, logn, Lq, K)
    coeffs = [0.5, 0.25, -0.5, 0.125, 0.0, 0.1, 0.0, -0.05]
    z = slots(np.random.default_rng(5), 1, ch.ct(Lq).N // 2)
    out = cr.polyeval(ch, coeffs, DELTA, encrypt(ch, s, z, DELTA), key, mutate=mutant)
    err = rel_error(coeffs, z, decode(ch, s, out, DELTA))
    assert err > 2.0**10 * ERR_REL, (mutant, err)   # no_scales moves least on this chain: its scales drift by q_i / 2^45 - 1 < 2^-12


@pytest.mark.parametrize("Lq,K", [(4, 2), (5, 2), (6, 4), (8, 2)])
def test_log2_qp_of_the_test_chains(oracle_mod, Lq, K, capsys):
    """log2 QP of the CKKS chains of the tests, printed for section 2.16 next to the HE-standard bounds (128-bit classical,
    ternary secret: 109 bits at N = 4096, 218 at 8192, 438 at 16384)"""
    moduli = cr.ckks_chain(oracle_mod, Lq, K)
    bits = sum(math.log2(q) for q in moduli)
    with capsys.disabled():
        print("\n[ckks chain] Lq = %d, K = %d: log2 QP = %.1f" % (Lq, K, bits))
    assert len(set(moduli)) == Lq + K and moduli[0].bit_length() == 60 and all(q.bit_length() == 46 for q in moduli[1:Lq])


def test_argument_rules():
    cr.check(1, 2, 1)
    cr.check(64, 8, 3)
    for d, Lq, K in [(0, 5, 2), (65, 9, 2), (8, 4, 2), (4, 5, 5), (64, 8, 4), (2, 2, 1)]:
        with pytest.raises(ValueError):
            cr.check(d, Lq, K)
    for bad in (math.inf, -math.inf, math.nan):
        with pytest.raises(ValueError):
            cr.check(2, 5, 2, coeffs=[1.0, bad, 0.0])
        with pytest.raises(ValueError):
            cr.check(2, 5, 2, scale_in=bad)
        with pytest.raises(ValueError):
            cr.check(2, 5, 2, scale_out=bad)
    for bad in (0.0, -1.0):
        with pytest.raises(ValueError):
            cr.check(2, 5, 2, scale_in=bad)


def test_coefficients_are_exact_integers():
    """the combination's coefficients: c_k = rint((a_k m) / s_k), c_0 = rint(a_0 m), m = S q_{Lc-1}; c_0 near 2^90 is normal"""
    moduli = [(1 << 60) - 1, (1 << 45) + 1, (1 << 45) + 3, (1 << 45) + 5, 7, 11]
    Lc, terms, c0 = cr.coefficients(moduli, 4, [1.0, 0.5, 0.0, 0.25], DELTA)
    assert Lc == 2
    m = DELTA * float(moduli[1])
    assert c0 == float(round(1.0 * m)) and c0 > 2.0**89
    assert [k for k, _ in terms] == [1, 3]
    assert all(c == float(round(c)) for _, c in terms)
