"""Polynomial evaluation at its limits without a GPU (DESIGN.md section 2.15): the restatement of the schedule (tests/polyeval_ref.py)
at degree 64 over six levels, with 7 ciphertext limbs and one or two special primes, decrypting under the oracle to p(slots) mod t with
the noise left on q_0 measured; and the emulated ct_lincomb body (tests/emu/emu_lincomb.cpp) at the top of its canonical range."""
import numpy as np
import pytest

import bases
import polyeval_ref as pr
from test_polyeval_cpu import _decrypt_slots, _encrypt_slots, _noise_bits, emu_lincomb, run_emu  # noqa: F401  (emu_lincomb: fixture)

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
T = 65537


def _nonzero_mod_t(rng, n, t=T):
    """n random int64 coefficients, none of them 0 mod t (a coefficient that is 0 mod t drops its power from the schedule)"""
    out = []
    while len(out) < n:
        c = int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64, endpoint=True))
        if c % t:
            out.append(c)
    return out


def limit_polynomials():
    """{name: coefficients a_0 .. a_d}: degree 64 with every coefficient non-zero mod t (INT64_MIN at a_0, INT64_MAX at a_64), degrees
    33 and 63 (the splits of k = 33 and of k = 63 are not powers of two), and a sparse degree 64 (a_64, a_1, a_0 only)"""
    rng = np.random.default_rng(64)
    full = [I64_MIN] + _nonzero_mod_t(rng, 63) + [I64_MAX]
    assert all(c % T for c in full)
    sparse = [-3, I64_MAX] + [0] * 62 + [I64_MIN]
    return {"d64": full, "d33": _nonzero_mod_t(rng, 34), "d63": _nonzero_mod_t(rng, 64), "d64_sparse": sparse}


POLYS = limit_polynomials()
# (Lq, K): six levels of products (D = 6 = Lq - 1) down to Lf = 1; with K = 2 the views at levels 7, 5 and 3 have a ragged last digit
CHAINS = [(7, 1), (7, 2)]


@pytest.mark.parametrize("logn", [10, 12])
@pytest.mark.parametrize("Lq,K", CHAINS)
@pytest.mark.parametrize("name", list(POLYS))
def test_restatement_decrypts_at_degree_64(oracle_mod, capsys, logn, Lq, K, name):
    """the default 60-bit basis, t = 65537: the restatement ends on q_0 alone and decrypts to p(slots) mod t slot by slot; the noise
    t e left on q_0 is printed (DESIGN.md 2.15 records it)"""
    coeffs = POLYS[name]
    B = 2
    top = oracle_mod.Oracle(logn, Lq + K)
    ch = pr.Chain(oracle_mod, logn, top.moduli, K)
    s = top.keygen_secret(70 + K)
    key = top.keygen_relin_grouped(K, 71 + K, T, s)
    z = np.random.default_rng(len(coeffs) * 10 + K).integers(0, T, (B, 2, top.N // 2), dtype=np.int64)
    ct = _encrypt_slots(ch.ct(Lq), np.ascontiguousarray(s[:Lq]), z, T, 80)
    stats = {}
    out = pr.polyeval(ch, T, coeffs, ct, key, stats=stats)
    Lf = Lq - pr.ceil_log2(len(coeffs) - 1)
    assert Lf == 1 and out.shape == (B, 2, 1, top.N)
    if name == "d64":   # every power 2 .. 64 is made: 63 products, and the combination has 64 terms
        assert stats["mul"] == 63
    s0 = np.ascontiguousarray(s[:1])
    assert np.array_equal(_decrypt_slots(ch.ct(1), s0, out, T), pr.poly_mod_t(coeffs, z, T))
    bits = _noise_bits(ch.ct(1), s0, out, T)
    q0 = top.moduli[0].bit_length()
    with capsys.disabled():
        print("\n[polyeval limits] N = %d, Lq = %d, K = %d, %s: noise %d bits, q_0 %d bits, budget left %d bits"
              % (top.N, Lq, K, name, bits, q0, q0 - 1 - bits))
    assert bits < q0 - 1


@pytest.mark.parametrize("basis,variant", [(None, "fast"), (None, "gen"), ("gen_mixed", "gen")])
def test_emulated_lincomb_at_the_top_of_the_range(oracle_mod, emu_lincomb, basis, variant):
    """64 terms, every input q - 1 and every coefficient -1 (c = q - 1 on every limb), the constant -1 and a plaintext addend of q - 1:
    the accumulator starts at 2q - 2, each Shoup product of (q - 1)(q - 1) is at the top of its canonical range, and every sum before a
    word_reduce is the largest that canonical inputs give (not the proven maximum, which shoup_lazy's quotient estimate sets)"""
    logn, L, B, n = 12, 3, 1, 64
    o = oracle_mod.Oracle(logn, L, bases.catalogue(oracle_mod)[basis][:L] if basis else None)
    top = np.array([q - 1 for q in o.moduli], dtype=np.uint64)[None, None, :, None]
    cts = [np.ascontiguousarray(np.broadcast_to(top, (B, 2, L, o.N))) for _ in range(n)]
    pt = np.ascontiguousarray(np.broadcast_to(top[0, 0], (L, o.N)))
    coeffs = [-1] * n
    for addend in (None, pt):
        want = pr.lincomb(o.moduli, cts, coeffs, -1, addend)
        # (q - 1)^2 = 1 mod q: 64 on both components, and the constant and addend take q - 2 more on c0
        assert all(int(want[0, 1, l, 0]) == 64 % q for l, q in enumerate(o.moduli))
        assert np.array_equal(run_emu(emu_lincomb[variant], logn, o.moduli, cts, coeffs, -1, pt=addend), want)
        alias = [c.copy() for c in cts]
        got = run_emu(emu_lincomb[variant], logn, o.moduli, alias, coeffs, -1, pt=addend, out=alias[-1])   # out = the last input
        assert np.array_equal(got, want)
