"""Scalar linear combinations and BGV polynomial evaluation without a GPU (DESIGN.md section 2.15): the product's ct_lincomb body run by
the host emulator (tests/emu/emu_lincomb.cpp) in both arithmetic variants against Python integers, the level keys restricted from the
top-level key, and the restatement of the schedule (tests/polyeval_ref.py) decrypting under the oracle to p(slots) mod t."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import bgv_ref
import polyeval_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
T = 65537


def _build(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_lincomb_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_lincomb.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "eval.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_lincomb.argtypes = [C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def emu_lincomb():
    return {v: _build(v) for v in ("gen", "fast")}


def run_emu(lib, logn, moduli, cts, coeffs, constant, pt=None, out=None):
    L, n = len(moduli), len(cts)
    B = cts[0].shape[0]
    if out is None:
        out = np.zeros_like(cts[0])
    ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in cts])
    cs = (C.c_int64 * n)(*[int(c) for c in coeffs])
    mods = (C.c_uint64 * L)(*[int(q) for q in moduli])
    assert lib.emu_lincomb(logn, L, mods, n, ptrs, cs, int(constant), None if pt is None else pt.ctypes.data, out.ctypes.data, B) == 0
    return out


@pytest.mark.parametrize("basis,variant", [(None, "fast"), (None, "gen"), ("gen_mixed", "gen")])
@pytest.mark.parametrize("n_terms", [1, 7, 8, 9, 64])
def test_emulated_lincomb_equals_python_integers(oracle_mod, emu_lincomb, basis, variant, n_terms):
    logn, L, B = 12, 2, 1
    o = oracle_mod.Oracle(logn, L, bases.catalogue(oracle_mod)[basis][:L] if basis else None)
    rng = np.random.default_rng(n_terms)
    cts = [o.fill_uniform(10 + i, 2 * B).reshape(B, 2, L, o.N) for i in range(n_terms)]
    for ct in cts[: max(1, n_terms // 2)]:   # inputs at q - 1: the largest lazy sums
        for l, q in enumerate(o.moduli):
            ct[:, :, l] = q - 1
    special = [I64_MIN, I64_MAX, 0, 1, -1]
    coeffs = [special[i] if i < len(special) else int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)) for i in range(n_terms)]
    if n_terms == 64:
        coeffs[5:] = [I64_MIN if i % 2 else -1 for i in range(59)]
    for constant in (I64_MAX, I64_MIN, 0):
        want = pr.lincomb(o.moduli, cts, coeffs, constant)
        assert np.array_equal(run_emu(emu_lincomb[variant], logn, o.moduli, cts, coeffs, constant), want)
    pt = o.fill_uniform(99, 1).reshape(L, o.N)
    alias = [c.copy() for c in cts]
    got = run_emu(emu_lincomb[variant], logn, o.moduli, alias, coeffs, -7, pt=pt, out=alias[0])   # out = the first input
    assert np.array_equal(got, pr.lincomb(o.moduli, cts, coeffs, -7, pt))


def test_restricted_keys_decrypt_products_at_every_level(oracle_mod):
    """Lq = 5, K = 2: levels 5 .. 2, the key of level 5 and 3 has a ragged last digit; each level's product decrypts to m1 m2 mod t"""
    logn, Lq, K = 10, 5, 2
    top = oracle_mod.Oracle(logn, Lq + K)
    ch = pr.Chain(oracle_mod, logn, top.moduli, K)
    s = top.keygen_secret(3)
    key = top.keygen_relin_grouped(K, 4, T, s)
    rng = np.random.default_rng(1)
    m1, m2 = (rng.integers(0, T, top.N).astype(np.uint64) for _ in range(2))
    from test_oracle_kat import negacyclic_mod_t
    want = negacyclic_mod_t(m1, m2, T)
    for l in range(Lq, K - 1, -1):
        o = ch.ct(l)
        sl = np.ascontiguousarray(s[:l])
        c1, c2 = o.encrypt(5, T, sl, m1), o.encrypt(6, T, sl, m2)
        kl = pr.restrict_key(key, Lq, K, l)
        assert kl.shape[0] == -(-l // K)
        prod = ch.ks(l).ct_mul_relin_grouped(K, c1[None], c2[None], kl, T)[0]
        assert np.array_equal(o.decrypt(sl, prod, T), want), l
        bad = np.ascontiguousarray(np.concatenate([key[:kl.shape[0], :, :l], key[:kl.shape[0], :, l:l + K]], axis=2))
        if l < Lq:   # without the special-prime rows the level's key is another key
            prod = ch.ks(l).ct_mul_relin_grouped(K, c1[None], c2[None], bad, T)[0]
            assert not np.array_equal(o.decrypt(sl, prod, T), want), l


def _encrypt_slots(o, s, z, t, seed):
    enc = bgv_ref.encoder(o.N, t)
    return np.stack([o.encrypt(seed + i, t, s, enc.encode(zi)) for i, zi in enumerate(z)])


def _decrypt_slots(o, s, ct, t):
    enc = bgv_ref.encoder(o.N, t)
    return np.stack([enc.decode(np.asarray(o.decrypt(s, c, t), dtype=np.uint64)) for c in ct]).astype(np.uint64)


def _noise_bits(o, s, ct, t):
    """log2 of the largest centred coefficient of the phase minus its message (the noise t e), per ciphertext"""
    out = []
    for c in ct:
        vals = bgv_ref.centred_values(o, o.phase(s, c))   # coefficient form
        m = [v % t for v in vals]
        out.append(max(abs(v - (mi if mi <= t // 2 else mi - t)) for v, mi in zip(vals, m)).bit_length())
    return max(out)


DEGREES = [[3, 5], [1, 0, 2], [0, -1, 0, 4], [2, 1, 1, 1, 1, 1, 1, 7], [9, 0, 3, 0, 0, 0, 0, 0, 1], [0, 0, 0, 0, 0, 0, 0, 0],
           [T - 1, 123456, -9, 65536, 8, 7, 6, 5, 4]]


@pytest.mark.parametrize("coeffs", DEGREES)
def test_restatement_decrypts_to_p_of_the_slots(oracle_mod, coeffs):
    """degrees 1, 2, 3, 7 and 8, random, zero and out-of-range coefficients; Lq = 4, K = 2 at N = 1024"""
    logn, Lq, K, B = 10, 4, 2, 2
    top = oracle_mod.Oracle(logn, Lq + K)
    ch = pr.Chain(oracle_mod, logn, top.moduli, K)
    s = top.keygen_secret(11)
    key = top.keygen_relin_grouped(K, 12, T, s)
    z = np.random.default_rng(len(coeffs)).integers(0, T, (B, 2, top.N // 2), dtype=np.int64)
    ct = _encrypt_slots(ch.ct(Lq), np.ascontiguousarray(s[:Lq]), z, T, 20)
    out = pr.polyeval(ch, T, coeffs, ct, key)
    Lf = Lq - pr.ceil_log2(len(coeffs) - 1)
    assert out.shape == (B, 2, Lf, top.N)
    assert np.array_equal(_decrypt_slots(ch.ct(Lf), np.ascontiguousarray(s[:Lf]), out, T), pr.poly_mod_t(coeffs, z, T))


def test_noise_budget_at_degree_8(oracle_mod, capsys):
    """the noise left after p of degree 8 (Lq = 4, K = 2, N = 1024, t = 65537, the default 60-bit basis): recorded in DESIGN.md 2.15"""
    logn, Lq, K = 10, 4, 2
    top = oracle_mod.Oracle(logn, Lq + K)
    ch = pr.Chain(oracle_mod, logn, top.moduli, K)
    s = top.keygen_secret(31)
    key = top.keygen_relin_grouped(K, 32, T, s)
    z = np.random.default_rng(2).integers(0, T, (2, 2, top.N // 2), dtype=np.int64)
    ct = _encrypt_slots(ch.ct(Lq), np.ascontiguousarray(s[:Lq]), z, T, 40)
    out = pr.polyeval(ch, T, [1, 2, 3, 4, 5, 6, 7, 8, 9], ct, key)
    o = ch.ct(1)
    bits = _noise_bits(o, np.ascontiguousarray(s[:1]), out, T)
    budget = o.moduli[0].bit_length() - 1 - bits
    with capsys.disabled():
        print("\n[polyeval] d = 8: noise %d bits, q_0 %d bits, budget left %d bits" % (bits, o.moduli[0].bit_length(), budget))
    assert budget > 0


@pytest.mark.parametrize("mutant", ["no_qinv", "g_above", "sum_after", "no_special_rows"])
def test_schedule_mutants_are_caught(oracle_mod, mutant):
    """each deliberate error of the schedule changes the decrypted slots"""
    logn, Lq, K = 10, 4, 2
    top = oracle_mod.Oracle(logn, Lq + K)
    ch = pr.Chain(oracle_mod, logn, top.moduli, K)
    s = top.keygen_secret(51)
    key = top.keygen_relin_grouped(K, 52, T, s)
    coeffs = [3, 1, 4, 1, 5, 9, 2]
    z = np.random.default_rng(5).integers(0, T, (1, 2, top.N // 2), dtype=np.int64)
    ct = _encrypt_slots(ch.ct(Lq), np.ascontiguousarray(s[:Lq]), z, T, 60)
    out = pr.polyeval(ch, T, coeffs, ct, key, mutate=mutant)
    Lf = out.shape[2]
    assert not np.array_equal(_decrypt_slots(ch.ct(Lf), np.ascontiguousarray(s[:Lf]), out, T), pr.poly_mod_t(coeffs, z, T))
