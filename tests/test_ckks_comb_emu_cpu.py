"""The CKKS combination fused into the final rescale (DESIGN.md sections 2.16, 4.12) without a GPU: the product's kernel bodies
(ckks_comb_tau_body, ckks_comb_limb_body of csrc/eval.cuh), run by the host emulator (tests/emu/emu_ckks_comb.cpp) in both arithmetic
variants, bit for bit against mod_switch_down(lincomb(cuts)) from Python integers and the oracle; and the product's host rounding
and exact reduction of the coefficients against Python integers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import ckks_polyeval_ref as cr
import polyeval_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_ckks_comb_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_ckks_comb.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "eval.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas",
                               "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_ckks_comb.argtypes = [C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_size_t]
    lib.emu_double_mod.argtypes = [C.c_double, C.c_uint64]
    lib.emu_double_mod.restype = C.c_uint64
    lib.emu_ckks_comb_coeff.argtypes = [C.c_double, C.c_double, C.c_double]
    lib.emu_ckks_comb_coeff.restype = C.c_double
    return lib


@pytest.fixture(scope="module")
def emu():
    return {v: _build(v) for v in ("gen", "fast")}


def run_emu(lib, logn, moduli, Lc, cts, coeffs, constant):
    n, B = len(cts), cts[0].shape[0]
    out = np.zeros((B, 2, Lc - 1, 1 << logn), dtype=np.uint64)
    ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in cts])
    levels = (C.c_uint * n)(*[c.shape[2] for c in cts])
    cs = (C.c_double * n)(*[float(c) for c in coeffs])
    mods = (C.c_uint64 * Lc)(*[int(q) for q in moduli[:Lc]])
    assert lib.emu_ckks_comb(logn, Lc, mods, n, ptrs, levels, cs, float(constant), out.ctypes.data, B) == 0
    return out


def reference(oracle_mod, logn, moduli, Lc, cts, coeffs, constant):
    cuts = [np.ascontiguousarray(c[:, :, :Lc]) for c in cts]
    comb = pr.lincomb(moduli[:Lc], cuts, [int(c) for c in coeffs], int(constant))
    B = comb.shape[0]
    return oracle_mod.Oracle(logn, Lc, moduli[:Lc]).mod_switch_down(comb.reshape(2 * B, Lc, -1), 0).reshape(B, 2, Lc - 1, -1)


BIG = [2.0**90, -2.0**200, -1.0, 2.0**53 - 1, -(2.0**63), 0.0, 1.0, 2.0**64 + 2.0**12]


def _case(oracle_mod, logn, moduli, Lc, n_terms, seed, extreme):
    """n_terms ciphertexts at levels Lc .. len(moduli) in turn (batch 2); `extreme`: every input q - 1 and every coefficient -1
    (w = q - 1, the largest lazy sums)"""
    top = len(moduli)
    rng = np.random.default_rng(seed)
    cts = []
    for i in range(n_terms):
        lv = Lc + i % (top - Lc + 1)
        o = oracle_mod.Oracle(logn, lv, moduli[:lv])
        ct = o.fill_uniform(seed * 100 + i, 4).reshape(2, 2, lv, o.N)
        if extreme:
            for l, q in enumerate(moduli[:lv]):
                ct[:, :, l] = q - 1
        cts.append(ct)
    if extreme:
        return cts, [-1.0] * n_terms, -1.0
    coeffs = [BIG[i] if i < len(BIG) else float(np.round(rng.normal() * 2.0**45)) for i in range(n_terms)]
    return cts, coeffs, 2.0**90 + 2.0**40


@pytest.mark.parametrize("logn", [12, 13, 14])
@pytest.mark.parametrize("variant,basis", [("fast", None), ("gen", None), ("gen", "gen_mixed"), ("fast", "ckks")])
@pytest.mark.parametrize("n_terms", [1, 8, 9, 64])
def test_emulated_fused_comb_equals_rescaled_lincomb(oracle_mod, emu, logn, variant, basis, n_terms):
    if n_terms == 64 and logn != 12:
        pytest.skip("64 terms: N = 4096 (the Python-integer reference is slow); 8 and 9 cover both parameter blocks at every N")
    if basis == "ckks":
        moduli = cr.ckks_chain(oracle_mod, 4, 2)[:4]
    elif basis:
        moduli = bases.catalogue(oracle_mod)[basis][:4]
    else:
        moduli = oracle_mod.Oracle(logn, 4).moduli
    Lc = 3
    for extreme in (False, True):
        cts, coeffs, constant = _case(oracle_mod, logn, moduli, Lc, n_terms, logn + n_terms, extreme)
        got = run_emu(emu[variant], logn, moduli, Lc, cts, coeffs, constant)
        assert np.array_equal(got, reference(oracle_mod, logn, moduli, Lc, cts, coeffs, constant)), extreme


def test_emulated_fused_comb_at_two_limbs(oracle_mod, emu):
    """Lc = 2, the smallest combination: one limb kept"""
    logn = 12
    moduli = cr.ckks_chain(oracle_mod, 5, 2)[:5]
    cts, coeffs, constant = _case(oracle_mod, logn, moduli, 2, 9, 7, False)
    for v in ("gen", "fast"):
        assert np.array_equal(run_emu(emu[v], logn, moduli, 2, cts, coeffs, constant), reference(oracle_mod, logn, moduli, 2, cts, coeffs, constant))


EXACT = [0.0, -0.0, 1.0, -1.0, 2.0**53 - 1, -(2.0**53 - 1), 2.0**53 + 2, 2.0**63, -(2.0**63), 2.0**64, 2.0**90, -(2.0**90), 2.0**200,
         -(2.0**200), 3.0 * 2.0**1000, 123456789.0 * 2.0**70]


def test_exact_reduction_against_python_integers(oracle_mod, emu):
    qs = cr.ckks_chain(oracle_mod, 4, 2) + bases.catalogue(oracle_mod)["gen_mixed"]
    for v in ("gen", "fast"):
        for q in qs:
            for c in EXACT:
                assert emu[v].emu_double_mod(c, q) == cr.residue(c, q), (c, q)


def test_rounding_half_to_even_against_python(emu):
    """ties k + 1/2 round to the even neighbour, as Python's round() (which the restatement uses)"""
    lib = emu["gen"]
    for k in (0, 1, 2, 3, -1, -2, 2**51, 2**52 - 1, -(2**52 - 1)):
        x = k + 0.5
        assert lib.emu_ckks_comb_coeff(x, 1.0, 1.0) == float(round(x)), k
        assert lib.emu_ckks_comb_coeff(x, 2.0, 2.0) == float(round((x * 2.0) / 2.0)), k
    rng = np.random.default_rng(1)
    for _ in range(2000):
        a, m, s = rng.normal(), float(2.0**90 * (1 + rng.random())), float(2.0**45 * (1 + rng.random()))
        assert lib.emu_ckks_comb_coeff(a, m, s) == float(round((a * m) / s))
