"""The product's seeded bodies (deeppowers_b200/csrc/keys.cuh: the seeded modes of keys_limb_body / keys_half_body, and expand_block)
without a GPU: run by the host emulator (tests/emu/emu_seeded.cpp) in both arithmetic variants and compared bit for bit with the
restatement of DESIGN.md section 2.23 (tests/seeded_ref.py) at N = 4096, 8192 and 16384 (the CTA-pair bodies), on the default basis
and a generic one."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import keys_ref as kr
import seeded_ref as sr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
SEED = bytes(range(50, 82))
T = 65537
ENC, RELIN, GALOIS = 6, 7, 8


def _build(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_seeded_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_seeded.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "keys.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_seeded_create.restype = C.c_void_p
    lib.emu_seeded_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_seeded_destroy.argtypes = [C.c_void_p]
    lib.emu_seeded_run.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_uint, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint,
                                   C.c_void_p, C.c_void_p, _u64p, C.c_size_t]
    lib.emu_seeded_expand.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_uint, _u64p, _u64p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def emu():
    return {v: _build(v) for v in ("gen", "fast")}


def _ctx(lib, log_n, moduli):
    h = lib.emu_seeded_create(log_n, len(moduli), (C.c_uint64 * len(moduli))(*[int(q) for q in moduli]))
    assert h
    return h


@pytest.mark.parametrize("variant,log_n,basis", [("gen", 12, None), ("fast", 12, None), ("gen", 13, "gen_mixed"), ("fast", 13, None),
                                                 ("gen", 14, None), ("fast", 14, None)])
def test_seeded_bodies_match_the_restatement(emu, oracle_mod, variant, log_n, basis):
    """c0 of seeded encryption (item numbers across 2^32), the b rows of a seeded relinearisation key (K = 2) and of Galois keys (K = 0),
    and both expansions"""
    if variant == "fast" and basis:
        pytest.skip("the fast variant takes k 2^32 + 1 moduli only")
    L = 4
    moduli = bases.catalogue(oracle_mod)[basis][:L] if basis else None
    o = oracle_mod.Oracle(log_n, L, moduli)
    lib = emu[variant]
    h = _ctx(lib, log_n, o.moduli)
    try:
        s = kr.secret(o, SEED)
        a_seed = sr.public_seed(SEED)
        n, first = 2, (1 << 32) - 1
        pt = o.fill_uniform(3, n)
        c0 = np.zeros((n, L, o.N), dtype=np.uint64)
        assert lib.emu_seeded_run(h, ENC, SEED, a_seed, 0, T, first, None, 0, s.ctypes.data, pt.ctypes.data, c0.reshape(-1), n) == 0
        want = sr.encrypt_seeded(o, T, s, SEED, first, pt)
        assert np.array_equal(c0, want[:, 0])
        ct = np.zeros((n, 2, L, o.N), dtype=np.uint64)
        assert lib.emu_seeded_expand(h, 0, a_seed, 0, first, None, 0, c0.reshape(-1), ct.reshape(-1), n) == 0
        assert np.array_equal(ct, want)
        K = 2
        nd = kr.digits(o, K)
        b = np.zeros((nd, L, o.N), dtype=np.uint64)
        assert lib.emu_seeded_run(h, RELIN, SEED, a_seed, K, T, 0, None, 0, s.ctypes.data, None, b.reshape(-1), nd) == 0
        rk = sr.relin_key_seeded(o, K, T, s, SEED)
        assert np.array_equal(b, rk[:, 0])
        elts = np.array([o.galois_elt(1), 2 * o.N - 1], dtype=np.uint64)
        gb = np.zeros((2, L, L, o.N), dtype=np.uint64)
        assert lib.emu_seeded_run(h, GALOIS, SEED, a_seed, 0, 0, 0, elts.ctypes.data, 2, s.ctypes.data, None, gb.reshape(-1), 2 * L) == 0
        gk = sr.galois_keys_seeded(o, 0, 0, s, SEED, [int(g) for g in elts])
        assert np.array_equal(gb, gk[:, :, 0])
        keys = np.zeros((2, L, 2, L, o.N), dtype=np.uint64)
        assert lib.emu_seeded_expand(h, 1, a_seed, 0, 0, elts.ctypes.data, 2, gb.reshape(-1), keys.reshape(-1), 2 * L) == 0
        assert np.array_equal(keys, gk)
    finally:
        lib.emu_seeded_destroy(h)
