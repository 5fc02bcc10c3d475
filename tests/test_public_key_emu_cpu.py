"""The product's public-key bodies (deeppowers_b200/csrc/keys.cuh: the public-key mode of keys_limb_body / keys_half_body, and
pub_enc_body) without a GPU: run by the host emulator (tests/emu/emu_public_keys.cpp) in both arithmetic variants and compared bit for
bit with the restatement of DESIGN.md section 2.14 (tests/public_key_ref.py) at N = 4096, 8192 and 16384 (both CTAs of the pair), on
the default basis and a generic one, for t = 65537 and t = 0."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import keys_ref as kr
import public_key_ref as pkr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
OWNER = bytes(range(50, 82))
ENCRYPTOR = bytes(range(150, 182))


def _build(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_public_keys_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_public_keys.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "keys.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_pk_create.restype = C.c_void_p
    lib.emu_pk_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_pk_destroy.argtypes = [C.c_void_p]
    lib.emu_pk_public_keygen.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, _u64p, _u64p]
    lib.emu_pk_encrypt_public.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, _u64p, _u64p, _u64p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def emu_libs():
    return {v: _build(v) for v in ("gen", "fast")}


# (log N, limbs, basis, variant): both variants on the default basis, the generic variant on a generic basis, at every ring degree
CASES = [(logn, L, basis, v) for logn, L in ((12, 4), (13, 3), (14, 2)) for basis, v in ((None, "fast"), (None, "gen"), ("gen_mixed", "gen"))]


@pytest.mark.parametrize("logn,L,basis,variant", CASES)
def test_emulated_public_key_bodies_equal_the_restatement(oracle_mod, emu_libs, logn, L, basis, variant):
    lib = emu_libs[variant]
    moduli = bases.catalogue(oracle_mod)[basis][:L] if basis else None
    o = oracle_mod.Oracle(logn, L, moduli)
    h = lib.emu_pk_create(logn, L, (C.c_uint64 * L)(*[int(q) for q in o.moduli]))
    assert h
    try:
        s = kr.secret(o, OWNER)
        pt = o.fill_uniform(logn, 2)
        for t in (65537, 0):
            pk = np.zeros((2, L, o.N), dtype=np.uint64)
            assert lib.emu_pk_public_keygen(h, OWNER, t, s.reshape(-1), pk.reshape(-1)) == 0
            assert np.array_equal(pk, pkr.public_keygen(o, t, s, OWNER)), t
            ct = np.zeros((2, 2, L, o.N), dtype=np.uint64)
            item0 = (1 << 32) + 7
            assert lib.emu_pk_encrypt_public(h, ENCRYPTOR, t, item0, pk.reshape(-1), pt.reshape(-1), ct.reshape(-1), 2) == 0
            assert np.array_equal(ct, pkr.encrypt_public(o, t, pk, ENCRYPTOR, item0, pt)), t
    finally:
        lib.emu_pk_destroy(h)
