"""The product's key generation, encryption and decryption bodies (deeppowers_b200/csrc/keys.cuh) without a GPU: run by the host
emulator (tests/emu/emu_keys.cpp) in both arithmetic variants and compared bit for bit with the restatement of DESIGN.md section
2.14 (tests/keys_ref.py) at N = 4096, 8192 and 16384 (the CTA-pair bodies), on the default basis and a generic one."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import keys_ref as kr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
SEED = bytes(range(50, 82))
T_BGV = 65537


def _build(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_keys_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_keys.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "keys.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_keys_create.restype = C.c_void_p
    lib.emu_keys_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_keys_destroy.argtypes = [C.c_void_p]
    lib.emu_keys_run.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint,
                                 C.c_void_p, C.c_void_p, _u64p, C.c_size_t]
    lib.emu_keys_decrypt.argtypes = [C.c_void_p, _u64p, _u64p, C.c_uint, _u64p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def emu_keys():
    return {v: _build(v) for v in ("gen", "fast")}


class EmuKeys:
    SECRET, ENC, RELIN, GALOIS = 0, 1, 2, 3

    def __init__(self, lib, log_n, moduli):
        self._l, self.N, self.L = lib, 1 << log_n, len(moduli)
        self._h = lib.emu_keys_create(log_n, self.L, (C.c_uint64 * self.L)(*[int(q) for q in moduli]))
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_keys_destroy(self._h)

    def _run(self, mode, shape, n_items, K=0, t=0, item0=0, elts=(), s=None, pt=None):
        out = np.zeros(shape, dtype=np.uint64)
        g = np.ascontiguousarray(elts, dtype=np.uint64)
        s = None if s is None else np.ascontiguousarray(s, dtype=np.uint64)
        pt = None if pt is None else np.ascontiguousarray(pt, dtype=np.uint64)
        rc = self._l.emu_keys_run(self._h, mode, SEED, K, t, item0, g.ctypes.data if len(g) else None, len(g),
                                  None if s is None else s.ctypes.data, None if pt is None else pt.ctypes.data, out.reshape(-1), n_items)
        assert rc == 0
        return out

    def secret(self):
        return self._run(self.SECRET, (self.L, self.N), 1)

    def encrypt(self, t, s, item0, pt):
        n = pt.shape[0]
        return self._run(self.ENC, (n, 2, self.L, self.N), n, t=t, item0=item0, s=s, pt=pt)

    def relin_key(self, K, t, s, nd):
        return self._run(self.RELIN, (nd, 2, self.L, self.N), nd, K=K, t=t, s=s)

    def galois_keys(self, K, t, s, nd, elts):
        return self._run(self.GALOIS, (len(elts), nd, 2, self.L, self.N), len(elts) * nd, K=K, t=t, elts=elts, s=s)

    def decrypt(self, s, ct):
        ct = np.ascontiguousarray(ct, dtype=np.uint64)
        out = np.empty((ct.shape[0], self.L, self.N), dtype=np.uint64)
        assert self._l.emu_keys_decrypt(self._h, ct.reshape(-1), np.ascontiguousarray(s).reshape(-1), ct.shape[1], out.reshape(-1), ct.shape[0]) == 0
        return out


# (log N, limbs, basis, variant): both variants on the default basis, the generic variant on a generic basis, at every ring degree
CASES = [(logn, L, basis, v) for logn, L in ((12, 4), (13, 4), (14, 3)) for basis, v in ((None, "fast"), (None, "gen"), ("gen_mixed", "gen"))]


@pytest.mark.parametrize("logn,L,basis,variant", CASES)
def test_emulated_bodies_equal_the_restatement(oracle_mod, emu_keys, logn, L, basis, variant):
    moduli = bases.catalogue(oracle_mod)[basis][:L] if basis else None
    o = oracle_mod.Oracle(logn, L, moduli)
    emu = EmuKeys(emu_keys[variant], logn, o.moduli)
    s = emu.secret()
    assert np.array_equal(s, kr.secret(o, SEED))
    pt = o.fill_uniform(logn, 2)
    for t in (T_BGV, 0):
        assert np.array_equal(emu.encrypt(t, s, 77, pt), kr.encrypt(o, t, s, SEED, 77, pt)), t
    for K in ((0, 1) if L < 4 else (0, 1, 2)):
        nd = kr.digits(o, K)
        assert np.array_equal(emu.relin_key(K, T_BGV, s, nd), kr.relin_key(o, K, T_BGV, s, SEED)), K
    elts = [o.galois_elt(3), 2 * o.N - 1]
    K = 1
    assert np.array_equal(emu.galois_keys(K, 0, s, kr.digits(o, K), elts), kr.galois_keys(o, K, 0, s, SEED, elts))
    for n_comp in (2, 3):
        ct = o.fill_uniform(5 + n_comp, 2 * n_comp).reshape(2, n_comp, L, o.N)
        assert np.array_equal(emu.decrypt(s, ct), kr.decrypt(o, s, ct))


@pytest.mark.parametrize("variant", ["gen", "fast"])
def test_emulated_per_limb_galois_keys_and_ragged_digits(oracle_mod, emu_keys, variant):
    """per-limb-digit Galois keys for several elements, and grouped keys with a ragged last digit (K = 3 over 5 ciphertext limbs)"""
    o = oracle_mod.Oracle(12, 8)
    emu = EmuKeys(emu_keys[variant], 12, o.moduli)
    s = emu.secret()
    elts = [o.galois_elt(1), o.galois_elt(-7), 2 * o.N - 1]
    assert np.array_equal(emu.galois_keys(0, T_BGV, s, 8, elts), kr.galois_keys(o, 0, T_BGV, s, SEED, elts))
    assert np.array_equal(emu.relin_key(3, T_BGV, s, 2), kr.relin_key(o, 3, T_BGV, s, SEED))
