"""The fused Horner addition of the grouped key switch (ks_grouped_kernel<..., ADD>, DESIGN.md §4.4b′) on the CPU: the kernel bodies run
through a host emulator (tests/emu/emu_grouped_add.cpp) and must give o.poly_add(o.rotate_grouped(...), addend) bit for bit, for
K = 1 … 4 special primes at N = 4096, 8192 and 16384 (the half-limb path), in both arithmetic variants, with addends of q − 1 in every
limb."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bases import catalogue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_libs = {}


def _build(variant):
    """tests/_emu/libdpfhe_emu_grouped_add_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_grouped_add_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_grouped_add.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc] + srcs
                              + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_ga_create.restype = C.c_void_p
    lib.emu_ga_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_ga_destroy.argtypes = [C.c_void_p]
    lib.emu_ga_rotate.argtypes = [C.c_void_p, C.c_uint, _u64p, C.c_void_p, _u64p, _u64p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_uint]
    _libs[variant] = lib
    return lib


class EmuGroupedAdd:
    def __init__(self, log_n, L, moduli, variant):
        self._l = _build(variant)
        arr = (C.c_uint64 * L)(*[int(m) for m in moduli])
        self._h = self._l.emu_ga_create(log_n, L, arr)
        assert self._h, "emu_ga_create rejected the parameters"
        self.L = L

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_ga_destroy(self._h)
            self._h = None

    def rotate(self, K, ct, key, galois, t_plain, addend=None, G=None):
        """rotate_grouped(ct) (+ addend through the fused form); ct, addend [batch][2][L-K][N]"""
        ct = np.ascontiguousarray(ct, dtype=np.uint64)
        add_ptr = None
        if addend is not None:
            addend = np.ascontiguousarray(addend, dtype=np.uint64)
            add_ptr = C.c_void_p(addend.ctypes.data)
        out = np.zeros_like(ct)
        assert self._l.emu_ga_rotate(self._h, int(K), ct.reshape(-1), add_ptr, np.ascontiguousarray(key, dtype=np.uint64).reshape(-1), out.reshape(-1),
                                     ct.shape[0], int(galois), int(t_plain), G or 2 * self.L) == 0
        return out


def _variants(moduli):
    return ("fast", "gen") if all(int(q) & 0xFFFFFFFF == 1 for q in moduli) else ("gen",)


def _inputs(o, oq, K, batch, seed):
    """ciphertexts and addends under the first L - K moduli (one addend ciphertext of q - 1 everywhere, one with a zero row) and a
    uniform grouped key"""
    Lq = o.L - K
    ct = oq.fill_uniform(seed, 2 * batch).reshape(batch, 2, Lq, o.N)
    add = oq.fill_uniform(seed + 1, 2 * batch).reshape(batch, 2, Lq, o.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    add[0] = (q - 1)[None, :, None]
    ct[-1, 0] = (q - 1)[:, None]
    add[-1, 1, 0] = 0
    dnum = o.grouped_digits(K)
    key = o.fill_uniform(seed + 2, 2 * dnum).reshape(dnum, 2, o.L, o.N)
    return ct, add, key


# (K, Lq): digits of K limbs, the last one ragged where K does not divide Lq
SHAPES = [(1, 3), (2, 4), (2, 5), (3, 4), (4, 4)]


@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("K,Lq", SHAPES)
def test_fused_add_is_rotate_then_add(oracle_mod, log_n, K, Lq):
    L = Lq + K
    o = oracle_mod.Oracle(log_n, L)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    batch = 3
    ct, add, key = _inputs(o, oq, K, batch, 40 + K)
    g = o.galois_elt(5)
    for t in (0, 65537):
        want = oq.poly_add(o.rotate_grouped(K, ct, g, key, t), add)
        for variant in _variants(o.moduli):
            e = EmuGroupedAdd(log_n, L, o.moduli, variant)
            # G = one group: every ciphertext a round of its own, so the accumulators' round parities alternate
            assert np.array_equal(e.rotate(K, ct, key, g, t, add, G=L), want), (variant, t)


def test_fused_add_generic_basis(oracle_mod):
    """gen_mixed: a 34-bit ciphertext modulus next to 59-bit ones, special primes of 55 and 45 bits"""
    mods = catalogue(oracle_mod)["gen_mixed"]
    K, L = 2, len(mods)
    o = oracle_mod.Oracle(12, L, mods)
    oq = oracle_mod.Oracle(12, L - K, mods[:L - K])
    ct, add, key = _inputs(o, oq, K, 2, 90)
    g = 2 * o.N - 1   # conjugation
    e = EmuGroupedAdd(12, L, mods, "gen")
    for t in (0, 65537):
        assert np.array_equal(e.rotate(K, ct, key, g, t, add), oq.poly_add(o.rotate_grouped(K, ct, g, key, t), add)), t


def test_addend_of_zero_is_the_rotation(oracle_mod, make_emu):
    """with a zero addend the fused form is the plain grouped rotation: of this emulator, of the suite's emulator of ks_grouped_kernel
    and of the oracle, bit for bit"""
    K, Lq = 2, 4
    o = oracle_mod.Oracle(13, Lq + K)
    oq = oracle_mod.Oracle(13, Lq, o.moduli[:Lq])
    ct, _, key = _inputs(o, oq, K, 2, 70)
    g = o.galois_elt(-7)
    e = EmuGroupedAdd(13, Lq + K, o.moduli, "fast")
    got = e.rotate(K, ct, key, g, 65537, np.zeros_like(ct))
    assert np.array_equal(got, e.rotate(K, ct, key, g, 65537))
    assert np.array_equal(got, make_emu(13, Lq + K).ks_grouped(K, 2, ct, None, key, 2, galois=g, t_plain=65537))
    assert np.array_equal(got, o.rotate_grouped(K, ct, g, key, 65537))
