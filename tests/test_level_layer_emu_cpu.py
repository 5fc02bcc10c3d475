"""The level layer's kernel bodies without a GPU (DESIGN.md sections 2.21 / 4.18): the hoisted multiply-accumulate
(rot_apply_grouped_rows with LV) and the fused Horner step (the grouped program in mode KS_ROTATE with ADD and LV) of
tests/emu/emu_level_layer.cpp, both arithmetic variants, reading a top-level key and its companions through the key-row map, against
the same bodies without LV on the key restricted to the level (tests/polyeval_ref.py:restrict_key) and the level's basis, bit for bit.
Covers K = 1 .. 4, every valid level including ragged last digits, N = 4096 .. 16384, the five bases of tests/bases.py, odd and even
batches and t = 0 / 65537 / 167772161."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import polyeval_ref as pr
from bases import catalogue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_libs = {}
T_BGV = 167772161


def _build(variant):
    """tests/_emu/libdpfhe_emu_level_layer_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_level_layer_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_level_layer.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        tmp = "%s.%d.tmp" % (so, os.getpid())   # built aside and renamed: parallel test workers never load a half-written library
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc]
                              + srcs + ["-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.emu_ll_create.restype = C.c_void_p
    lib.emu_ll_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_ll_destroy.argtypes = [C.c_void_p]
    lib.emu_ll_rot_apply.argtypes = [C.c_void_p, C.c_uint, C.c_int, _u64p, _u64p, _u64p, C.c_uint32, C.c_uint, _u64p, _u64p, C.c_size_t,
                                     C.c_uint64]
    lib.emu_ll_horner.argtypes = [C.c_void_p, C.c_uint, C.c_int, _u64p, _u64p, C.c_uint32, _u64p, C.c_uint, _u64p, _u64p, C.c_size_t, C.c_uint64]
    _libs[variant] = lib
    return lib


def _variants(moduli):
    return ["gen"] + (["fast"] if all((int(q) - 1) % (1 << 32) == 0 for q in moduli) else [])


def _uniform(rng, mods, shape):
    out = np.empty(shape, dtype=np.uint64)
    for i, q in enumerate(mods):
        out[..., i, :] = rng.integers(0, int(q), size=out[..., i, :].shape, dtype=np.uint64)
    return out


class View:
    """the level view {q_0 .. q_{l-1}, p_0 .. p_{K-1}} of a top basis `mods` (Lq + K moduli) in one arithmetic variant"""

    def __init__(self, log_n, mods, K, l, variant):
        self.N, self.K, self.l, self.Lq = 1 << log_n, K, l, len(mods) - K
        self.top = np.array(mods, dtype=np.uint64)
        self.low = np.array(list(mods[:l]) + list(mods[self.Lq:]), dtype=np.uint64)
        self._l = _build(variant)
        arr = (C.c_uint64 * len(self.low))(*[int(m) for m in self.low])
        self._h = self._l.emu_ll_create(log_n, len(self.low), arr)
        assert self._h, "emu_ll_create rejected the parameters"

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_ll_destroy(self._h)

    def restrict(self, key):
        return pr.restrict_key(key, self.Lq, self.K, self.l)

    def rot_apply(self, lv, key, ct, U, galois, t):
        batch = ct.shape[0]
        acc = np.zeros((batch, 2, self.l + self.K, self.N), dtype=np.uint64)
        mods = self.top if lv else self.low
        assert self._l.emu_ll_rot_apply(self._h, self.K, int(lv), ct.reshape(-1), U.reshape(-1), np.ascontiguousarray(key).reshape(-1), int(galois),
                                        len(mods), mods, acc.reshape(-1), batch, int(t)) == 0
        return acc

    def horner(self, lv, key, a, addend, galois, t):
        out = np.zeros(a.shape, dtype=np.uint64)
        mods = self.top if lv else self.low
        assert self._l.emu_ll_horner(self._h, self.K, int(lv), a.reshape(-1), addend.reshape(-1), int(galois), np.ascontiguousarray(key).reshape(-1),
                                     len(mods), mods, out.reshape(-1), a.shape[0], int(t)) == 0
        return out


def _check_level(mods, log_n, K, l, t, seed, batch):
    rng = np.random.default_rng(seed)
    N, Lq = 1 << log_n, len(mods) - K
    dnum, dl = -(-Lq // K), -(-l // K)
    key = _uniform(rng, mods, (dnum, 2, Lq + K, N))
    a = _uniform(rng, mods[:l], (batch, 2, l, N))
    addend = _uniform(rng, mods[:l], (batch, 2, l, N))
    galois = pow(5, 1 + seed % 7, 2 * N)
    for variant in _variants(mods):
        v = View(log_n, mods, K, l, variant)
        low = v.restrict(key)
        U = _uniform(rng, v.low, (batch, dl, l + K, N))
        got = v.rot_apply(True, key[:dl], a, U, galois, t)   # the top-level key's digits the level reads
        assert np.array_equal(got, v.rot_apply(False, low, a, U, galois, t)), variant
        assert got.any()
        got = v.horner(True, key, a, addend, galois, t)
        assert np.array_equal(got, v.horner(False, low, a, addend, galois, t)), variant
        assert got.any()


def _default_mods(oracle_mod, log_n, L):
    return [int(q) for q in oracle_mod.Oracle(log_n, L).moduli]


# (K, Lq): every valid level of each; K = 2, Lq = 7 and K = 3, Lq = 7 have ragged last digits at odd / non-multiple levels
SHAPES = [(1, 3), (2, 4), (2, 7), (3, 7), (4, 5)]


@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_every_level(oracle_mod, log_n, shape):
    K, Lq = SHAPES[shape]
    mods = _default_mods(oracle_mod, log_n, Lq + K)
    levels = range(K, Lq) if log_n == 12 else [K, Lq - 1]   # every level at N = 4096, the ends at the larger degrees
    for l in levels:
        t = (0, 65537, T_BGV)[(l + shape) % 3]
        _check_level(mods, log_n, K, l, t, seed=100 * shape + 10 * log_n + l, batch=3 if log_n == 12 else 1)


@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_other_bases(oracle_mod, basis):
    mods = [int(q) for q in catalogue(oracle_mod)[basis]]
    for K, l in ((1, 2), (2, 3)):
        if len(mods) - K >= l:
            _check_level(mods, 12, K, l, T_BGV, seed=sum(map(ord, basis)) + K, batch=2)
