"""The fused key switch at N <= 8192 (ks_fused_kernel, one 4096-point block per CTA, DESIGN.md §4.4) on the CPU: its bodies run
through a host emulator (tests/emu/emu_fused_blk.cpp) with the CTA pair's barriers as phase order, and must give the oracle's
ct x ct multiply + relinearise, bare key switch and rotation bit for bit, for L = 1 … 6 limbs at N = 4096 and 8192, in both
arithmetic variants, on the default basis and on every generic basis of tests/bases.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from bases import NAMES, N_LIMBS, catalogue, selects

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_libs = {}
KS_MUL_RELIN, KS_PLAIN, KS_ROTATE = 0, 1, 2


def _build(variant):
    """tests/_emu/libdpfhe_emu_fused_blk_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_fused_blk_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_fused_blk.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc] + srcs
                              + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_fb_create.restype = C.c_void_p
    lib.emu_fb_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_fb_destroy.argtypes = [C.c_void_p]
    lib.emu_fb_ks.argtypes = [C.c_void_p, C.c_int, _u64p, _u64p, _u64p, _u64p, C.c_size_t, C.c_uint32, C.c_int]
    _libs[variant] = lib
    return lib


class EmuFusedBlk:
    def __init__(self, log_n, L, moduli, variant):
        self._l = _build(variant)
        arr = (C.c_uint64 * L)(*[int(m) for m in moduli])
        self._h = self._l.emu_fb_create(log_n, L, arr)
        assert self._h, "emu_fb_create rejected the parameters"
        self.lift_reduce = selects(moduli)[1]

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_fb_destroy(self._h)
            self._h = None

    def ks(self, mode, a, b, key, galois=0, lift_reduce=None):
        """mode KS_MUL_RELIN: a x b relinearised; KS_PLAIN: key switch of the digits a [batch][L][N]; KS_ROTATE: rotation of a"""
        a = np.ascontiguousarray(a, dtype=np.uint64)
        b = np.ascontiguousarray(a if b is None else b, dtype=np.uint64)
        batch = a.shape[0]
        out = np.zeros((batch, 2) + a.shape[-2:], dtype=np.uint64)
        lr = self.lift_reduce if lift_reduce is None else lift_reduce
        assert self._l.emu_fb_ks(self._h, mode, a.reshape(-1), b.reshape(-1), np.ascontiguousarray(key, dtype=np.uint64).reshape(-1),
                                 out.reshape(-1), batch, int(galois), int(lr)) == 0
        return out


def _variants(moduli):
    return ("fast", "gen") if all(int(q) & 0xFFFFFFFF == 1 for q in moduli) else ("gen",)


def _check_all_modes(o, log_n, L, moduli, seed, lift_reduce=None):
    """ct x ct, the bare key switch and two rotations (one of them the conjugation) against the oracle; rows of q - 1 and of zero
    next to uniform ones"""
    batch = 2
    q = np.array(o.moduli, dtype=np.uint64)
    a = o.fill_uniform(seed, 2 * batch).reshape(batch, 2, L, o.N)
    b = o.fill_uniform(seed + 1, 2 * batch).reshape(batch, 2, L, o.N)
    a[0, 1] = (q - 1)[:, None]
    b[1, 0] = (q - 1)[:, None]
    b[1, 1, L - 1] = 0
    key = o.fill_uniform(seed + 2, 2 * L).reshape(L, 2, L, o.N)
    d = o.fill_uniform(seed + 3, batch).reshape(batch, L, o.N)
    d[0, 0] = q[0] - 1
    want = {"mul": o.ct_mul_relin(a, b, key), "ks": np.stack([np.stack(o.keyswitch(d[k], key)) for k in range(batch)]),
            "rot": o.rotate(a, o.galois_elt(5), key), "conj": o.rotate(a, 2 * o.N - 1, key)}
    for variant in _variants(moduli):
        e = EmuFusedBlk(log_n, L, moduli, variant)
        got = {"mul": e.ks(KS_MUL_RELIN, a, b, key, lift_reduce=lift_reduce), "ks": e.ks(KS_PLAIN, d, None, key, lift_reduce=lift_reduce),
               "rot": e.ks(KS_ROTATE, a, None, key, o.galois_elt(5), lift_reduce),
               "conj": e.ks(KS_ROTATE, a, None, key, 2 * o.N - 1, lift_reduce)}
        for k in want:
            assert np.array_equal(got[k], want[k]), (variant, k)


@pytest.mark.parametrize("log_n", [12, 13])
@pytest.mark.parametrize("L", range(1, N_LIMBS + 1))
def test_default_basis(oracle_mod, log_n, L):
    o = oracle_mod.Oracle(log_n, L)
    _check_all_modes(o, log_n, L, o.moduli, 10 + L)


@pytest.mark.parametrize("log_n", [12, 13])
def test_default_basis_with_lift_reduction(oracle_mod, log_n):
    """the word reduction of the digit lift, which the default basis may skip, gives the same bits"""
    o = oracle_mod.Oracle(log_n, 4)
    _check_all_modes(o, log_n, 4, o.moduli, 30, lift_reduce=True)


@pytest.mark.parametrize("log_n", [12, 13])
@pytest.mark.parametrize("L", range(1, N_LIMBS + 1))
@pytest.mark.parametrize("name", NAMES)
def test_generic_bases(oracle_mod, name, log_n, L):
    mods = catalogue(oracle_mod)[name][:L]
    o = oracle_mod.Oracle(log_n, L, mods)
    _check_all_modes(o, log_n, L, mods, 50 + L)
