"""shoup_w_from_companion (modarith.cuh): a Shoup factor w < q rebuilt from its companion ws = floor(w * 2^64 / q) alone.

The fused ct x ct kernel's multiply-accumulate reads only the companions of the key row and rebuilds each key word from its own
(DESIGN.md §4.4), so the rebuild must be exact for every w < q of every modulus the fast kernels accept: the lazy values, and with
them the results, are bit-identical only then.  The host build (both arithmetic variants) is compiled with g++ and checked
against Python integers; the fast device form (two 32 x 32 products and a carry chain, inline PTX) is restated here word by word
with Python integers on the same cases, since its decomposition is what the carry chain relies on."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import arith_cases as ac
import bases

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deeppowers_b200", "csrc")
M64, M32 = 1 << 64, 1 << 32
N_RANDOM = 4000

SRC = r"""
#include "modarith.cuh"
extern "C" void recover(const uint64_t *ws, uint64_t *out, size_t n, uint64_t q, uint32_t nqh) {
    dpfhe::LimbParams p = {};
    p.q = q;
    p.nqh = nqh;
    for (size_t k = 0; k < n; ++k) out[k] = dpfhe::DPFHE_VNS::shoup_w_from_companion(ws[k], p);
}
"""


@pytest.fixture(scope="module")
def recover(tmp_path_factory):
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("companion")
    src = d / "companion.cpp"
    src.write_text(SRC)
    libs = {}
    for v, fast in (("gen", 0), ("fast", 1)):
        so = str(d / ("libcompanion_%s.so" % v))
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % fast, "-I", CSRC, str(src), "-o", so])
        lib = ctypes.CDLL(so)
        lib.recover.restype = None
        lib.recover.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint64, ctypes.c_uint32]
        libs[v] = lib

    def run(v, q, ws):
        a = np.array(ws, dtype=np.uint64)
        out = np.zeros_like(a)
        nqh = (-(q >> 32)) % M32 if bases.is_fast(q) else 0
        libs[v].recover(a.ctypes.data, out.ctypes.data, len(a), q, nqh)
        return [int(x) for x in out]
    return run


def companion(w, q):
    return (w << 64) // q


def fast_form(ws, q):
    """the device's fast form: ws q + q - 1 = wl + 2^32 (wh + qh + wl qh) + 2^64 wh qh, hi64 from the carry of the middle sum"""
    qh, wl, wh = q >> 32, ws % M32, ws >> 32
    s = wl * qh                                  # mul.wide.u32 S, wl, qh
    sh = (s >> 32) + (((s % M32) + wh + qh) >> 32)   # add.cc / addc twice: the carries out of the low word
    assert sh < M32
    return (wh * qh + sh) % M64                  # mul.wide.u32 B, wh, qh; add.cc / addc


def w_values(q, seed):
    """corners and seeded uniform values.  ws q = w 2^64 - r with r = w 2^64 mod q, so lo64(ws q) is 0 only for w = 0 (q is odd),
    is 2^64 - 1 for r = 1 (w = 2^-64 mod q), and ws q + q - 1 is exactly w 2^64 for r = q - 1 (w = -2^-64 mod q)"""
    inv = pow(M64, -1, q)
    ws = [0, 1, 2, q - 2, q - 1, q // 2, q // 2 + 1, inv, q - inv]
    rng = random.Random(seed)
    ws += [rng.randrange(q) for _ in range(N_RANDOM)]
    return ws


def moduli():
    """(id, modulus, fast): the default basis, the k 2^32 + 1 bases without its shortcuts and a generic basis"""
    out = [("default%d" % k, q, True) for k, q in enumerate(ac.default_basis(4))]
    cat = bases.derive(ac._Primality)
    for name in ("fast_mixed", "fast_narrow", "gen_mixed"):
        out += [("%s%d" % (name, k), q, bases.is_fast(q)) for k, q in enumerate(cat[name])]
    out.append(("smallest_generic", bases.SMALLEST_GENERIC, False))
    out.append(("largest_generic", bases.LARGEST_GENERIC, False))
    return out


MODULI = moduli()


@pytest.mark.parametrize("mid,q,fast", MODULI, ids=[m[0] for m in MODULI])
def test_rebuild_exact(recover, mid, q, fast):
    ws_w = w_values(q, ac.seed_of("companion", mid))
    ws = [companion(w, q) for w in ws_w]
    for v in ("gen", "fast") if fast else ("gen",):
        got = recover(v, q, ws)
        bad = [(w, s, g) for w, s, g in zip(ws_w, ws, got) if g != w]
        assert not bad, (v, mid, bad[:5])
    if fast:
        bad = [(w, s) for w, s in zip(ws_w, ws) if fast_form(s, q) != w]
        assert not bad, ("fast form", mid, bad[:5])


def test_cases_reach_the_corners():
    """every modulus's cases reach lo64(ws q) = 0 and 2^64 - 1 and ws q + q - 1 = w 2^64, and hi64(ws q) alone (the rebuild
    without its rounding term) is wrong on every w but 0"""
    for mid, q, _ in MODULI:
        ws_w = w_values(q, ac.seed_of("companion", mid))
        lows = {(companion(w, q) * q) % M64 for w in ws_w}
        assert 0 in lows and M64 - 1 in lows, mid
        assert any(companion(w, q) * q + q - 1 == w << 64 for w in ws_w if w), mid
        assert all(((companion(w, q) * q) >> 64 == w) == (w == 0) for w in ws_w), mid
