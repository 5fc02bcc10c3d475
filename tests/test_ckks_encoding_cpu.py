"""CKKS slot encoding (DESIGN.md section 2.12) without a GPU: the C restatement (tests/ckks_ref.c) against exact arithmetic and
the O(N^2) definition, and the product's kernel bodies, run by the host emulator (tests/emu/emu_ckks.cpp), against the
restatement bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import ckks_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")


def _build_emu_ckks(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_ckks_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_ckks.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_ckks_create.restype = C.c_void_p
    lib.emu_ckks_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_ckks_destroy.argtypes = [C.c_void_p]
    lib.emu_ckks_twiddles.argtypes = [C.c_void_p, _f64p]
    lib.emu_ckks_encode.argtypes = [C.c_void_p, _f64p, _u64p, C.c_size_t, C.c_double]
    lib.emu_ckks_decode.argtypes = [C.c_void_p, _u64p, _f64p, C.c_size_t, C.c_double]
    return lib


class EmuCkks:
    def __init__(self, lib, log_n, moduli):
        self._l, self.N, self.L = lib, 1 << log_n, len(moduli)
        self._h = lib.emu_ckks_create(log_n, self.L, (C.c_uint64 * self.L)(*[int(q) for q in moduli]))
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_ckks_destroy(self._h)

    def twiddles(self):
        out = np.empty(2 * self.N)
        self._l.emu_ckks_twiddles(self._h, out)
        return out

    def encode(self, z, scale):
        z = np.ascontiguousarray(z, dtype=np.complex128).reshape(-1, self.N // 2)
        pt = np.empty((z.shape[0], self.L, self.N), dtype=np.uint64)
        assert self._l.emu_ckks_encode(self._h, z.view(np.float64).reshape(-1), pt.reshape(-1), z.shape[0], scale) == 0
        return pt

    def decode(self, pt, scale):
        pt = np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, self.L, self.N)
        z = np.empty((pt.shape[0], self.N // 2), dtype=np.complex128)
        assert self._l.emu_ckks_decode(self._h, pt.reshape(-1), z.view(np.float64).reshape(-1), pt.shape[0], scale) == 0
        return z


@pytest.fixture(scope="module")
def emu_ckks():
    return {v: _build_emu_ckks(v) for v in ("gen", "fast")}


def _slot_exponents(n):
    return np.array([pow(5, j, 2 * n) for j in range(n // 2)], dtype=np.int64)


def _rand_slots(rng, shape):
    return rng.uniform(-1, 1, shape) + 1j * rng.uniform(-1, 1, shape)


def _to_pt(o, coeffs):
    """signed Python-integer coefficients -> [L][N] evaluation form"""
    res = np.array([[c % q for c in coeffs] for q in o.moduli], dtype=np.uint64)
    return o.ntt_fwd(res[None])[0]


# ---- 1. twiddles
@pytest.mark.parametrize("logn", [12, 13, 14])
def test_twiddles_restatement_equals_product(oracle_mod, emu_ckks, logn):
    n = 1 << logn
    ref = ckks_ref.twiddles(logn)
    got = EmuCkks(emu_ckks["fast"], logn, oracle_mod.Oracle(logn, 1).moduli).twiddles()
    assert np.array_equal(ref.view(np.uint64), got.view(np.uint64))


def test_twiddles_correctly_rounded():
    mpmath = pytest.importorskip("mpmath")
    logn = 14
    n = 1 << logn
    ref = ckks_ref.twiddles(logn)
    mpmath.mp.prec = 160
    want = np.empty(2 * n)
    for k in range(n):
        x = mpmath.mpf(k) / n
        want[2 * k], want[2 * k + 1] = float(mpmath.cospi(x)), float(mpmath.sinpi(x))
    assert np.array_equal(ref.view(np.uint64), want.view(np.uint64))


# ---- 2. encode accuracy against the definition
def _definition_coeffs(z, n, scale):
    """scale * m_k for every k from m_k = (2/N) Re sum_j z_j zeta_j^-k, in long double"""
    e = _slot_exponents(n)
    ang = np.pi * np.arange(2 * n, dtype=np.longdouble) / n
    cos_t, sin_t = np.cos(ang), np.sin(ang)
    zr, zi = z.real.astype(np.longdouble), z.imag.astype(np.longdouble)
    out = np.empty(n, dtype=np.longdouble)
    for k in range(n):
        idx = (-e * k) % (2 * n)                 # zeta_j^-k = exp(i pi (-e_j k) / N)
        out[k] = (zr * cos_t[idx] - zi * sin_t[idx]).sum()
    return out * (np.longdouble(2) / n) * np.longdouble(scale)


def test_encode_matches_definition(oracle_mod):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 3)
    z = _rand_slots(np.random.default_rng(3), n // 2)
    for scale in (2.0**40, 2.0**70):
        _, cf = ckks_ref.encode(o, z, scale, with_coeffs=True)
        exact = _definition_coeffs(z, n, scale)
        err = np.abs(cf[0].astype(np.longdouble) - exact)
        bound = logn * 2.0**-53 * scale * np.abs(z).max()   # DESIGN.md 2.12: pre-rounding error
        if scale == 2.0**40:
            assert err.max() <= 1 and err.max() <= 0.5 + bound
        else:   # the coefficients are far beyond 2^53, so err is the pre-rounding error itself (plus < 1 of rounding)
            assert np.abs(exact).max() > 2.0**60
            assert err.max() <= bound + 1


@pytest.mark.parametrize("c", [0.75, -1.25 + 0.0j, 3.0])
def test_encode_constant_slots(oracle_mod, c):
    logn, n, scale = 12, 4096, 2.0**40
    o = oracle_mod.Oracle(logn, 2)
    _, cf = ckks_ref.encode(o, np.full(n // 2, c, dtype=np.complex128), scale, with_coeffs=True)
    want = np.zeros(n)
    want[0] = np.rint(scale * np.real(c))
    assert np.array_equal(cf[0], want)


# ---- 3. exact reduction
def test_exact_reduction_large_scale_and_2_63(oracle_mod):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 5)
    rng = np.random.default_rng(5)
    z = _rand_slots(rng, (2, n // 2))
    z[1, :] = 2.0**23 + 1j * 0.0     # coefficient 0 at 2^63, the others near zero
    z[1, 7] = -(2.0**23)              # ... and straddling -2^63 / 2^63 through the others
    for scale in (2.0**80, 2.0**40):
        pt, cf = ckks_ref.encode(o, z, scale, with_coeffs=True)
        assert np.abs(cf).max() >= 2.0**62
        for v in range(2):
            want = _to_pt(o, [int(x) for x in cf[v]])
            assert np.array_equal(pt[v], want)


# ---- 4. decode accuracy against exact CRT arithmetic
def test_decode_exact_crt(oracle_mod):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 4)
    Q = 1
    for q in o.moduli:
        Q *= q
    rng = np.random.default_rng(7)
    scale = 2.0**50
    coeffs = [int(v) for v in rng.integers(-2**62, 2**62, n)]
    coeffs[0], coeffs[1], coeffs[2], coeffs[3] = (Q - 1) // 2, -((Q - 1) // 2), 3 * 2**70 + 5, -(2**65) - 1
    got = ckks_ref.decode(o, _to_pt(o, coeffs)[None], scale)[0]
    e = _slot_exponents(n)
    c = np.array([float(v / int(scale)) for v in coeffs], dtype=np.longdouble)
    ang = np.pi * np.arange(2 * n, dtype=np.longdouble) / n
    cos_t, sin_t = np.cos(ang), np.sin(ang)
    bound = 2.0**-53 * 2 * logn * np.abs(c).sum()
    for j in range(0, n // 2, 37):
        idx = (e[j] * np.arange(n)) % (2 * n)
        want = complex((c * cos_t[idx]).sum(), (c * sin_t[idx]).sum())
        assert abs(got[j] - want) <= bound


@pytest.mark.parametrize("X", ["half", "-half", "big", "-big"])
def test_decode_constant_centring(oracle_mod, X):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 5)
    Q = 1
    for q in o.moduli:
        Q *= q
    x = {"half": (Q - 1) // 2, "-half": -((Q - 1) // 2), "big": 2**64 + 12345, "-big": -(2**64) - 12345}[X]
    coeffs = [x] + [0] * (n - 1)
    scale = 2.0**40
    got = ckks_ref.decode(o, _to_pt(o, coeffs)[None], scale)[0]
    want = x / int(scale)
    assert np.all(got.imag == 0)
    assert np.all(np.abs(got.real - want) <= abs(want) * o.L * 2.0**-52)


# ---- 5. scheme semantics
def test_rotation_conjugation_product(oracle_mod):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 3)
    rng = np.random.default_rng(9)
    z1, z2 = _rand_slots(rng, n // 2), _rand_slots(rng, n // 2)
    scale = 2.0**30
    p1, p2 = ckks_ref.encode(o, z1, scale), ckks_ref.encode(o, z2, scale)
    for k in (1, 5, -3):
        perm = o.galois_perm(o.galois_elt(k))
        rot = np.ascontiguousarray(p1[0][:, perm])
        assert np.allclose(ckks_ref.decode(o, rot, scale)[0], np.roll(z1, -k), atol=1e-6)
    conj = np.ascontiguousarray(p1[0][:, o.galois_perm(2 * n - 1)])
    assert np.allclose(ckks_ref.decode(o, conj, scale)[0], np.conj(z1), atol=1e-6)
    prod = o.poly_mul_pointwise(p1, p2)
    assert np.allclose(ckks_ref.decode(o, prod, scale * scale)[0], z1 * z2, atol=1e-6)


# ---- 6. the kernel bodies, emulated, against the restatement
def _emu_cases():
    cases = [(logn, None, v) for logn in (12, 13, 14) for v in (None,)]
    cases += [(logn, "gen_mixed", None) for logn in (12, 14)]
    cases += [(logn, "fast_mixed", v) for logn in (12, 14) for v in ("fast", "gen")]
    return cases


@pytest.mark.parametrize("logn,basis,variant", _emu_cases())
def test_emulated_bodies_match_restatement(oracle_mod, emu_ckks, logn, basis, variant):
    n = 1 << logn
    moduli = bases.catalogue(oracle_mod)[basis][:4] if basis else None
    o = oracle_mod.Oracle(logn, 4, moduli)
    if variant is None:
        variant = "fast" if all(bases.is_fast(q) for q in o.moduli) else "gen"
    emu = EmuCkks(emu_ckks[variant], logn, o.moduli)
    rng = np.random.default_rng(logn)
    z = _rand_slots(rng, (2, n // 2)) * 4
    for scale in (2.0**40, 2.0**80):
        pt = ckks_ref.encode(o, z, scale)
        assert np.array_equal(emu.encode(z, scale), pt)
        want = ckks_ref.decode(o, pt, scale)
        assert np.array_equal(emu.decode(pt, scale).view(np.uint64), want.view(np.uint64))
    # decoding plaintexts that are not encodings (uniform residues: every coefficient near +-Q/2 somewhere)
    u = o.fill_uniform(11, 2)
    assert np.array_equal(emu.decode(u, 2.0**50).view(np.uint64), ckks_ref.decode(o, u, 2.0**50).view(np.uint64))
