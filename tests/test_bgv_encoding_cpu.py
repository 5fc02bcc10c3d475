"""BGV slot encoding (DESIGN.md section 2.13) without a GPU: the reference (tests/slots.py's SlotEncoder with the oracle's
transforms) against the definition, and the product's kernel bodies, run by the host emulator (tests/emu/emu_bgv.cpp), against
the reference bit for bit and against Python integers at every threshold."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import bgv_ref
from bgv_ref import INT64_MAX, INT64_MIN, T_VALUES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")


def _build_emu_bgv(variant):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_bgv_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_bgv.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"),
                               "-x", "c++", "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_bgv_create.restype = C.c_void_p
    lib.emu_bgv_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_bgv_destroy.argtypes = [C.c_void_p]
    lib.emu_bgv_zeta.restype = C.c_uint64
    lib.emu_bgv_zeta.argtypes = [C.c_void_p, C.c_uint64]
    lib.emu_bgv_encode.argtypes = [C.c_void_p, _i64p, _u64p, C.c_size_t, C.c_uint64]
    lib.emu_bgv_decode.argtypes = [C.c_void_p, _u64p, _u64p, C.c_size_t, C.c_uint64]
    return lib


class EmuBgv:
    def __init__(self, lib, log_n, moduli):
        self._l, self.N, self.L = lib, 1 << log_n, len(moduli)
        self._h = lib.emu_bgv_create(log_n, self.L, (C.c_uint64 * self.L)(*[int(q) for q in moduli]))
        assert self._h

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_bgv_destroy(self._h)

    def zeta(self, t):
        return int(self._l.emu_bgv_zeta(self._h, t))

    def encode(self, slots, t):
        z = np.ascontiguousarray(slots, dtype=np.int64).reshape(-1, 2, self.N // 2)
        pt = np.empty((z.shape[0], self.L, self.N), dtype=np.uint64)
        assert self._l.emu_bgv_encode(self._h, z.reshape(-1), pt.reshape(-1), z.shape[0], t) == 0
        return pt

    def decode(self, pt, t):
        pt = np.ascontiguousarray(pt, dtype=np.uint64).reshape(-1, self.L, self.N)
        z = np.empty((pt.shape[0], 2, self.N // 2), dtype=np.uint64)
        assert self._l.emu_bgv_decode(self._h, pt.reshape(-1), z.reshape(-1), pt.shape[0], t) == 0
        return z


@pytest.fixture(scope="module")
def emu_bgv():
    return {v: _build_emu_bgv(v) for v in ("gen", "fast")}


def _rand_slots(rng, n_vec, n):
    return rng.integers(INT64_MIN, INT64_MAX, (n_vec, 2, n // 2), dtype=np.int64, endpoint=True)


# ---- 1. the reference against the definition m(zeta^(2i+1)) by Horner in Python integers
@pytest.mark.parametrize("logn", [12, 14])
def test_slot_encoder_evaluates_the_definition(logn):
    n, t = 1 << logn, 167772161
    enc = bgv_ref.encoder(n, t)
    assert enc.zeta == pow(3, (t - 1) // (2 * n), t)   # 3 is the least quadratic non-residue mod t
    rng = np.random.default_rng(logn)
    m = rng.integers(0, t, n).astype(np.uint64)
    got = enc.evaluate(m)
    coeffs = [int(c) for c in m]
    for i in list(rng.integers(0, n, 6)) + [0, n - 1]:
        x, acc = pow(enc.zeta, 2 * int(i) + 1, t), 0
        for c in reversed(coeffs):
            acc = (acc * x + c) % t
        assert int(got[i]) == acc
    # slot (0, c) is m(zeta^(5^c)), slot (1, c) is m(zeta^(-5^c)); encode is the inverse of decode
    slots = enc.decode(m)
    for c in (0, 1, n // 2 - 1):
        e = pow(5, c, 2 * n)
        for r, ex in ((0, e), (1, 2 * n - e)):
            x, acc = pow(enc.zeta, ex, t), 0
            for cf in reversed(coeffs):
                acc = (acc * x + cf) % t
            assert int(slots[r, c]) == acc
    assert np.array_equal(enc.encode(slots.astype(np.int64)), m)


# ---- 2. zeta and the plaintext moduli the product accepts
@pytest.mark.parametrize("logn", [12, 13, 14])
def test_zeta_equals_slot_encoder(oracle_mod, emu_bgv, logn):
    emu = EmuBgv(emu_bgv["fast"], logn, oracle_mod.Oracle(logn, 1).moduli)
    for t in T_VALUES:
        assert emu.zeta(t) == bgv_ref.encoder(1 << logn, t).zeta


def test_invalid_plaintext_moduli_rejected(oracle_mod, emu_bgv):
    for logn in (12, 14):
        n = 1 << logn
        emu = EmuBgv(emu_bgv["fast"], logn, oracle_mod.Oracle(logn, 1).moduli)
        composite = (2 * n + 1) ** 2                  # 1 mod 2N
        big = 3 * 2**30 + 1                           # prime, 1 mod 2^15, above 2^31
        for t in (0, 1, 2, composite, 1000003, 65539, big, 2**31 + 1, 2**32 + 1, 2**61 - 1):
            assert emu.zeta(t) == 0, t
            with pytest.raises(AssertionError):
                emu.encode(np.zeros((1, 2, n // 2), dtype=np.int64), t)
        assert emu.zeta(2147352577) != 0
    # 65537 = 1 mod 2^16 only: valid up to N = 32768, 786433 = 3 * 2^18 + 1 likewise
    assert EmuBgv(emu_bgv["gen"], 14, oracle_mod.Oracle(14, 1).moduli).zeta(786433) == bgv_ref.encoder(1 << 14, 786433).zeta


# ---- 3. the emulated bodies against the reference
def _emu_cases():
    cases = [(logn, None, None) for logn in (12, 13, 14)]
    cases += [(logn, "gen_mixed", None) for logn in (12, 14)]
    cases += [(logn, "fast_mixed", v) for logn in (12, 14) for v in ("fast", "gen")]
    return cases


@pytest.mark.parametrize("logn,basis,variant", _emu_cases())
def test_emulated_bodies_match_reference(oracle_mod, emu_bgv, logn, basis, variant):
    n = 1 << logn
    moduli = bases.catalogue(oracle_mod)[basis][:4] if basis else None
    o = oracle_mod.Oracle(logn, 4, moduli)
    if variant is None:
        variant = "fast" if all(bases.is_fast(q) for q in o.moduli) else "gen"
    emu = EmuBgv(emu_bgv[variant], logn, o.moduli)
    rng = np.random.default_rng(logn + 7)
    for t in T_VALUES:
        z = _rand_slots(rng, 2, n)
        z[1] = rng.integers(-t, t, (2, n // 2))
        pt = bgv_ref.encode(o, z, t)
        assert np.array_equal(emu.encode(z, t), pt)
        assert np.array_equal(emu.decode(pt, t), z % t)
    # decoding plaintexts that are not encodings (uniform residues: centred values anywhere in (-Q/2, Q/2])
    u = o.fill_uniform(11, 2)
    for t in (T_VALUES[1], T_VALUES[2]):
        assert np.array_equal(emu.decode(u, t), bgv_ref.decode(o, u, t))


# ---- 4. thresholds, against Python integers
def _floor_mod_cases(t):
    return [INT64_MIN, INT64_MIN + 1, -t, -t - 1, -t + 1, -1, 0, 1, t - 1, t, t + 1, INT64_MAX, INT64_MAX - 1]


@pytest.mark.parametrize("variant", ["gen", "fast"])
def test_slot_reduction_thresholds(oracle_mod, emu_bgv, variant):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 2, None if variant == "fast" else bases.catalogue(oracle_mod)["gen_mixed"][:2])
    emu = EmuBgv(emu_bgv[variant], logn, o.moduli)
    for t in T_VALUES:
        vals = _floor_mod_cases(t)
        z = np.zeros((2, n // 2), dtype=np.int64)
        z.reshape(-1)[: len(vals)] = vals
        z[1, -len(vals):] = vals
        want_slots = np.array([[int(v) % t for v in row] for row in z.tolist()], dtype=np.uint64)   # Python's floor-mod
        m = bgv_ref.encoder(n, t).encode(want_slots.astype(np.int64))
        assert np.array_equal(emu.encode(z, t)[0], bgv_ref.to_rns_eval(o, m, t))
        assert np.array_equal(emu.decode(emu.encode(z, t), t)[0], want_slots)


@pytest.mark.parametrize("variant", ["gen", "fast"])
def test_centred_lift_thresholds(oracle_mod, emu_bgv, variant):
    """coefficients exactly floor(t/2), floor(t/2)+1, 0 and t-1 at even and odd positions in both halves"""
    logn, n = 13, 8192
    o = oracle_mod.Oracle(logn, 3, None if variant == "fast" else bases.catalogue(oracle_mod)["gen_mixed"][:3])
    emu = EmuBgv(emu_bgv[variant], logn, o.moduli)
    rng = np.random.default_rng(3)
    for t in T_VALUES:
        h = t // 2
        m = rng.integers(0, t, n).astype(np.uint64)
        for k, v in enumerate((h, h + 1, 0, t - 1, h, h + 1, 0, t - 1)):
            for pos in (2 * k, 2 * k + 1, n // 2 + 2 * k, n - 1 - 2 * k):
                m[pos] = v
        enc = bgv_ref.encoder(n, t)
        slots = enc.decode(m).astype(np.int64)        # = SlotEncoder.evaluate(m), in slot order
        assert np.array_equal(enc.encode(slots), m)
        want = np.array([[(c if c <= h else c - t) % q for c in m.tolist()] for q in o.moduli], dtype=np.uint64)
        assert np.array_equal(emu.encode(slots, t)[0], o.ntt_fwd(want[None])[0])


@pytest.mark.parametrize("variant", ["gen", "fast"])
def test_decode_centring_thresholds(oracle_mod, emu_bgv, variant):
    logn, n = 12, 4096
    o = oracle_mod.Oracle(logn, 4, None if variant == "fast" else bases.catalogue(oracle_mod)["gen_mixed"][:4])
    emu = EmuBgv(emu_bgv[variant], logn, o.moduli)
    Q, q0 = bgv_ref.modulus_product(o), o.moduli[0]
    special = [0, 1, (Q - 1) // 2, (Q + 1) // 2, Q - 1, Q - q0, (Q - 1) // 2 - 1, (Q + 1) // 2 + 1]
    rng = np.random.default_rng(5)
    X = [int(v) for v in rng.integers(0, 2**62, n)]
    for k, v in enumerate(special):
        for pos in (k, n // 2 + k, n - 1 - k):
            X[pos] = v
    pt = bgv_ref.residues_of(o, X)
    for t in T_VALUES:
        coeffs = np.array([(x - Q if x > (Q - 1) // 2 else x) % t for x in X], dtype=np.uint64)
        want = bgv_ref.encoder(n, t).decode(coeffs)
        assert np.array_equal(emu.decode(pt, t)[0], want)
        assert np.array_equal(bgv_ref.decode(o, pt, t)[0], want)
