"""The product's compact-ciphertext bodies (deeppowers_b200/csrc/compact.cuh) without a GPU: run tile by tile by the host emulator
(tests/emu/emu_compact.cpp) in both arithmetic variants and compared with the restatement of DESIGN.md section 2.24
(tests/compact_ref.py) at the thresholds of the switch and of the decryption: x = 0, 1 and q0 - 1, z next to q0 / 2, j = +-(t - 1) / 2,
prod next to q0 / 2 and phi = -2^(bits - 1).  The emulator built from a mutated body (the correction j dropped, a coefficient's bit
offset off by one, c1' lifted without centring) must fail the same comparison."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bases
import compact_ref as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deeppowers_b200", "csrc")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
T = 65537

# (name, text of compact.cuh, its replacement)
MUTANTS = [
    ("no_j", "y = jr > (A.t >> 1) ? Q - jr + A.t : Q - jr;", "y = Q;"),
    ("bit_offset", "const int s = (int)(i * bits) - (int)lo;", "const int s = (int)(i * bits + 1) - (int)lo;"),
    ("uncentred_lift", "return c1 >> (A.bits - 1) ? c1 - ((u64)1 << A.bits) + A.q : c1;", "return c1;"),
]


def _build(variant, mutant=None):
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    tag = variant + ("_" + mutant[0] if mutant else "")
    so = os.path.join(out_dir, "libdpfhe_emu_compact_%s.so" % tag)
    inc = [CSRC]
    if mutant:
        mdir = os.path.join(out_dir, "compact_" + mutant[0])
        os.makedirs(mdir, exist_ok=True)
        text = open(os.path.join(CSRC, "compact.cuh")).read()
        assert text.count(mutant[1]) == 1, "the mutated line is no longer in compact.cuh"
        with open(os.path.join(mdir, "compact.cuh"), "w") as f:
            f.write(text.replace(mutant[1], mutant[2]))
        inc = [mdir, CSRC]
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_compact.cpp"), os.path.join(CSRC, "host_params.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("types.hpp", "modarith.cuh", "kernel_bodies.cuh", "compact.cuh", "host_params.hpp")]
    if mutant or not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        cmd = [gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++"]
        for d in inc:
            cmd += ["-I", d]
        subprocess.check_call(cmd + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_compact_pack.argtypes = [C.c_uint64, C.c_uint, C.c_uint, C.c_uint64, _u64p, _u64p, C.c_size_t]
    lib.emu_compact_unpack.argtypes = [C.c_int, C.c_uint64, C.c_uint, C.c_uint, C.c_uint64, _u64p, _u64p, _u64p, C.c_size_t]
    return lib


@pytest.fixture(scope="module")
def emu():
    return {v: _build(v) for v in ("gen", "fast")}


def _threshold_x(q0, bits, t, N, rng):
    """a polynomial pair [2][N] of coefficients at the switch's thresholds, the rest uniform"""
    r_inv = pow(pow(2, bits, q0), -1, q0)
    xs = [0, 1, q0 - 1]
    xs += [z * r_inv % q0 for z in ((q0 - 1) // 2, (q0 + 1) // 2, (q0 - 3) // 2, (q0 + 3) // 2)]   # z next to q0 / 2
    if t:
        for j in ((t - 1) // 2, -(t - 1) // 2, (t + 1) // 2 - t):
            z0 = -j * q0 % t   # -z q0^-1 = j (mod t)
            for z in (z0, z0 + t, z0 + t * (q0 // t - 2)):
                xs.append(z * r_inv % q0)
    x = rng.integers(0, q0, size=2 * N, dtype=np.uint64)
    x[:len(xs)] = xs
    x[N:N + len(xs)] = xs[::-1]
    return x.reshape(2, N)


def _run_all(lib, q0, log_n, bits, t, rng):
    """True when pack, lift and finish of the emulator match the restatement on threshold inputs"""
    N = 1 << log_n
    x = _threshold_x(q0, bits, t, N, rng)
    out = np.zeros(2 * N * bits // 64, dtype=np.uint64)
    lib.emu_compact_pack(q0, log_n, bits, t, x.reshape(-1), out, 2)
    want = cr.pack(np.array([[cr.switch(int(v), q0, bits, t)[0] for v in row] for row in x], dtype=object), bits)
    ok = np.array_equal(out, want.reshape(-1))
    # decryption side: c0', c1' of a packed pair, prod [N] with the thresholds of the centred product and phi = -2^(bits-1)
    half = 1 << (bits - 1)
    y = rng.integers(0, 1 << bits, size=(2, N), dtype=np.uint64)
    y[1, :6] = [0, 1, half - 1, half, half + 1, (1 << bits) - 1]
    y[0, :4] = [half, half, 0, half - 1]
    prod = rng.integers(0, q0, size=N, dtype=np.uint64)
    prod[:8] = [0, 0, (q0 - 1) // 2, (q0 + 1) // 2, q0 - 1, 1, (q0 - 1) // 2 - half, (q0 + 1) // 2 + half]
    cct = cr.pack(y, bits).reshape(-1)
    lifted = np.zeros(N, dtype=np.uint64)
    lib.emu_compact_unpack(0, q0, log_n, bits, t, cct, np.zeros(1, dtype=np.uint64), lifted, 1)
    ok &= [int(v) for v in lifted] == [cr.lift(int(c), q0, bits) for c in y[1]]
    pt = np.zeros(N, dtype=np.uint64)
    lib.emu_compact_unpack(1, q0, log_n, bits, t, cct, prod, pt, 1)
    want_pt = []
    for c0, p in zip(y[0], prod):
        v = int(p) - q0 if int(p) > q0 // 2 else int(p)
        ph = (int(c0) + v) % (1 << bits)
        want_pt.append(cr.plain_coeff(ph - (1 << bits) if ph >= half else ph, q0, bits, t))
    ok &= [int(v) for v in pt] == want_pt
    return bool(ok)


@pytest.mark.parametrize("variant,log_n,basis", [("gen", 12, None), ("fast", 12, None), ("gen", 13, "gen_mixed"), ("fast", 14, None)])
@pytest.mark.parametrize("t", [T, 3, 0])
def test_compact_bodies_match_the_restatement(emu, oracle_mod, variant, log_n, basis, t):
    """every bits from 2 (t permitting) to the largest with N 2^bits < q0"""
    if variant == "fast" and basis:
        pytest.skip("the fast variant takes k 2^32 + 1 moduli only")
    q0 = int((bases.catalogue(oracle_mod)[basis] if basis else oracle_mod.Oracle(log_n, 1).moduli)[0])
    rng = np.random.default_rng(log_n * 7 + t)
    lo = max(2, (t.bit_length() + 1) if t else 2)
    for bits in sorted({lo, lo + 1, 31, 32, 33, cr.max_bits(log_n, q0)}):
        if bits < lo or bits > cr.max_bits(log_n, q0):
            continue
        assert _run_all(emu[variant], q0, log_n, bits, t, rng), "bits = %d" % bits


@pytest.mark.parametrize("mutant", MUTANTS, ids=[m[0] for m in MUTANTS])
def test_mutated_bodies_are_caught(oracle_mod, mutant):
    lib = _build("gen", mutant)
    q0 = int(oracle_mod.Oracle(12, 1).moduli[0])
    rng = np.random.default_rng(5)
    assert not _run_all(lib, q0, 12, 33, T, rng)
