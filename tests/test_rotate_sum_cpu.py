"""Summed rotations and slot sums without a GPU (DESIGN.md section 2.17).

The bodies of dpfhe_rotate_sum_grouped's kernels run through a host emulator (tests/emu/emu_rotate_sum.cpp) and must give the
oracle restatement (tests/slot_sum_ref.py) bit for bit; the restatement itself is pinned against the oracle's hoisted rotations,
decrypts its slot sums exactly, and tells apart the deliberate mistakes; the summed accumulator holds its lazy bound at the
threshold; dpfhe_slotsum_steps returns the documented order and rejects what lies outside its limits."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bgv_ref
import slot_sum_ref as ssr
from bases import catalogue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_libs = {}


def _build(variant):
    """tests/_emu/libdpfhe_emu_rotate_sum_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_rotate_sum_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_rotate_sum.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc] + srcs
                              + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_rs_create.restype = C.c_void_p
    lib.emu_rs_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_rs_destroy.argtypes = [C.c_void_p]
    lib.emu_rs_rotate_sum.argtypes = [C.c_void_p, C.c_uint, _u64p, C.c_uint, _u64p, _u64p, _u64p, C.c_size_t, C.c_uint64]
    lib.emu_rs_mac.argtypes = [C.c_void_p, C.c_uint, _u64p, _u64p, C.c_uint, _u64p, _u64p, _u64p, C.c_size_t]
    lib.emu_rs_schedule.argtypes = [C.c_uint, np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")]
    _libs[variant] = lib
    return lib


@pytest.fixture(scope="module")
def emu_rotate_sum():
    return _build


class EmuRotateSum:
    def __init__(self, build, log_n, moduli, variant):
        self._l = build(variant)
        arr = (C.c_uint64 * len(moduli))(*[int(m) for m in moduli])
        self._h = self._l.emu_rs_create(log_n, len(moduli), arr)
        assert self._h, "emu_rs_create rejected the parameters"

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_rs_destroy(self._h)
            self._h = None

    def rotate_sum(self, K, ct, galois, keys, t_plain):
        ct = np.ascontiguousarray(ct, dtype=np.uint64)
        out = np.zeros_like(ct)
        g = np.ascontiguousarray(galois, dtype=np.uint64)
        assert self._l.emu_rs_rotate_sum(self._h, int(K), ct.reshape(-1), len(g), g, np.ascontiguousarray(keys, dtype=np.uint64).reshape(-1),
                                         out.reshape(-1), ct.shape[0], int(t_plain)) == 0
        return out

    def mac(self, K, ct, U, galois, keys, L, N):
        ct = np.ascontiguousarray(ct, dtype=np.uint64)
        acc = np.zeros((ct.shape[0], 2, L, N), dtype=np.uint64)
        g = np.ascontiguousarray(galois, dtype=np.uint64)
        assert self._l.emu_rs_mac(self._h, int(K), ct.reshape(-1), np.ascontiguousarray(U, dtype=np.uint64).reshape(-1), len(g), g,
                                  np.ascontiguousarray(keys, dtype=np.uint64).reshape(-1), acc.reshape(-1), ct.shape[0]) == 0
        return acc


def _variants(moduli):
    return ("fast", "gen") if all(int(q) & 0xFFFFFFFF == 1 for q in moduli) else ("gen",)


def _inputs(o, oq, K, n_rot, batch, seed):
    """uniform ciphertexts (one c0 row of q - 1) and n_rot uniform grouped keys, with the Galois elements of rotations 1, -2, 3, ..."""
    ct = oq.fill_uniform(seed, 2 * batch).reshape(batch, 2, oq.L, o.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    ct[-1, 0] = (q - 1)[:, None]
    dnum = o.grouped_digits(K)
    keys = o.fill_uniform(seed + 1, n_rot * 2 * dnum).reshape(n_rot, dnum, 2, o.L, o.N)
    galois = [o.galois_elt((m + 1) * (-1) ** m) for m in range(n_rot)]
    return ct, galois, keys


# (K, Lq): digits of K limbs, the last one ragged where K does not divide Lq
SHAPES = [(1, 3), (2, 4), (2, 5), (3, 4), (4, 4)]
N_ROT = [1, 2, 7, 15]


@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_emulated_bodies_equal_the_restatement(oracle_mod, emu_rotate_sum, log_n, shape):
    K, Lq = SHAPES[shape]
    n_rot = N_ROT[(shape + log_n) % len(N_ROT)]
    o = oracle_mod.Oracle(log_n, Lq + K)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    ct, galois, keys = _inputs(o, oq, K, n_rot, 2, 10 * shape + log_n)
    for t in (0, 65537):
        want = ssr.rotate_sum(o, K, ct, galois, keys, t)
        for variant in _variants(o.moduli):
            got = EmuRotateSum(emu_rotate_sum, log_n, o.moduli, variant).rotate_sum(K, ct, galois, keys, t)
            assert np.array_equal(got, want), (variant, t, n_rot)


@pytest.mark.parametrize("n_rot", N_ROT)
def test_every_rotation_count(oracle_mod, emu_rotate_sum, n_rot):
    K, Lq = 2, 4
    o = oracle_mod.Oracle(12, Lq + K)
    oq = oracle_mod.Oracle(12, Lq, o.moduli[:Lq])
    ct, galois, keys = _inputs(o, oq, K, n_rot, 3, 100 + n_rot)
    for t in (0, 65537):
        want = ssr.rotate_sum(o, K, ct, galois, keys, t)
        for variant in _variants(o.moduli):
            assert np.array_equal(EmuRotateSum(emu_rotate_sum, 12, o.moduli, variant).rotate_sum(K, ct, galois, keys, t), want), (variant, t)


def test_generic_basis(oracle_mod, emu_rotate_sum):
    """gen_mixed: a 34-bit ciphertext modulus next to 59-bit ones, special primes of 55 and 45 bits"""
    mods = catalogue(oracle_mod)["gen_mixed"]
    K, L = 2, len(mods)
    o = oracle_mod.Oracle(12, L, mods)
    oq = oracle_mod.Oracle(12, L - K, mods[:L - K])
    ct, galois, keys = _inputs(o, oq, K, 7, 2, 90)
    e = EmuRotateSum(emu_rotate_sum, 12, mods, "gen")
    for t in (0, 65537):
        assert np.array_equal(e.rotate_sum(K, ct, galois, keys, t), ssr.rotate_sum(o, K, ct, galois, keys, t)), t


@pytest.mark.parametrize("K,Lq", [(1, 3), (2, 4), (3, 4)])
def test_one_rotation_is_hoisted_rotation_plus_add(oracle_mod, K, Lq):
    o = oracle_mod.Oracle(12, Lq + K)
    oq = oracle_mod.Oracle(12, Lq, o.moduli[:Lq])
    ct, galois, keys = _inputs(o, oq, K, 1, 2, 30 + K)
    for t in (0, 65537):
        rot = o.rotate_hoisted_grouped(K, ct, galois, keys, t)[0]
        assert np.array_equal(ssr.rotate_sum(o, K, ct, galois, keys, t), oq.poly_add(rot, ct)), t


def test_lazy_bound_at_its_threshold(oracle_mod, emu_rotate_sum):
    """all-(q - 1) ciphertexts, lifts and keys, n_rot = 15 and K = 1 (the largest dnum here): the most products of the largest
    operands; every accumulator is the exact sum mod q_i.  The Shoup products of these operands are 1 or q + 1, well inside
    their SB*q bound, so this does not reach the trim threshold: test_trim_schedule_keeps_every_row_below_16q pins that."""
    K, Lq, n_rot, log_n = 1, 5, 15, 12
    L, N = Lq + K, 1 << log_n
    o = oracle_mod.Oracle(log_n, L)
    q = [int(x) for x in o.moduli]
    dnum = o.grouped_digits(K)
    qa = np.array(q, dtype=np.uint64)
    ct = np.broadcast_to((qa[:Lq] - 1)[None, None, :, None], (1, 2, Lq, N)).copy()
    U = np.broadcast_to((qa - 1)[None, None, :, None], (1, dnum, L, N)).copy()
    keys = np.broadcast_to((qa - 1)[None, None, None, :, None], (n_rot, dnum, 2, L, N)).copy()
    galois = [o.galois_elt(m + 1) for m in range(n_rot)]
    Pspec = 1
    for k in range(K):
        Pspec *= q[Lq + k]
    for variant in _variants(q):
        acc = EmuRotateSum(emu_rotate_sum, log_n, q, variant).mac(K, ct, U, galois, keys, L, N)
        for i in range(L):
            prods = n_rot * dnum * (q[i] - 1) ** 2
            pm = Pspec % q[i]
            want0 = (prods + (pm * (q[i] - 1) * (1 + n_rot) if i < Lq else 0)) % q[i]
            want1 = (prods + (pm * (q[i] - 1) if i < Lq else 0)) % q[i]
            assert (acc[0, 0, i] == want0).all() and (acc[0, 1, i] == want1).all(), (variant, i)


@pytest.mark.parametrize("variant", ["fast", "gen"])
def test_trim_schedule_keeps_every_row_below_16q(emu_rotate_sum, variant):
    """the running bound of rot_sum_grouped_rows, as the kernel body keeps it, against the bound itself: a row starts below SB*q,
    each addition adds SB*q, a trim takes it to 8q; the bound never passes 16q after an addition, and a row is trimmed exactly
    when the next addition could pass 16q (the most additions: 15 rotations x (15 digits + the carried term), K = 1 at 16 limbs)"""
    n = 15 * 16
    trim = np.zeros(n, dtype=np.int32)
    SB = emu_rotate_sum(variant).emu_rs_schedule(n, trim)
    assert SB in (2, 4)
    b = SB
    for k in range(n):
        b += SB
        assert b <= 16, (k, b)
        want = b + SB > 16
        assert bool(trim[k]) == want, (k, b)
        if want:
            b = 8
    assert trim.any()


def _encrypt_slots(o, s, z, t, seed):
    enc = bgv_ref.encoder(o.N, t)
    return np.stack([o.encrypt(seed + i, t, s, enc.encode(zi)) for i, zi in enumerate(z)])


def _decrypt_slots(o, s, ct, t):
    enc = bgv_ref.encoder(o.N, t)
    return np.stack([enc.decode(np.asarray(o.decrypt(s, c, t), dtype=np.uint64)) for c in ct]).astype(np.uint64)


def _keys(o, K, t, s, steps, seed):
    return np.stack([o.keygen_galois_grouped(K, seed + k, t, s, o.galois_elt(st)) for k, st in enumerate(steps)])


@pytest.mark.parametrize("stride,radices", [(1, [2, 2]), (1, [4, 4, 4]), (3, [8, 2]), (5, [16]), (1, [3, 4, 4, 4, 4])])
def test_slot_sum_decrypts_to_the_windowed_sums(oracle_mod, stride, radices):
    K, Lq, t = 2, 4, 65537
    o = oracle_mod.Oracle(12, Lq + K)
    oq = oracle_mod.Oracle(12, Lq, o.moduli[:Lq])
    s = o.keygen_secret(7)
    sq = np.ascontiguousarray(s[:Lq])
    gks = _keys(o, K, t, s, ssr.steps(stride, radices), 500)
    rng = np.random.default_rng(stride)
    z = rng.integers(0, t, size=(2, 2, o.N // 2))
    ct = _encrypt_slots(oq, sq, z, t, 40)
    out = ssr.slot_sum(o, K, ct, stride, radices, gks, t)
    count = int(np.prod(radices))
    assert np.array_equal(_decrypt_slots(oq, sq, out, t), ssr.windowed_sum(z, stride, count, t).astype(np.uint64))


def test_mistakes_are_told_apart(oracle_mod):
    """dropping the carried c1 changes the bits and the plaintext; dividing every rotation separately and summing changes the bits,
    not the plaintext"""
    K, Lq, t = 2, 4, 65537
    o = oracle_mod.Oracle(12, Lq + K)
    oq = oracle_mod.Oracle(12, Lq, o.moduli[:Lq])
    s = o.keygen_secret(9)
    sq = np.ascontiguousarray(s[:Lq])
    steps = [1, 2, 3]
    gks = _keys(o, K, t, s, steps, 600)
    z = np.random.default_rng(1).integers(0, t, size=(1, 2, o.N // 2))
    ct = _encrypt_slots(oq, sq, z, t, 60)
    galois = [o.galois_elt(k) for k in steps]
    good = ssr.rotate_sum(o, K, ct, galois, gks, t)
    want = ssr.windowed_sum(z, 1, 4, t).astype(np.uint64)
    assert np.array_equal(_decrypt_slots(oq, sq, good, t), want)
    bad = ssr.rotate_sum(o, K, ct, galois, gks, t, drop_c1=True)
    assert not np.array_equal(bad, good)
    assert not np.array_equal(_decrypt_slots(oq, sq, bad, t), want)
    rots = o.rotate_hoisted_grouped(K, ct, galois, gks, t)
    separate = ct
    for r in rots:
        separate = oq.poly_add(separate, r)
    assert not np.array_equal(separate, good)
    assert np.array_equal(_decrypt_slots(oq, sq, separate, t), want)


def _steps_call(stride, radices, with_out=True):
    import deeppowers_b200 as dp
    lib = dp.load_library()
    rs = (C.c_uint * max(len(radices), 1))(*radices)
    n = C.c_size_t(0)
    out = (C.c_int * 256)()
    rc = lib.dpfhe_slotsum_steps(stride, rs, len(radices), out if with_out else None, C.byref(n))
    return rc, [out[k] for k in range(n.value)] if with_out and rc == 0 else n.value


def test_slotsum_steps_order_and_limits():
    import deeppowers_b200 as dp
    for stride, radices in [(1, [2, 2, 2, 2, 2, 2]), (1, [4, 4, 4]), (1, [8, 8]), (1, [16, 4]), (1, [3, 4, 4, 4, 4]), (768, [4]), (7, [2, 3])]:
        rc, got = _steps_call(stride, radices)
        assert rc == 0 and got == ssr.steps(stride, radices), (stride, radices)
        assert dp.slotsum_steps(stride, radices) == got
        assert _steps_call(stride, radices, with_out=False) == (0, sum(r - 1 for r in radices))
    assert _steps_call(1, [16, 16, 16])[1] == ssr.steps(1, [16, 16, 16])   # 4096 <= 8192
    assert _steps_call(2, [16, 16, 16])[0] == 0                              # 8192: N/2 at N = 16384
    for stride, radices in [(0, [2]), (1, []), (1, [1]), (1, [17]), (1, [0, 2]), (3, [16, 16, 16]), (1, [2] * 14), (1, [2] * 17),
                            (8193, [2]), (1 << 40, [2])]:
        assert _steps_call(stride, radices)[0] != 0, (stride, radices)
    with pytest.raises(dp.DpfheError):
        dp.slotsum_steps(1, [1])
