"""Multiply-and-rescale (DESIGN.md sections 2.19 / 4.16) without a GPU.

The restatement (tests/mul_rescale_ref.py) is pinned two ways: its accumulator divided by P alone is the inner product of the
oracle's own composition (tests/ct_dot_ref.py: ct_tensor, poly_add, keyswitch_grouped), bit for bit, and its result times
P' = P * q_{Lq-1} is the accumulator minus s * w over the integers (CRT), w the centred lifts of the K + 1 divided residues.
The kernel bodies (tests/emu/emu_mul_rescale.cpp, both arithmetic variants, in the kernel's role order) give the restatement bit for
bit over K = 1 .. 4 with ragged digits, N = 4096 .. 16384, 1 / 9 / 64 pairs and the five bases of tests/bases.py; their division
alone, on crafted accumulators, puts the dropped limb's y on both sides of its centring threshold and every one of the five rows of
K = 4 at q - 1 (the lazy bound's worst case), against the oracle's division by the last K + 1 limbs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ct_dot_ref as cdr
import mul_rescale_ref as mrr
from bases import catalogue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_libs = {}
T_BGV = 167772161
# (K, Lq): digits of K limbs, the last one ragged where K does not divide Lq; Lq = 2 leaves one limb
SHAPES = [(1, 2), (1, 3), (2, 4), (2, 5), (3, 4), (4, 4)]


def _build(variant):
    """tests/_emu/libdpfhe_emu_mul_rescale_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_mul_rescale_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_mul_rescale.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        tmp = "%s.%d.tmp" % (so, os.getpid())   # built aside and renamed: parallel test workers never load a half-written library
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-x", "c++", "-I", csrc]
                              + srcs + ["-o", tmp])
        os.replace(tmp, so)
    lib = C.CDLL(so)
    lib.emu_mr_create.restype = C.c_void_p
    lib.emu_mr_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_mr_destroy.argtypes = [C.c_void_p]
    lib.emu_mr_mul_rescale.argtypes = [C.c_void_p, C.c_uint, C.c_int, _u64p, C.c_uint, C.c_uint, _u32p, _u32p, _u64p, _u64p, C.c_size_t,
                                       C.c_uint64, C.c_uint]
    lib.emu_mr_divide.argtypes = [C.c_void_p, C.c_uint, _u64p, C.c_uint64, _u64p, C.c_size_t]
    _libs[variant] = lib
    return lib


class EmuMulRescale:
    def __init__(self, log_n, moduli, variant):
        self._l = _build(variant)
        arr = (C.c_uint64 * len(moduli))(*[int(m) for m in moduli])
        self._h = self._l.emu_mr_create(log_n, len(moduli), arr)
        assert self._h, "emu_mr_create rejected the parameters"
        self.L, self.N = len(moduli), 1 << log_n

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_mr_destroy(self._h)
            self._h = None

    def mul_rescale(self, K, pool, ia, ib, key, t_plain, dot, groups=2):
        """pool [n_pool][batch][2][Lq][N]; pair t is (pool[ia[t]], pool[ib[t]]) -> [batch][2][Lq-1][N]"""
        pool = np.ascontiguousarray(pool, dtype=np.uint64)
        b, Lq = pool.shape[1], pool.shape[3]
        out = np.zeros((b, 2, Lq - 1, self.N), dtype=np.uint64)
        ia, ib = np.ascontiguousarray(ia, dtype=np.uint32), np.ascontiguousarray(ib, dtype=np.uint32)
        assert self._l.emu_mr_mul_rescale(self._h, int(K), int(dot), pool.reshape(-1), pool.shape[0], len(ia), ia, ib,
                                          np.ascontiguousarray(key, dtype=np.uint64).reshape(-1), out.reshape(-1), b, int(t_plain), groups) == 0
        return out

    def divide(self, K, acc, t_plain):
        """acc [n][L][N] -> [n][L-K-1][N]"""
        acc = np.ascontiguousarray(acc, dtype=np.uint64)
        out = np.zeros((acc.shape[0], self.L - K - 1, self.N), dtype=np.uint64)
        assert self._l.emu_mr_divide(self._h, int(K), acc.reshape(-1), int(t_plain), out.reshape(-1), acc.shape[0]) == 0
        return out


def _variants(moduli):
    return ("fast", "gen") if all(int(q) & 0xFFFFFFFF == 1 for q in moduli) else ("gen",)


def _contexts(oracle_mod, log_n, K, Lq, moduli=None):
    o = oracle_mod.Oracle(log_n, Lq + K, moduli)
    return o, oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])


def _pool(oq, n_pool, batch, seed):
    """uniform ciphertexts with one row of q - 1 and one of 0"""
    pool = oq.fill_uniform(seed, n_pool * batch * 2).reshape(n_pool, batch, 2, oq.L, oq.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    pool[0, -1, 0] = (q - 1)[:, None]
    pool[-1, 0, 1] = 0
    return pool


def _pairs(n, n_pool):
    ia = [(2 * t) % n_pool for t in range(n)]
    ib = [(2 * t + 1) % n_pool for t in range(n)]
    ib[-1] = ia[-1]   # a square
    return ia, ib


def _crt(res, mods):
    """[len(mods)][n] residues -> the integers in [0, prod(mods)) (object array)"""
    M = 1
    for q in mods:
        M *= q
    x = 0
    for l, q in enumerate(mods):
        Ml = M // q
        x = x + res[l].astype(object) * (Ml * pow(Ml, -1, q))
    return x % M, M


# ---- the restatement itself ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K,Lq", SHAPES)
def test_accumulator_is_the_oracles_inner_product_times_p(oracle_mod, K, Lq):
    """the accumulator divided by P alone (the oracle's dpo_mod_down_special with K limbs) is the oracle's composition of the
    inner product, bit for bit: acc = P D + sum_g U_g o evk[g] is checked against code that never forms it"""
    o, oq = _contexts(oracle_mod, 12, K, Lq)
    pool = _pool(oq, 3, 2, 40 + K + Lq)
    key = o.fill_uniform(50 + K, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    a_list, b_list = [pool[0], pool[2]], [pool[1], pool[2]]
    acc = mrr.accumulator(o, K, a_list, b_list, key)
    for t in (0, 65537):
        got = o.mod_down_special(K, acc.reshape(-1, o.L, o.N), t).reshape(2, 2, Lq, o.N)
        assert np.array_equal(got, cdr.ct_dot(o, oq, K, a_list, b_list, key, t)), t


@pytest.mark.parametrize("L,K,t", [(6, 2, 65537), (6, 2, 0), (5, 1, T_BGV), (8, 4, 0), (7, 2, 65537)])
def test_restatement_against_integers(oracle_mod, L, K, t):
    """out * P' = acc - s * w exactly, with w the sum of the centred lifts of the K + 1 divided residues of acc / s"""
    o = oracle_mod.Oracle(12, L)
    Lq = L - K
    oq = oracle_mod.Oracle(12, Lq, o.moduli[:Lq])
    ol = oracle_mod.Oracle(12, Lq - 1, o.moduli[:Lq - 1])
    a = oq.fill_uniform(10 + L, 2).reshape(1, 2, Lq, o.N)
    b = oq.fill_uniform(20 + L, 2).reshape(1, 2, Lq, o.N)
    key = o.fill_uniform(30 + L, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    out = mrr.mul_rescale(o, K, [a, a], [b, a], key, t)
    acc = mrr.accumulator(o, K, [a, a], [b, a], key)
    mods = [int(q) for q in o.moduli]
    divided = mods[Lq - 1:]   # q_{Lq-1}, p_0 .. p_{K-1}
    Pp = 1
    for m in divided:
        Pp *= m
    s = t if t else 1
    for c in range(2):
        X, _ = _crt(o.ntt_inv(acc[0, c]), mods)
        O, Ql = _crt(ol.ntt_inv(out[0, c]), mods[:Lq - 1])
        w = 0
        for m in divided:
            Pm = Pp // m
            y = (X % m) * pow(s * Pm % m, -1, m) % m
            y = np.where(y > m // 2, y - m, y)
            w = w + y * Pm
        diff = X - s * w
        assert all(v % Pp == 0 for v in diff)
        assert all((v // Pp) % Ql == r for v, r in zip(diff, O))


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_emulated_bodies_every_shape_and_degree(oracle_mod, log_n, shape):
    K, Lq = SHAPES[shape]
    n_terms = (1, 9, 64)[(shape + log_n) % 3]
    o, oq = _contexts(oracle_mod, log_n, K, Lq)
    n_pool = min(2 * n_terms, 6)
    pool = _pool(oq, n_pool, 3, 800 + 10 * shape + log_n)
    ia, ib = _pairs(n_terms, n_pool)
    key = o.fill_uniform(900 + shape, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    t = (0, 65537, T_BGV)[(shape + 2 * log_n) % 3]
    want = mrr.mul_rescale(o, K, [pool[i] for i in ia], [pool[i] for i in ib], key, t)
    for variant in _variants(o.moduli):
        e = EmuMulRescale(log_n, o.moduli, variant)
        assert np.array_equal(e.mul_rescale(K, pool, ia, ib, key, t, dot=True), want), (variant, n_terms)
        if n_terms == 1:   # phase 1 in mode KS_MUL_RELIN
            assert np.array_equal(e.mul_rescale(K, pool, ia, ib, key, t, dot=False), want), variant


@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_emulated_bodies_on_other_bases(oracle_mod, basis):
    mods = catalogue(oracle_mod)[basis]
    K, log_n = 2, 12
    o, oq = _contexts(oracle_mod, log_n, K, len(mods) - K, mods)
    key = o.fill_uniform(1000, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    for n_terms, t in ((1, T_BGV), (9, 0), (64, 65537)):
        pool = _pool(oq, min(2 * n_terms, 6), 3, 1010 + n_terms)
        ia, ib = _pairs(n_terms, pool.shape[0])
        want = mrr.mul_rescale(o, K, [pool[i] for i in ia], [pool[i] for i in ib], key, t)
        for variant in _variants(mods):
            got = EmuMulRescale(log_n, mods, variant).mul_rescale(K, pool, ia, ib, key, t, dot=n_terms > 1)
            assert np.array_equal(got, want), (variant, n_terms)


# ---- the division on crafted accumulators -----------------------------------------------------------------------------------------

def _crafted_acc(o, K, ys, kept):
    """an accumulator [L][N] whose divided rows give the residues ys[m] (m = 0: the dropped limb q_{Lq-1}, m = 1 + k: special prime k)
    as y = INTT(acc_m) (s Phat'_m)^-1 mod m, and whose kept rows are `kept` [Lq-1][N] (evaluation form); s is folded in by the caller
    through the returned closure, one accumulator per plaintext modulus"""
    L, N = o.L, o.N
    Lq = L - K
    mods = [int(q) for q in o.moduli]
    divided = list(range(Lq - 1, L))

    def build(t):
        s = t if t else 1
        coef = np.zeros((L, N), dtype=np.uint64)
        for j, l in enumerate(divided):
            m = mods[l]
            f = s % m
            for l2 in divided:
                if l2 != l:
                    f = f * mods[l2] % m
            coef[l] = np.array([int(v) * f % m for v in ys[j]], dtype=np.uint64)
        ev = o.ntt_fwd(coef[None])[0]
        ev[:Lq - 1] = kept
        return ev
    return build


def _thresholds(q, n):
    """0, 1, h - 1, h, h + 1, q - 2, q - 1 (h = floor(q / 2)) tiled over n coefficients"""
    h = q // 2
    vals = [0, 1, h - 1, h, h + 1, q - 2, q - 1]
    return [vals[i % len(vals)] for i in range(n)]


@pytest.mark.parametrize("K,Lq", [(2, 4), (1, 2), (2, 5)])
def test_dropped_limb_y_at_its_threshold(oracle_mod, K, Lq):
    """the dropped limb's y at 0, 1, h - 1, h, h + 1, q - 2, q - 1 (the special rows at theirs, shifted), kept rows uniform: the
    emulated division is the oracle's division by the last K + 1 limbs bit for bit, so `>` against `>=` at h is told apart"""
    log_n = 12
    o, _ = _contexts(oracle_mod, log_n, K, Lq)
    N, mods = o.N, [int(q) for q in o.moduli]
    ys = [_thresholds(mods[Lq - 1], N)] + [_thresholds(mods[Lq + k], N)[3 * (k + 1):] + _thresholds(mods[Lq + k], N)[:3 * (k + 1)]
                                           for k in range(K)]
    kept = o.fill_uniform(77, 1)[0][:Lq - 1]
    build = _crafted_acc(o, K, ys, kept)
    for t in (0, 65537, T_BGV):
        acc = build(t)
        want = o.mod_down_special(K + 1, acc[None], t)
        for variant in _variants(o.moduli):
            assert np.array_equal(EmuMulRescale(log_n, o.moduli, variant).divide(K, acc[None], t), want), (variant, t)
    # the crafted rows are where they were meant to be: the oracle's own y of the dropped limb (s = 1) is the tiled thresholds
    acc = build(0)
    y = o.ntt_inv(acc[None])[0][Lq - 1]
    P = 1
    for k in range(K):
        P *= mods[Lq + k]
    assert [int(v) * pow(P, -1, mods[Lq - 1]) % mods[Lq - 1] for v in y[:7]] == _thresholds(mods[Lq - 1], 7)


@pytest.mark.parametrize("which", ["q_minus_1", "half_plus_1"])
def test_lazy_bound_five_rows(oracle_mod, which):
    """K = 4: all five divided rows above half (every y = q - 1, or every y = h + 1) and every kept accumulator word at q - 1, the
    largest sum of the per-term reduced lifts; the emulated division is the oracle's, bit for bit"""
    log_n, K, Lq = 12, 4, 4
    o, _ = _contexts(oracle_mod, log_n, K, Lq)
    N, mods = o.N, [int(q) for q in o.moduli]
    divided = mods[Lq - 1:]
    ys = [[m - 1] * N if which == "q_minus_1" else [m // 2 + 1] * N for m in divided]
    kept = np.broadcast_to(np.array(mods[:Lq - 1], dtype=np.uint64)[:, None] - np.uint64(1), (Lq - 1, N)).copy()
    build = _crafted_acc(o, K, ys, kept)
    for t in (0, T_BGV):
        acc = build(t)
        want = o.mod_down_special(K + 1, acc[None], t)
        for variant in _variants(o.moduli):
            assert np.array_equal(EmuMulRescale(log_n, o.moduli, variant).divide(K, acc[None], t), want), (variant, t)
