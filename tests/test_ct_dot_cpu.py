"""Encrypted inner products without a GPU (DESIGN.md section 2.18 / 4.15).

The restatement (tests/ct_dot_ref.py: the oracle's ct_tensor, poly_add and keyswitch_grouped composed) is pinned against the
oracle's ct x ct product and Python integers, decrypts to the slot-wise sum of products and tells the deliberate mistakes apart;
the kernel bodies (ks_phase1 in mode KS_DOT with the unchanged grouped bodies, compiled for the host by tests/emu/emu_ct_dot.cpp,
both arithmetic variants) give the restatement bit for bit on both sides of the reduction cadence; the summed tensor product holds
its lazy bound with every operand word at q - 1."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bgv_ref
import ckks
import ct_dot_ref as cdr
from bases import LARGEST_GENERIC, SMALLEST_GENERIC, catalogue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_libs = {}

# the reduction cadence folds D_1 every 8 pairs and D_0, D_2 every 16: both sides of each boundary, and the largest call
N_TERMS = [1, 2, 7, 8, 9, 15, 16, 17, 33, 64]
# (K, Lq): digits of K limbs, the last one ragged where K does not divide Lq
SHAPES = [(1, 3), (2, 4), (2, 5), (3, 4), (4, 4)]


def _build(variant):
    """tests/_emu/libdpfhe_emu_ct_dot_<variant>.so: the bodies of one arithmetic variant compiled for the host"""
    if variant in _libs:
        return _libs[variant]
    out_dir = os.path.join(ROOT, "tests", "_emu")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libdpfhe_emu_ct_dot_%s.so" % variant)
    csrc = os.path.join(ROOT, "deeppowers_b200", "csrc")
    srcs = [os.path.join(ROOT, "tests", "emu", "emu_ct_dot.cpp"), os.path.join(csrc, "host_params.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in ("types.hpp", "modarith.cuh", "ntt_core.cuh", "kernel_bodies.cuh", "host_params.hpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DDPFHE_FAST=%d" % (variant == "fast"), "-DDPFHE_DOT_TRACK", "-x", "c++",
                               "-I", csrc] + srcs + ["-o", so])
    lib = C.CDLL(so)
    lib.emu_dot_create.restype = C.c_void_p
    lib.emu_dot_create.argtypes = [C.c_uint, C.c_uint, C.c_void_p]
    lib.emu_dot_destroy.argtypes = [C.c_void_p]
    lib.emu_dot_ct_dot.argtypes = [C.c_void_p, C.c_uint, _u64p, C.c_uint, C.c_uint, _u32p, _u32p, _u64p, _u64p, C.c_size_t, C.c_uint64, C.c_uint]
    lib.emu_dot_sums.argtypes = [C.c_void_p, C.c_uint, _u64p, C.c_uint, C.c_uint, _u32p, _u32p, _u64p]
    lib.emu_dot_track.argtypes = [np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")]
    _libs[variant] = lib
    return lib


class EmuDot:
    def __init__(self, log_n, moduli, variant):
        self._l = _build(variant)
        arr = (C.c_uint64 * len(moduli))(*[int(m) for m in moduli])
        self._h = self._l.emu_dot_create(log_n, len(moduli), arr)
        assert self._h, "emu_dot_create rejected the parameters"
        self.L, self.N = len(moduli), 1 << log_n

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.emu_dot_destroy(self._h)
            self._h = None

    def ct_dot(self, K, pool, ia, ib, key, t_plain, groups=2):
        """pool [n_pool][batch][2][Lq][N]; pair t is (pool[ia[t]], pool[ib[t]])"""
        pool = np.ascontiguousarray(pool, dtype=np.uint64)
        out = np.zeros(pool.shape[1:], dtype=np.uint64)
        ia, ib = np.ascontiguousarray(ia, dtype=np.uint32), np.ascontiguousarray(ib, dtype=np.uint32)
        assert self._l.emu_dot_ct_dot(self._h, int(K), pool.reshape(-1), pool.shape[0], len(ia), ia, ib, np.ascontiguousarray(key).reshape(-1),
                                      out.reshape(-1), pool.shape[1], int(t_plain), groups) == 0
        return out

    def sums(self, pool, ia, ib):
        """pool [n_pool][1][2][Lq][N] -> the raw sums [3][Lq][N] (below 15q, congruent)"""
        pool = np.ascontiguousarray(pool, dtype=np.uint64)
        Lq = pool.shape[3]
        out = np.zeros((3, Lq, self.N), dtype=np.uint64)
        ia, ib = np.ascontiguousarray(ia, dtype=np.uint32), np.ascontiguousarray(ib, dtype=np.uint32)
        assert self._l.emu_dot_sums(self._h, Lq, pool.reshape(-1), pool.shape[0], len(ia), ia, ib, out.reshape(-1)) == 0
        return out

    def track(self):
        t = np.zeros(2)
        self._l.emu_dot_track(t)
        return float(t[0]), float(t[1])


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
    """n pairs over a pool: distinct operands while they last, then repeats, one square"""
    ia = [(2 * t) % n_pool for t in range(n)]
    ib = [(2 * t + 1) % n_pool for t in range(n)]
    ib[-1] = ia[-1]
    return ia, ib


# ---- the restatement itself ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K,Lq", SHAPES)
def test_one_pair_is_the_ct_product(oracle_mod, K, Lq):
    o, oq = _contexts(oracle_mod, 12, K, Lq)
    pool = _pool(oq, 2, 2, 10 + K)
    evk = o.fill_uniform(20 + K, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    for t in (0, 65537):
        assert np.array_equal(cdr.ct_dot(o, oq, K, [pool[0]], [pool[1]], evk, t), o.ct_mul_relin_grouped(K, pool[0], pool[1], evk, t)), t


def test_tensor_sums_against_integers(oracle_mod):
    o, oq = _contexts(oracle_mod, 12, 2, 4)
    n = 9
    pool = _pool(oq, 2 * n, 1, 31)
    d = cdr.tensor_sum(oq, list(pool[0::2]), list(pool[1::2]))
    cols = [0, 1, 17, oq.N - 1]
    for l, q in enumerate(oq.moduli):
        for c in cols:
            a = [[int(pool[2 * i, 0, k, l, c]) for k in range(2)] for i in range(n)]
            b = [[int(pool[2 * i + 1, 0, k, l, c]) for k in range(2)] for i in range(n)]
            want = [sum(x[0] * y[0] for x, y in zip(a, b)) % q, sum(x[0] * y[1] + x[1] * y[0] for x, y in zip(a, b)) % q,
                    sum(x[1] * y[1] for x, y in zip(a, b)) % q]
            assert [int(d[0, k, l, c]) for k in range(3)] == want, (l, c)


# ---- semantics ------------------------------------------------------------------------------------------------------------------

def _encrypt_slots(oq, sq, z, t, seed):
    enc = bgv_ref.encoder(oq.N, t)
    return np.stack([oq.encrypt(seed + i, t, sq, enc.encode(zi)) for i, zi in enumerate(z)])


def _decrypt_slots(oq, sq, ct, t):
    enc = bgv_ref.encoder(oq.N, t)
    return np.asarray(enc.decode(np.asarray(oq.decrypt(sq, ct, t), dtype=np.uint64))).astype(np.uint64)


@pytest.mark.parametrize("K,Lq", SHAPES)
def test_bgv_decrypts_to_the_sum_of_products(oracle_mod, K, Lq):
    t, n = 65537, 5
    o, oq = _contexts(oracle_mod, 12, K, Lq)
    s = o.keygen_secret(3)
    sq = np.ascontiguousarray(s[:Lq])
    evk = o.keygen_relin_grouped(K, 4, t, s)
    rng = np.random.default_rng(K * 10 + Lq)
    z = rng.integers(0, t, size=(n + 1, 2, o.N // 2))
    cts = _encrypt_slots(oq, sq, z, t, 50)
    # pairs (0,1) (1,2) ... : every operand but the ends appears twice; then a square
    a = [cts[i][None] for i in range(n)]
    b = [cts[i + 1][None] for i in range(n - 1)] + [cts[n - 1][None]]
    zi = z.astype(object)
    want = (sum(zi[i] * zi[i + 1] for i in range(n - 1)) + zi[n - 1] * zi[n - 1]) % t
    got = _decrypt_slots(oq, sq, cdr.ct_dot(o, oq, K, a, b, evk, t)[0], t)
    assert np.array_equal(got.reshape(want.shape), want.astype(np.uint64))


def test_bgv_sum_of_squares(oracle_mod):
    t, n, K, Lq = 65537, 4, 2, 4
    o, oq = _contexts(oracle_mod, 12, K, Lq)
    s = o.keygen_secret(5)
    sq = np.ascontiguousarray(s[:Lq])
    evk = o.keygen_relin_grouped(K, 6, t, s)
    z = np.random.default_rng(2).integers(0, t, size=(n, 2, o.N // 2))
    cts = _encrypt_slots(oq, sq, z, t, 70)
    ops = [c[None] for c in cts]
    want = (z.astype(object) ** 2).sum(axis=0) % t
    got = _decrypt_slots(oq, sq, cdr.ct_dot(o, oq, K, ops, ops, evk, t)[0], t)
    assert np.array_equal(got.reshape(want.shape), want.astype(np.uint64))


def _key_switch_noise(oq, sq, out, d3, t):
    """centred (phase(out) - phase(d3 under 1, s, s^2)) / t: what the key switch and its rounding added"""
    diff = oq.poly_add(oq.phase(sq, out)[None], _negate(oq, oq.phase(sq, d3))[None])[0]
    vals = bgv_ref.centred_values(oq, diff)   # the oracle's phase is in coefficient form
    assert all(v % t == 0 for v in vals)
    return max(abs(v) // t for v in vals)


def _negate(oq, x):
    q = np.array(oq.moduli, dtype=np.uint64)[:, None]
    return np.where(x == 0, x, q - x)


def test_mistakes_are_told_apart_and_noise_is_lower(oracle_mod):
    """key-switching D_1 instead of D_2, or adding D_0 / D_1 without the factor P, changes bits and plaintext; n separate products
    summed change the bits, not the plaintext, and carry n key-switching terms where the inner product carries one"""
    t, n, K, Lq = 65537, 8, 2, 4
    o, oq = _contexts(oracle_mod, 12, K, Lq)
    s = o.keygen_secret(8)
    sq = np.ascontiguousarray(s[:Lq])
    evk = o.keygen_relin_grouped(K, 9, t, s)
    z = np.random.default_rng(3).integers(0, t, size=(2 * n, 2, o.N // 2))
    cts = _encrypt_slots(oq, sq, z, t, 90)
    a, b = [c[None] for c in cts[:n]], [c[None] for c in cts[n:]]
    zi = z.astype(object)
    want = (sum(zi[i] * zi[n + i] for i in range(n)) % t).astype(np.uint64)
    good = cdr.ct_dot(o, oq, K, a, b, evk, t)
    assert np.array_equal(_decrypt_slots(oq, sq, good[0], t).reshape(want.shape), want)
    for bad in (cdr.ct_dot(o, oq, K, a, b, evk, t, switch_component=1), cdr.ct_dot_unscaled(o, oq, K, a, b, evk, t)):
        assert not np.array_equal(bad, good)
        assert not np.array_equal(_decrypt_slots(oq, sq, bad[0], t).reshape(want.shape), want)
    parts = [o.ct_mul_relin_grouped(K, x, y, evk, t) for x, y in zip(a, b)]
    separate = parts[0]
    for p in parts[1:]:
        separate = oq.poly_add(separate, p)
    assert not np.array_equal(separate, good)
    assert np.array_equal(_decrypt_slots(oq, sq, separate[0], t).reshape(want.shape), want)
    d3 = cdr.tensor_sum(oq, a, b)[0]
    noise_dot = _key_switch_noise(oq, sq, good[0], d3, t)
    noise_sep = _key_switch_noise(oq, sq, separate[0], d3, t)
    print("key-switching noise, %d pairs: inner product %d, separate products summed %d" % (n, noise_dot, noise_sep))
    assert 0 < noise_dot < noise_sep


def test_ckks_inner_product_with_rescale(oracle_mod):
    """t = 0: the plain rounding; the result rescaled by the last ciphertext modulus decodes to sum_i z_i w_i"""
    K, Lq, n, log_n = 2, 4, 6, 12
    o, oq = _contexts(oracle_mod, log_n, K, Lq)
    N = o.N
    s = o.keygen_secret(11)
    sq = np.ascontiguousarray(s[:Lq])
    evk = o.keygen_relin_grouped(K, 12, 1, s)
    slots = list(range(8))
    scale = float(2 ** 50)   # 2^40 after the rescale: its rounding (half a unit per coefficient) stays far below the tolerance
    rng = np.random.default_rng(4)
    z = rng.uniform(-1, 1, size=(2 * n, len(slots))) + 1j * rng.uniform(-1, 1, size=(2 * n, len(slots)))
    cts = [ckks.encrypt(oq, sq, ckks.encode(zi, slots, N, scale), 200 + i)[None] for i, zi in enumerate(z)]
    out = cdr.ct_dot(o, oq, K, cts[:n], cts[n:], evk, 0)
    low = oq.mod_switch_down(out.reshape(2, Lq, N), 0)
    ol = oracle_mod.Oracle(log_n, Lq - 1, oq.moduli[:Lq - 1])
    got = ckks.decode(ckks.decrypt_coeffs(ol, np.ascontiguousarray(sq[:Lq - 1]), low), slots, N, scale * scale / oq.moduli[-1])
    want = (z[:n] * z[n:]).sum(axis=0)
    assert np.abs(got - want).max() < 2.0 ** -20, np.abs(got - want).max()


# ---- the kernel bodies ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_terms", N_TERMS)
def test_emulated_bodies_equal_the_restatement(oracle_mod, n_terms):
    """default basis, K = 2 over four limbs, three ciphertexts over two groups (two rounds: both parities of the double buffers)"""
    K, Lq, log_n, batch = 2, 4, 12, 3
    o, oq = _contexts(oracle_mod, log_n, K, Lq)
    n_pool = min(2 * n_terms, 12)
    pool = _pool(oq, n_pool, batch, 300 + n_terms)
    ia, ib = _pairs(n_terms, n_pool)
    evk = o.fill_uniform(400 + n_terms, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    for t in (0, 65537):
        want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], evk, t)
        for variant in _variants(o.moduli):
            assert np.array_equal(EmuDot(log_n, o.moduli, variant).ct_dot(K, pool, ia, ib, evk, t), want), (variant, t)


@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_emulated_bodies_every_shape_and_degree(oracle_mod, log_n, shape):
    K, Lq = SHAPES[shape]
    n_terms = N_TERMS[(3 * shape + log_n) % len(N_TERMS)]
    o, oq = _contexts(oracle_mod, log_n, K, Lq)
    n_pool = min(2 * n_terms, 6)
    pool = _pool(oq, n_pool, 2, 500 + 10 * shape + log_n)
    ia, ib = _pairs(n_terms, n_pool)
    evk = o.fill_uniform(600 + shape, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    t = (0, 65537)[(shape + log_n) % 2]
    want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], evk, t)
    for variant in _variants(o.moduli):
        assert np.array_equal(EmuDot(log_n, o.moduli, variant).ct_dot(K, pool, ia, ib, evk, t, groups=1), want), (variant, n_terms)


@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_emulated_bodies_on_other_bases(oracle_mod, basis):
    mods = catalogue(oracle_mod)[basis]
    K, log_n = 2, 12
    o, oq = _contexts(oracle_mod, log_n, K, len(mods) - K, mods)
    evk = o.fill_uniform(700, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    for n_terms in (9, 17, 64):
        n_pool = 6
        pool = _pool(oq, n_pool, 2, 710 + n_terms)
        ia, ib = _pairs(n_terms, n_pool)
        want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], evk, 65537)
        for variant in _variants(mods):
            assert np.array_equal(EmuDot(log_n, mods, variant).ct_dot(K, pool, ia, ib, evk, 65537), want), (variant, n_terms)


# ---- the lazy bound ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("which", ["largest_60", "smallest_34", "default"])
def test_lazy_bound_at_its_limit(oracle_mod, which):
    """64 pairs of q - 1 (and of 0, and mixed) words: the sums are the exact integers mod q, every 128-bit running sum stays below
    2^(2b+4) and every folded value below 15q < 2^64"""
    log_n = 12
    if which == "default":
        moduli = oracle_mod.Oracle(log_n, 2).moduli
    else:
        moduli = [LARGEST_GENERIC if which == "largest_60" else SMALLEST_GENERIC, catalogue(oracle_mod)["gen_mixed"][0]]
    N, Lq = 1 << log_n, 2
    q = [int(x) for x in moduli]
    qa = np.array(q, dtype=np.uint64)
    top = np.broadcast_to((qa - 1)[None, None, :, None], (1, 2, Lq, N)).copy()
    zero = np.zeros_like(top)
    mixed = top.copy()
    mixed[0, :, :, 1::2] = 0
    mixed[0, 1, :, ::4] = 1
    pool = np.stack([top, zero, mixed])
    for variant in _variants(moduli):
        e = EmuDot(log_n, moduli, variant)
        e.track()
        for n in (64, 17, 16, 8):
            for ia, ib in (([0] * n, [0] * n), ([1] * n, [0] * n), ([2] * n, [0] * n), ([0, 2] * (n // 2) + [0] * (n % 2), [2] * n)):
                got = e.sums(pool, ia, ib)
                for l in range(Lq):
                    assert (got[:, l] < np.uint64(15 * q[l])).all()
                    for c in (0, 1, 2, 4):
                        a = [[int(pool[i, 0, k, l, c]) for k in range(2)] for i in ia]
                        b = [[int(pool[i, 0, k, l, c]) for k in range(2)] for i in ib]
                        want = [sum(x[0] * y[0] for x, y in zip(a, b)), sum(x[0] * y[1] + x[1] * y[0] for x, y in zip(a, b)),
                                sum(x[1] * y[1] for x, y in zip(a, b))]
                        assert [int(got[k, l, c]) % q[l] for k in range(3)] == [w % q[l] for w in want], (variant, n, l, c)
        sum_max, red_max = e.track()
        assert 0 < sum_max < 16.0 and 0 < red_max < 15.0, (sum_max, red_max)
        if which != "smallest_34":   # moduli just below a power of two come close to the precondition's limit
            assert sum_max > 15.0, sum_max
