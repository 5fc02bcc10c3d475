"""Calls at level l on the top-level context (DESIGN.md sections 2.20 / 4.17): every *_level entry point, bit for bit against the same
call on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the key restricted to that basis (tests/polyeval_ref.py:restrict_key),
over K = 1 .. 4, every valid level with ragged last digits, every ring degree, the moduli bases of tests/bases.py and three plaintext
moduli; aliasing, several grid rounds, restarting round numbers, level calls interleaved with top-level calls on one and two streams,
the host forms, the argument checks, the launch count and the level state's device memory; and x -> x^8 decrypted on ONE context
with ONE key in BGV and CKKS, a rotation sum at level Lq - 1 and the C++ example."""
import os
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ckks_polyeval_ref as cr  # noqa: E402
import polyeval_ref as pr  # noqa: E402
from bases import catalogue  # noqa: E402
from test_gpu_parity import dev, dp, host  # noqa: E402,F401  (dp is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_BGV = 167772161
GALOIS = [pow(5, k, 1 << 13) for k in range(1, 16)]   # odd, below 2N for every N here


@pytest.fixture(scope="module", autouse=True)
def _release_cached_blocks():
    """the library allocates with cudaMalloc, which cannot use blocks torch keeps cached: hand this module's back when it is done"""
    yield
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def _oracles(oracle_mod):
    cache = {}

    def get(log_n, L, moduli=None):
        key = (log_n, L, tuple(moduli) if moduli else None)
        if key not in cache:
            cache[key] = oracle_mod.Oracle(log_n, L, moduli)
        return cache[key]

    return get


@pytest.fixture
def ctxs(dp, _oracles):
    """(context, oracle) by (log N, L, moduli), as test_gpu_parity's fixture, but the contexts live for one test only: each holds a few
    hundred MiB of key-switch scratch at N = 8192 and more at 16384, and this module makes one per level of many bases, on a device
    that other work shares"""
    made = {}
    torch.cuda.empty_cache()   # blocks torch still caches for earlier tests are out of reach of the library's cudaMalloc

    def get(log_n, L, moduli=None):
        key = (log_n, L, tuple(moduli) if moduli else None)
        if key not in made:
            made[key] = dp.Context(log_n, L, moduli)
        return made[key], _oracles(log_n, L, moduli)

    yield get
    for c in made.values():
        c.close()
    torch.cuda.empty_cache()


def _uniform(rng, mods, shape):
    """canonical residues [..., len(mods), N] (the limb axis second to last)"""
    out = np.empty(shape, dtype=np.uint64)
    for i, q in enumerate(mods):
        out[..., i, :] = rng.integers(0, int(q), size=out[..., i, :].shape, dtype=np.uint64)
    return out


class Level:
    """the top-level context c over L limbs (K special) and the level context cl over {q_0 .. q_{l-1}, p_0 .. p_{K-1}}"""

    def __init__(self, ctxs, log_n, L, K, l, moduli=None):
        self.c, o = ctxs(log_n, L, moduli)
        self.mods = [int(q) for q in o.moduli]
        self.K, self.l, self.Lq, self.L, self.N = K, l, L - K, L, o.N
        self.cl, _ = ctxs(log_n, l + K, self.mods[:l] + self.mods[L - K:])
        self.dnum = self.c.grouped_digits(K)

    def cts(self, rng, n, batch):
        return _uniform(rng, self.mods[:self.l], (n, batch, 2, self.l, self.N))

    def keys(self, rng, n):
        """n top-level keys [dnum][2][L][N] and their restrictions to the level"""
        top = _uniform(rng, self.mods, (n, self.dnum, 2, self.L, self.N))
        return top, [pr.restrict_key(k, self.Lq, self.K, self.l) for k in top]

    def out(self, batch, drop=0):
        return torch.full((batch, 2, self.l - drop, self.N), -1, dtype=torch.int64, device="cuda")


def _check_all(v, rng, batch, t, n_dot=9, n_rot=1, calls=("mul", "rot", "dot", "mul_rs", "dot_rs", "rot_sum")):
    """every level call against the level context's call; at l = Lq also against the top-level call itself"""
    K, l, c, cl = v.K, v.l, v.c, v.cl
    pool = [dev(x) for x in v.cts(rng, max(2, n_dot), batch)]
    top, low = v.keys(rng, max(1, n_rot))
    dtop, dlow = [dev(k) for k in top], [dev(k) for k in low]
    ia = [k % len(pool) for k in range(n_dot)]
    ib = [(k + 1) % len(pool) for k in range(n_dot)]
    rescale_ok = l >= 2 and t < v.mods[l - 1]
    top_level = l == v.Lq
    for name in calls:
        if name in ("mul_rs", "dot_rs") and not rescale_ok:
            continue
        drop = 1 if name.endswith("_rs") else 0
        got, want = v.out(batch, drop), v.out(batch, drop)
        if name == "mul":
            c.ct_mul_relin_grouped_level(K, l, pool[0], pool[1], dtop[0], got, batch, t)
            cl.ct_mul_relin_grouped(K, pool[0], pool[1], dlow[0], want, batch, t)
        elif name == "rot":
            c.rotate_grouped_level(K, l, pool[0], GALOIS[0], dtop[0], got, batch, t)
            cl.rotate_grouped(K, pool[0], GALOIS[0], dlow[0], want, batch, t)
        elif name == "dot":
            c.ct_dot_grouped_level(K, l, [pool[i] for i in ia], [pool[i] for i in ib], dtop[0], got, batch, t)
            cl.ct_dot_grouped(K, [pool[i] for i in ia], [pool[i] for i in ib], dlow[0], want, batch, t)
        elif name == "mul_rs":
            c.ct_mul_relin_rescale_grouped_level(K, l, pool[0], pool[1], dtop[0], got, batch, t)
            cl.ct_mul_relin_rescale_grouped(K, pool[0], pool[1], dlow[0], want, batch, t)
        elif name == "dot_rs":
            c.ct_dot_rescale_grouped_level(K, l, [pool[i] for i in ia], [pool[i] for i in ib], dtop[0], got, batch, t)
            cl.ct_dot_rescale_grouped(K, [pool[i] for i in ia], [pool[i] for i in ib], dlow[0], want, batch, t)
        else:
            c.rotate_sum_grouped_level(K, l, pool[0], GALOIS[:n_rot], dtop[:n_rot], got, batch, t)
            cl.rotate_sum_grouped(K, pool[0], GALOIS[:n_rot], dlow[:n_rot], want, batch, t)
        torch.cuda.synchronize()
        assert torch.equal(got, want), (name, l)
        assert bool((got != -1).any()), name
        if top_level:   # l = Lq: the context's own call, bit for bit
            same = v.out(batch, drop)
            if name == "mul":
                c.ct_mul_relin_grouped(K, pool[0], pool[1], dtop[0], same, batch, t)
            elif name == "rot":
                c.rotate_grouped(K, pool[0], GALOIS[0], dtop[0], same, batch, t)
            elif name == "dot":
                c.ct_dot_grouped(K, [pool[i] for i in ia], [pool[i] for i in ib], dtop[0], same, batch, t)
            elif name == "mul_rs":
                c.ct_mul_relin_rescale_grouped(K, pool[0], pool[1], dtop[0], same, batch, t)
            elif name == "dot_rs":
                c.ct_dot_rescale_grouped(K, [pool[i] for i in ia], [pool[i] for i in ib], dtop[0], same, batch, t)
            else:
                c.rotate_sum_grouped(K, pool[0], GALOIS[:n_rot], dtop[:n_rot], same, batch, t)
            assert torch.equal(got, same), name


# (log N, L, K): K = 1 .. 4, ragged last digits (K = 2, Lq = 7; K = 3, Lq = 7; K = 4, Lq = 6), every ring degree
SHAPES = [(12, 3, 1), (12, 5, 1), (12, 6, 2), (12, 9, 2), (12, 10, 3), (12, 10, 4), (13, 6, 2), (13, 8, 3), (14, 6, 2), (14, 5, 1)]


def _levels(L, K):
    return list(range(K, L - K + 1))


@pytest.mark.parametrize("log_n,L,K,l", [(n, L, K, l) for n, L, K in SHAPES for l in _levels(L, K)])
def test_every_level_against_level_context(ctxs, log_n, L, K, l):
    v = Level(ctxs, log_n, L, K, l)
    rng = np.random.default_rng(1000 * log_n + 100 * L + 10 * K + l)
    _check_all(v, rng, 3, [0, 65537, T_BGV][(L + l) % 3])


@pytest.mark.parametrize("n_dot,n_rot", [(1, 1), (64, 15)])
def test_pairs_and_rotations(ctxs, n_dot, n_rot):
    """1 and 64 pairs, 1 and 15 summed rotations, at a ragged level"""
    v = Level(ctxs, 13, 9, 2, 5)
    _check_all(v, np.random.default_rng(7 + n_dot), 2, 65537, n_dot=n_dot, n_rot=n_rot, calls=("dot", "dot_rs", "rot_sum"))


@pytest.mark.parametrize("t", [0, 65537, T_BGV])
@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_bases_and_plain_moduli(ctxs, oracle_mod, basis, t):
    mods = catalogue(oracle_mod)[basis][:7]
    v = Level(ctxs, 12, len(mods), 2, 3, mods)
    _check_all(v, np.random.default_rng(sum(map(ord, basis)) + t % 97), 2, t)


@pytest.mark.parametrize("log_n", [13, 14])
def test_generic_arithmetic_at_larger_degrees(ctxs, oracle_mod, log_n):
    """the generic-arithmetic instances at N = 8192 and 16384 (the default basis selects the fast ones)"""
    mods = catalogue(oracle_mod)["gen_mixed"][:7]
    for K, l in ((1, 3), (2, 3)):
        v = Level(ctxs, log_n, len(mods), K, l, mods)
        _check_all(v, np.random.default_rng(log_n + K), 2, T_BGV)


def test_aliased_operands(ctxs):
    """a and b the same buffer (a square), a buffer in several pairs"""
    v = Level(ctxs, 12, 7, 2, 3)
    K, l, c, cl, batch = v.K, v.l, v.c, v.cl, 3
    rng = np.random.default_rng(5)
    a = dev(v.cts(rng, 1, batch)[0])
    top, low = v.keys(rng, 1)
    dtop, dlow = dev(top[0]), dev(low[0])
    for f_lvl, f_ref, drop in ((c.ct_mul_relin_grouped_level, cl.ct_mul_relin_grouped, 0),
                               (c.ct_mul_relin_rescale_grouped_level, cl.ct_mul_relin_rescale_grouped, 1)):
        got, want = v.out(batch, drop), v.out(batch, drop)
        f_lvl(K, l, a, a, dtop, got, batch, 65537)
        f_ref(K, a, a, dlow, want, batch, 65537)
        assert torch.equal(got, want)
    got, want = v.out(batch), v.out(batch)
    c.ct_dot_grouped_level(K, l, [a, a, a], [a, a, a], dtop, got, batch, 0)
    cl.ct_dot_grouped(K, [a, a, a], [a, a, a], dlow, want, batch, 0)
    assert torch.equal(got, want)


def _fresh(dp, monkeypatch, env, log_n, L):
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    c = dp.Context(log_n, L)
    for k in env:
        monkeypatch.delenv(k)
    return c


@pytest.mark.parametrize("rounds_extra", [0, 1])
def test_grid_rounds(dp, ctxs, monkeypatch, rounds_extra):
    """one CTA per SM: a batch of exactly three grid rounds of the level's groups, and one past them"""
    L, K, l, log_n = 7, 2, 3, 12
    c = _fresh(dp, monkeypatch, {"DPFHE_KS_OCC": "1"}, log_n, L)
    v = Level(ctxs, log_n, L, K, l)
    v.c = c
    batch = 3 * (torch.cuda.get_device_properties(0).multi_processor_count // (l + K)) + rounds_extra
    _check_all(v, np.random.default_rng(50 + rounds_extra), batch, 65537, n_dot=3, calls=("mul", "dot_rs", "rot"))
    c.close()


def test_round_numbering_restarts(dp, ctxs, monkeypatch):
    """round numbers that restart inside a sequence of level and top-level calls keep the bits"""
    L, K, log_n = 7, 2, 12
    c = _fresh(dp, monkeypatch, {"DPFHE_EPOCH_LIMIT": "40"}, log_n, L)
    for rep in range(4):   # ~10 rounds per launch against a limit of 40
        for l in (3, 5):
            v = Level(ctxs, log_n, L, K, l)
            v.c = c
            _check_all(v, np.random.default_rng(60 + l), 9, 65537, n_dot=2, calls=("mul", "mul_rs") if rep % 2 else ("dot", "rot"))
    c.close()


@pytest.mark.parametrize("two_streams", [False, True])
def test_interleaved_with_top_level_calls(ctxs, two_streams):
    """level calls between top-level calls on the same context, on one stream or alternating between two: every result is the bits
    of the call made alone (the context orders its calls across streams)"""
    L, K, log_n, batch = 7, 2, 13, 4
    top_v, lvl_v = Level(ctxs, log_n, L, K, L - K), Level(ctxs, log_n, L, K, 3)
    c = top_v.c
    rng = np.random.default_rng(70)
    top_ct, lvl_ct = dev(top_v.cts(rng, 1, batch)[0]), dev(lvl_v.cts(rng, 1, batch)[0])
    key, low = lvl_v.keys(rng, 1)
    dkey, dlow = dev(key[0]), dev(low[0])
    want_top, want_lvl = top_v.out(batch), lvl_v.out(batch, 1)
    c.ct_mul_relin_grouped(K, top_ct, top_ct, dkey, want_top, batch, 65537)
    lvl_v.cl.ct_mul_relin_rescale_grouped(K, lvl_ct, lvl_ct, dlow, want_lvl, batch, 65537)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()] if two_streams else [torch.cuda.current_stream()] * 2
    outs = []
    for k in range(6):
        st = streams[k % 2]
        with torch.cuda.stream(st):
            o_top, o_lvl = top_v.out(batch), lvl_v.out(batch, 1)
        c.ct_mul_relin_grouped(K, top_ct, top_ct, dkey, o_top, batch, 65537, stream=st.cuda_stream)
        c.ct_mul_relin_rescale_grouped_level(K, 3, lvl_ct, lvl_ct, dkey, o_lvl, batch, 65537, stream=streams[(k + 1) % 2].cuda_stream)
        outs.append((o_top, o_lvl))
    torch.cuda.synchronize()
    for o_top, o_lvl in outs:
        assert torch.equal(o_top, want_top) and torch.equal(o_lvl, want_lvl)


def test_host_forms_over_several_chunks(ctxs):
    v = Level(ctxs, 12, 7, 2, 3)
    K, l, c, cl, batch, n_terms = v.K, v.l, v.c, v.cl, 700, 3   # the host forms split the batch into several chunks
    rng = np.random.default_rng(80)
    a, b = v.cts(rng, n_terms, batch), v.cts(rng, n_terms, batch)
    top, low = v.keys(rng, 1)
    h_out = np.zeros((batch, 2, l - 1, v.N), dtype=np.uint64)
    want = v.out(batch, 1)
    c.ct_mul_relin_rescale_grouped_level_host(K, l, a[0], b[0], top[0], h_out, 65537)
    cl.ct_mul_relin_rescale_grouped(K, dev(a[0]), dev(b[0]), dev(low[0]), want, batch, 65537)
    assert np.array_equal(h_out, host(want).reshape(h_out.shape))
    c.ct_dot_rescale_grouped_level_host(K, l, a, b, top[0], h_out, 0)
    cl.ct_dot_rescale_grouped(K, [dev(x) for x in a], [dev(x) for x in b], dev(low[0]), want, batch, 0)
    assert np.array_equal(h_out, host(want).reshape(h_out.shape))


def test_checks_launches_and_device_bytes(dp, oracle_mod):
    L, K, log_n, batch = 7, 2, 12, 2
    c = dp.Context(log_n, L)
    o = oracle_mod.Oracle(log_n, L)
    mods = [int(q) for q in o.moduli]
    Lq, N = L - K, o.N
    rng = np.random.default_rng(90)
    key = dev(_uniform(rng, mods, (c.grouped_digits(K), 2, L, N)))
    a3 = dev(_uniform(rng, mods[:3], (batch, 2, 3, N)))
    # launch count: a level call launches what the top-level call launches (companions + kernel; rotation sums 1 + 4)
    top = dev(_uniform(rng, mods[:Lq], (batch, 2, Lq, N)))
    o_top = torch.empty((batch, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.ct_mul_relin_grouped(K, top, top, key, o_top, batch, 0)
    c.ct_mul_relin_rescale_grouped(K, top, top, key, o_top[:, :, :Lq - 1].contiguous(), batch, 0)
    c.rotate_sum_grouped(K, top, GALOIS[:1], [key], o_top, batch, 0)
    torch.cuda.synchronize()
    bytes0 = c.device_bytes()
    o3, o2 = torch.empty((batch, 2, 3, N), dtype=torch.int64, device="cuda"), torch.empty((batch, 2, 2, N), dtype=torch.int64, device="cuda")
    calls = [(lambda: c.ct_mul_relin_grouped_level(K, 3, a3, a3, key, o3, batch, 0), 2),
             (lambda: c.rotate_grouped_level(K, 3, a3, GALOIS[0], key, o3, batch, 0), 2),
             (lambda: c.ct_dot_grouped_level(K, 3, [a3, a3], [a3, a3], key, o3, batch, 0), 2),
             (lambda: c.ct_mul_relin_rescale_grouped_level(K, 3, a3, a3, key, o2, batch, 0), 2),
             (lambda: c.ct_dot_rescale_grouped_level(K, 3, [a3], [a3], key, o2, batch, 0), 2),
             (lambda: c.rotate_sum_grouped_level(K, 3, a3, GALOIS[:1], [key], o3, batch, 0), 5)]
    for k, (call, n) in enumerate(calls):
        n0 = c.launch_count()
        call()
        torch.cuda.synchronize()
        assert c.launch_count() - n0 == n, k
    bytes1 = c.device_bytes()
    # the level's tables (and nothing else) were added: less than one restricted key with its companions
    grown = bytes1 - bytes0
    restricted = 2 * (-(-3 // K)) * 2 * (3 + K) * N * 8
    assert 0 < grown < restricted, (grown, restricted)
    for call, _ in calls:   # repeat calls allocate nothing
        call()
    torch.cuda.synchronize()
    assert c.device_bytes() == bytes1
    c.ct_mul_relin_grouped_level(K, 4, top[:, :, :4].contiguous(), top[:, :, :4].contiguous(), key,
                                 torch.empty((batch, 2, 4, N), dtype=torch.int64, device="cuda"), batch, 0)
    torch.cuda.synchronize()
    assert c.device_bytes() - bytes1 > 0   # a second level: its own tables
    c._chk(c._l.dpfhe_context_trim(c._h))
    after = c.device_bytes()
    c.ct_mul_relin_grouped_level(K, 3, a3, a3, key, o3, batch, 0)   # rebuilt on demand
    torch.cuda.synchronize()
    assert c.device_bytes() - after == grown
    # rejected calls leave the output untouched and name the level
    mark = torch.full((batch, 2, 3, N), -7, dtype=torch.int64, device="cuda")
    mark2 = torch.full((batch, 2, 2, N), -7, dtype=torch.int64, device="cuda")
    a1 = dev(_uniform(rng, mods[:1], (batch, 2, 1, N)))
    asc = sorted(mods)   # ascending: q_2 is below the special primes, so only the level's own check refuses t = q_2
    cs = dp.Context(log_n, L, asc)
    bad = [
        (lambda: c.ct_mul_relin_grouped_level(K, 1, a1, a1, key, mark, batch, 0), "level 1"),                  # below K
        (lambda: c.ct_mul_relin_grouped_level(K, Lq + 1, a3, a3, key, mark, batch, 0), "level %d" % (Lq + 1)),  # above Lq
        (lambda: c.rotate_sum_grouped_level(K, 1, a1, GALOIS[:1], [key], mark, batch, 0), "level 1"),
        (lambda: c.ct_dot_rescale_grouped_level(K, Lq + 1, [a3], [a3], key, mark2, batch, 0), "level %d" % (Lq + 1)),
        (lambda: cs.ct_mul_relin_rescale_grouped_level(K, 3, a3, a3, key, mark2, batch, asc[2]), "level 3"),     # special primes > t >= q_{l-1}
        (lambda: c.ct_mul_relin_grouped_level(K, 3, a3, a3, key, mark, batch, mods[-1]), None),                 # t >= a special prime
        (lambda: c.ct_mul_relin_grouped_level(K, 3, mark, a3, key, mark, batch, 0), None),                      # output overlaps an input
    ]
    for k, (call, msg) in enumerate(bad):
        with pytest.raises(dp.DpfheError) as e:
            call()
        if msg:
            assert msg in str(e.value), (k, str(e.value))
        assert bool((mark == -7).all()) and bool((mark2 == -7).all()), k
    cs.close()
    c1 = dp.Context(log_n, 3)   # K = 1, Lq = 2: the rescale at level 1 is refused by the level check
    k1 = dev(_uniform(rng, [int(q) for q in oracle_mod.Oracle(log_n, 3).moduli], (2, 2, 3, N)))
    m1 = torch.full((batch, 2, 1, N), -7, dtype=torch.int64, device="cuda")
    with pytest.raises(dp.DpfheError) as e:
        c1.ct_mul_relin_rescale_grouped_level(1, 1, a1, a1, k1, m1, batch, 0)
    assert "level 1" in str(e.value) and bool((m1 == -7).all())
    c1.close()
    n0 = c.launch_count()   # an empty batch is fine and launches nothing
    c.ct_mul_relin_grouped_level(K, 3, a3, a3, key, mark, 0, 0)
    c.ct_dot_rescale_grouped_level(K, 3, [a3], [a3], key, mark2, 0, 0)
    c.rotate_sum_grouped_level(K, 3, a3, GALOIS[:1], [key], mark, 0, 0)
    assert c.launch_count() == n0 and bool((mark == -7).all())
    c.close()


# ---- decryption chains on ONE context -------------------------------------------------------------------------------------------
SEED = bytes(range(40, 72))


def _keys(c, K, t):
    L, N = c.L, c.N
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    c.generate_secret(SEED, sk)
    evk = torch.empty((c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_relin_key(K, t, sk, bytes(range(1, 33)), evk)
    return sk, evk


def test_bgv_power_chain_and_rotation_sum(ctxs):
    """x -> x^2 -> x^4 -> x^8 down to l = Lq - 3 with one context and one key, slot for slot with the factors q_l^-1 mod t; then a
    rotation sum at level Lq - 1 decrypts to the slots of x^2 plus those of its rotation"""
    K, L, log_n, t = 2, 7, 13, T_BGV
    c, o = ctxs(log_n, L)
    mods = [int(q) for q in o.moduli]
    N, Lq, B = c.N, L - K, 2
    sk, evk = _keys(c, K, t)
    prefix = {l: ctxs(log_n, l, mods[:l])[0] for l in range(Lq - 3, Lq + 1)}
    rng = np.random.default_rng(21)
    x = rng.integers(-50, 50, size=(B, N), dtype=np.int64)
    pts = torch.empty((B, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].bgv_encode(torch.from_numpy(x).cuda(), pts, B, t)
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].encrypt(t, sk[:Lq].contiguous(), SEED, 0, pts, ct, B)

    def slots(ct):
        low = prefix[ct.shape[2]]
        ph = torch.empty((ct.shape[0], low.L, N), dtype=torch.int64, device="cuda")
        low.decrypt(sk[:low.L].contiguous(), ct.contiguous(), 2, ph, ct.shape[0])
        s = torch.empty((ct.shape[0], N), dtype=torch.int64, device="cuda")
        low.bgv_decode(ph, s, ct.shape[0], t)
        return host(s).astype(object)

    want = x.astype(object) % t
    levels = []
    for l in (Lq, Lq - 1, Lq - 2):
        sq = torch.empty((B, 2, l - 1, N), dtype=torch.int64, device="cuda")
        c.ct_mul_relin_rescale_grouped_level(K, l, ct, ct, evk, sq, B, t)
        ct = sq
        want = want * want * pow(mods[l - 1], -1, t) % t
        assert np.array_equal(slots(ct), want), l
        levels.append(sq)
    # the rotation sum at Lq - 1 (on x^2) against the level's single rotation and the ciphertext itself
    gk = torch.empty((c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, t, sk, [GALOIS[0]], bytes(range(2, 34)), gk)
    x2 = levels[0]
    rs, rot = torch.empty_like(x2), torch.empty_like(x2)
    c.rotate_sum_grouped_level(K, Lq - 1, x2, GALOIS[:1], [gk], rs, B, t)
    c.rotate_grouped_level(K, Lq - 1, x2, GALOIS[0], gk, rot, B, t)
    assert np.array_equal(slots(rs), (slots(x2) + slots(rot)) % t)
    assert not np.array_equal(slots(rot), slots(x2))


def test_ckks_power_chain(oracle_mod):
    """x^8 in CKKS with one context and one key; DESIGN.md section 2.20 records the measured errors"""
    import deeppowers_b200
    K, Lq, log_n = 2, 5, 13
    mods = cr.ckks_chain(oracle_mod, Lq, K)
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    prefix = {l: deeppowers_b200.Context(log_n, l, mods[:l]) for l in (Lq, Lq - 3)}
    N, B = c.N, 2
    sk, evk = _keys(c, K, 0)
    rng = np.random.default_rng(22)
    z = rng.uniform(-1, 1, (B, N // 2)) + 1j * rng.uniform(-1, 1, (B, N // 2))
    scale = float(mods[1])
    pts = torch.empty((B, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].ckks_encode(torch.from_numpy(z).cuda(), pts, B, scale)
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].encrypt(0, sk[:Lq].contiguous(), SEED, 0, pts, ct, B)
    for l in (Lq, Lq - 1, Lq - 2):
        sq = torch.empty((B, 2, l - 1, N), dtype=torch.int64, device="cuda")
        c.ct_mul_relin_rescale_grouped_level(K, l, ct, ct, evk, sq, B, 0)
        ct = sq
        scale = scale * scale / mods[l - 1]
    low = prefix[Lq - 3]
    ph = torch.empty((B, low.L, N), dtype=torch.int64, device="cuda")
    low.decrypt(sk[:low.L].contiguous(), ct.contiguous(), 2, ph, B)
    out = torch.empty((B, N // 2), dtype=torch.complex128, device="cuda")
    low.ckks_decode(ph, out, B, scale)
    err = np.abs(out.cpu().numpy() - z ** 8).max()
    print("CKKS x^8 on one context: scale 2^%.2f, error 2^%.2f" % (np.log2(scale), np.log2(err)))
    assert err < 2.0**-20
    for x in [c] + list(prefix.values()):
        x.close()


def test_cpp_example(tmp_path):
    """examples/encrypted_power_chain.cpp against libdpfhe.so alone: x^8 with one evaluator and one key within its bound"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    libdir = os.path.join(ROOT, "deeppowers_b200")
    exe = str(tmp_path / "encrypted_power_chain")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "encrypted_power_chain.cpp"),
                           "-L", libdir, "-ldpfhe", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "one evaluator and one key" in r.stdout
