"""The host build of the scalar arithmetic (modarith.cuh) and of the register-level transform pieces (ntt_core.cuh) through the
element-wise harness tests/devarith/devarith.cu, against exact integers and against the emulator the rest of the CPU suite runs.

tests/test_gpu_devarith.py then compares the device build with this host build word for word, so that DESIGN.md §3's claim, that
the host arithmetic computes the device's lazy values, is tested rather than assumed.  This file needs nvcc but no GPU: building
the two libraries is also the sm_90a cross-compile of the harness's device code."""
import os
import sys

import numpy as np
import pytest

import arith_cases as ac

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devarith"))
import harness  # noqa: E402

CONFIGS = ac.configs()
IDS = [c[0] for c in CONFIGS]
N_SUB = 3000          # random cases per op and modulus checked with Python integers (all of them run)
N_SUB_16 = 200


@pytest.fixture(scope="module")
def arith():
    cache = {}

    def get(cid):
        if cid not in cache:
            _, variant, mods, ts = CONFIGS[IDS.index(cid)]
            cache[cid] = harness.DevArith(variant, mods, ts)
        return cache[cid]
    return get


def test_harness_builds_for_sm90a():
    paths = harness.build()
    assert [os.path.basename(p) for p in paths] == ["libdpfhe_devarith_gen.so", "libdpfhe_devarith_fast.so"]
    for v in harness.VARIANTS:
        lib = harness.load(v)
        assert lib.devarith_fast() == (v == "fast")
        with open(harness.so_path(v), "rb") as f:
            assert b"sm_90a" in f.read(), "no sm_90a code object in %s" % v


def test_constants_match_exact_integers(arith):
    """the limb constants and Mod32 the harness gets from the product's host code are what their comments say"""
    for cid, _, mods, ts in CONFIGS:
        da = arith(cid)
        for l, q in enumerate(mods):
            lp = da.limb_params(l)
            b = q.bit_length()
            assert (lp["q"], lp["q2"], lp["qsb"], lp["q8"], lp["nq"]) == (q, 2 * q, ac.SB * q, 8 * q, ac.M64 - q)
            assert lp["bar_shift"] == b - 2 and lp["bar_mu"] == (1 << (b - 2 + 64)) // q and lp["mu32"] == ac.M64 // q
            assert lp["nqh"] == ((-(q >> 32)) % ac.M32 if ac.bases.is_fast(q) else 0)
        for k, t in enumerate(ts):
            r32 = ac.M32 % t
            assert da.mod32(k) == {"t": t, "r32": r32, "r32_s": (r32 << 32) // t, "one_s": ac.M32 // t}


def _fail_msg(cid, op, idx, bad):
    i, o, e = bad[0]
    return "%s %s [%d]: input %s -> output %s: %s (%d such cases shown)" % (cid, op, idx, [hex(v) for v in i], [hex(v) for v in o], e, len(bad))


def host_cases(da, cid, idx, q, lp, op, seed):
    """structured + N_RANDOM uniform cases, their host outputs, and the Python-checked subsample"""
    rng = np.random.default_rng(seed)
    s = ac.structured(op, q, lp, rng)
    r = ac.uniform(op, q, lp, rng, ac.N_RANDOM_16 if op in ac.TRANSFORM16 else ac.N_RANDOM)
    return s, r, da.host(op, idx, s), da.host(op, idx, r)


# corners the cases must reach on every modulus (measured on the host build first; see each comment)
REQUIRED = {
    "mulhi_approx": {"short_by_2"},                 # the estimate exactly two short
    "shoup_lazy": {"band_3"},                       # [3q, 4q): the whole of [0, SB q)
    "shoup_exact": {"band_1"},
    "gs_bfly": {"band_3"},
    "ct_bfly": {"band_3"},                          # the Shoup product inside the butterfly in [3q, 4q)
    "inv16": {"band_3"},
    # [0, 3q) is the documented range, but an exhaustive scan over every high word (the quotient estimate depends on nothing
    # else) shows [2q, 3q) unreachable for the smallest generic, the smallest fast and the largest 60-bit modulus: the three
    # truncations of the estimate never add up to 2
    "word_reduce": {"band_1"},
    "pti_fold": {"band_1"},
    "csub": {"kept", "low_word_borrow"},
}


def reached_ok(op, got, cid, lp):
    """what the measurement shows reachable beyond REQUIRED: the lazy products with estimates and the forward passes"""
    if op in REQUIRED:
        return REQUIRED[op] <= got
    top = max([int(b.split("_")[1]) for b in got if b.startswith("band_")] or [-1])
    if op in ac.FWD16:
        return top >= ac.fwd_bound_after(int(op.split("_")[1]), 4) - 2   # within 2q of the pass's bound
    if op in ("barrett_lazy", "mulmod_lazy"):
        return top >= (1 if cid == "gen-largest" else 2)   # [2q, 3q): one more q than an exact quotient gives canonical factors
    if op == "barrett_lazy_long":
        return top >= 4
    return True


@pytest.mark.parametrize("cid", IDS)
def test_host_build_exact(arith, cid):
    """every op on every modulus of the configuration: congruent, inside its documented range, exact where it must be, and
    the cases reach the corners those ranges are about"""
    da = arith(cid)
    _, _, mods, ts = CONFIGS[IDS.index(cid)]
    for l, q in enumerate(mods):
        lp = da.limb_params(l)
        for op in ac.ops_for(lp, False):
            s, r, hs, hr = host_cases(da, cid, l, q, lp, op, seed=ac.seed_of(cid, q, op))
            n_sub = N_SUB_16 if op in ac.TRANSFORM16 else N_SUB
            bad = ac.check(op, q, lp, s, hs) or ac.check(op, q, lp, r[:n_sub], hr[:n_sub])
            assert not bad, _fail_msg(cid, op, l, bad)
            sub = ac.corners(op, q, np.concatenate([s, r[:n_sub]]), np.concatenate([hs, hr[:n_sub]]))
            full = sub if op == "mulhi_approx" else ac.corners(op, q, np.concatenate([s, r]), np.concatenate([hs, hr]))
            assert reached_ok(op, full, cid, lp), "%s %s [%d]: the cases reach only %s" % (cid, op, l, sorted(full))
    for k, t in enumerate(ts):
        for op in ac.U32_OPS:
            s, r, hs, hr = host_cases(da, cid, k, t, None, op, seed=ac.seed_of(cid, t, op))
            bad = ac.check(op, t, None, s, hs) or ac.check(op, t, None, r[:N_SUB], hr[:N_SUB])
            assert not bad, _fail_msg(cid, op, k, bad)
            if op == "reduce64_32":
                assert "x=2^64-1" in ac.corners(op, t, s, hs)
            if op == "shoup32":   # canonical output for any 32-bit multiplicand, over all of them
                assert int(hr[:, 0].max()) < t and np.any(r[:, 0] >= np.uint64(2 * t))


# the harness op and the emulator export (tests/emu/emu.cpp) that compute the same thing, with the emulator's arguments
EMU_OPS = {
    "mulmod": ("mulmod", lambda i: i), "word_reduce": ("word_reduce", lambda i: i), "canon": ("canon", lambda i: i),
    "canon_store": ("canon_store", lambda i: i), "mulmod_lazy": ("mulmod_lazy", lambda i: i),
    "barrett_lazy_long": ("barrett_long", lambda i: i), "pti_fold": ("pti_fold", lambda i: i),
    "shoup_lazy": ("shoup_lazy", lambda i: i[:2]), "shoup_exact": ("shoup_exact", lambda i: i[:2]),
}


@pytest.mark.parametrize("cid", IDS)
def test_host_build_is_the_emulators_arithmetic(arith, make_emu, cid):
    """the harness's host build computes, word for word, what the emulator the CPU suite trusts computes"""
    da = arith(cid)
    _, variant, mods, _ = CONFIGS[IDS.index(cid)]
    e = make_emu(12, len(mods), mods, variant=variant)
    assert e.moduli == mods
    for l, q in enumerate(mods):
        lp = da.limb_params(l)
        for op, (emu_op, args) in EMU_OPS.items():
            rng = np.random.default_rng(7)
            x = np.concatenate([ac.structured(op, q, lp, rng), ac.uniform(op, q, lp, rng, 500)])
            got = da.host(op, l, x)[:, 0].tolist()
            want = [e.scalar(emu_op, l, *args(i)) for i in x.tolist()]
            diff = [k for k in range(len(want)) if got[k] != want[k]]
            assert not diff, "%s %s [%d]: input %s: harness %d, emulator %d" % (cid, op, l, x[diff[0]].tolist(), got[diff[0]], want[diff[0]])
