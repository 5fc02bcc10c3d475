"""The persistent key-switch kernels at N = 16384 (DESIGN.md §4.4, "N = 16384": one limb per CTA in two halves, 64 KiB of shared
memory, three CTAs per SM, accumulator rows in scratch owned by the CTA's slot) on the GPU, bit for bit against the oracle, over
three and more grid rounds and on the boundaries of the grid's groups and rounds:

1. the fused kernel in every mode (ct x ct, bare key switch, rotation, conjugation) for L = 1, 2, 4, 5, 8 and 16, on the default
   grid and under DPFHE_KS_OCC=1;
2. the same with single-buffered digit slots (DPFHE_KS_SINGLE=1), the hoisted-rotation fallback (the fused kernel's FILTER instance)
   in one and in several chunks, one context driven through launches of different grids with and without restarts of the round
   numbering, and fused launches interleaved with the other persistent kernels, which share the digit slots;
3. the tuning switches DPFHE_KS_PF, DPFHE_KS_OCC, DPFHE_KS_PROF, DPFHE_FORCE_GENERIC and a generic basis;
4. the hybrid, grouped, multiply-and-rescale, inner-product, hoisting and level kernels.

The tests cannot read the occupancy the runtime picks.  Cases under DPFHE_KS_OCC=1 therefore pin the grid exactly (one CTA per SM
whenever the kernel fits at all); cases on the default grid assume the three CTAs per SM of the fused, hybrid and grouped kernels
and say so; hoisting cases use batches that give at least three rounds at any occupancy up to the four CTAs per SM of the context's
digit slots.  Group and round counts in the docstrings are for 132 SMs; every test computes its own and asserts them with `grid`.

Each test makes its own contexts and closes them (an N = 16384 context holds 264 MiB of digit and accumulator scratch).  Expected
results are computed once per input set and shared by the cases that slice it.  The file takes 90 to 110 s on an H100 80GB HBM3
(SXM, 700 W power limit) with an 8-core host, most of it in the oracle."""
import os
from collections import OrderedDict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import bases  # noqa: E402
import ct_dot_ref  # noqa: E402
import mul_rescale_ref as mrr  # noqa: E402
import polyeval_ref as pr  # noqa: E402
from test_gpu_grouped import grouped_inputs  # noqa: E402
from test_gpu_parity import dev, dp, edge_polys, host, hybrid_inputs  # noqa: E402,F401  (dp is a fixture)

LOG_N = 14
T = 65537
BOUNDARIES = [(1, -1), (1, 0), (1, 1), (3, 0), (3, 1)]   # batch = rounds * groups + extra
UNCAPPED = 1 << 30


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid(group, batch, occ=3, cap=0, occ_cap=True):
    """(groups, rounds) of one persistent launch, as launch_persistent (deeppowers_b200/csrc/kernels.cu:1416-1453) sizes it: the
    resident CTAs occ * SMs, capped by DPFHE_KS_OCC (cap) CTAs per SM unless the kernel ignores the cap (the hoisting kernels:
    occ_cap = False) and by the context's 4 * SMs digit slots, rounded down to whole groups of `group` CTAs and to at most `batch`
    groups; one ciphertext per group and round.  A group is L CTAs: every ciphertext limb for the fused kernel, every limb of the
    context (special primes included) for the hybrid and grouped kernels."""
    n = sms()
    G = occ * n
    if occ_cap and cap > 0:
        G = min(G, cap * n)
    G = min(G, 4 * n)
    G = min(G // group * group, batch * group)
    assert G > 0
    groups = G // group
    return groups, -(-batch // groups)


def hoist_batch(group):
    """at least three rounds of a hoisting kernel (ks_hoist_kernel, ks_hoistg_kernel: no DPFHE_KS_OCC cap) at any occupancy up to
    the four CTAs per SM of the digit slots"""
    batch = 3 * grid(group, UNCAPPED, occ=4, occ_cap=False)[0] + 1
    for occ in (1, 2, 3, 4):
        assert grid(group, batch, occ=occ, occ_cap=False)[1] >= 3, occ
    return batch


def rounds_of(rounds, extra):
    return rounds + 1 if extra > 0 else rounds


def check(got, want, groups, what=""):
    """bit for bit; on a mismatch names the ciphertexts and the grid rounds they fell in"""
    got = got.reshape(want.shape)
    bad = [k for k in range(want.shape[0]) if not np.array_equal(got[k], want[k])]
    assert not bad, "%s: ciphertexts %s of %d differ (rounds %s)" % (what, bad[:8], want.shape[0], sorted({k // groups for k in bad})[:8])


def per_ct(fn, n):
    """fn(k) for k < n on the host's cores (the oracle's single-ciphertext calls release the interpreter lock)"""
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        return list(ex.map(fn, range(n)))


def with_edges(o, n_polys, seed):
    """edge_polys, with its all-zero, all-(q - 1) and alternating rows repeated as the last three polynomials"""
    x = edge_polys(o, n_polys, seed)
    x[-3:] = x[:3].copy()
    return x


_REF = OrderedDict()


def cached(key, make):
    """inputs and expected results by key, the two most recent kept (a large batch at N = 16384 is hundreds of MiB)"""
    if key not in _REF:
        while len(_REF) >= 2:
            _REF.popitem(last=False)
        _REF[key] = make()
    _REF.move_to_end(key)
    return _REF[key]


@pytest.fixture
def make(dp, oracle_mod, monkeypatch):
    """make(L, env={}, moduli=None) -> (context, oracle): a context created with the environment variables `env` set, closed when
    the test ends.  The library allocates with cudaMalloc, which cannot use blocks torch still caches, so those go back first."""
    made = []
    torch.cuda.empty_cache()

    def get(L, env=None, moduli=None):
        env = env or {}
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        c = dp.Context(LOG_N, L, moduli)
        for k in env:
            monkeypatch.delenv(k)
        made.append(c)
        o = oracle_mod.Oracle(LOG_N, L, moduli)
        assert c.moduli == o.moduli
        return c, o

    yield get
    for c in made:
        c.close()
    torch.cuda.empty_cache()


# ---- 1 / 2: the fused kernel on group and round boundaries, double- and single-buffered -----------------------------------------

FUSED_MODES = ["mul", "keyswitch", "rot", "conj"]
GRIDS = {"default": {}, "occ1": {"DPFHE_KS_OCC": "1"},
         "single": {"DPFHE_KS_SINGLE": "1"}, "single_occ1": {"DPFHE_KS_SINGLE": "1", "DPFHE_KS_OCC": "1"}}


def fused_ref(oracle_mod, mode, L, moduli=None):
    """(inputs, key, expected) of one fused mode for three rounds and one of the default grid"""
    def build():
        o = oracle_mod.Oracle(LOG_N, L, moduli)
        B = 3 * grid(L, UNCAPPED)[0] + 1
        seed = 1000 * L + FUSED_MODES.index(mode)
        key = o.fill_uniform(seed + 7, 2 * L).reshape(L, 2, L, o.N)
        if mode == "keyswitch":
            d = with_edges(o, B, seed)
            want = np.stack(per_ct(lambda k: np.stack(o.keyswitch(d[k], key)), B))
            return (d,), key, want
        a = with_edges(o, 2 * B, seed).reshape(B, 2, L, o.N)
        if mode == "mul":
            b = with_edges(o, 2 * B, seed + 1)[::-1].copy().reshape(B, 2, L, o.N)
            return (a, b), key, o.ct_mul_relin(a, b, key)
        return (a,), key, o.rotate(a, galois(o, mode), key)
    return cached(("fused", mode, L, tuple(moduli) if moduli else None), build)


def galois(o, mode):
    return 2 * o.N - 1 if mode == "conj" else o.galois_elt(3)


def run_fused(c, o, mode, xs, key, out, batch, first=0):
    """one fused launch on ciphertexts first .. first + batch - 1 of the device inputs xs"""
    args = [x[first:first + batch] for x in xs]
    if mode == "mul":
        c.ct_mul_relin(args[0], args[1], key, out, batch)
    elif mode == "keyswitch":
        c.keyswitch(args[0], key, out, batch)
    else:
        c.rotate(args[0], galois(o, mode), key, out, batch)


# default grid and DPFHE_KS_OCC=1 for every mode at L = 1, 2, 4, 8, 16 and for ct x ct at L = 5; single-buffered for ct x ct and the
# rotation at L = 2, 4, 8, 16.  Ordered so that the cases of one input set follow each other.
FUSED_CASES = [(m, L, g) for m in FUSED_MODES for L in (1, 2, 4, 5, 8, 16) for g in GRIDS
               if (L != 5 or m == "mul") and ("single" not in g or (m in ("mul", "rot") and L in (2, 4, 8, 16)))]


@pytest.mark.parametrize("mode,L,grid_name", FUSED_CASES)
def test_fused_kernel_on_group_and_round_boundaries(make, oracle_mod, mode, L, grid_name):
    """batches rounds * groups + extra for (rounds, extra) in BOUNDARIES.  Groups of L CTAs: default grid (three CTAs per SM, 396
    CTAs) 396, 198, 99, 79, 49 and 24 groups for L = 1, 2, 4, 5, 8, 16; DPFHE_KS_OCC=1 (132 CTAs, exact) 132, 66, 33, 26, 16 and 8,
    L = 5 leaving two SMs without a CTA.  So 1 to 4 rounds per group; L = 1 has no digit exchange and its leader posts no ticket,
    L = 16 has 24 groups.  With DPFHE_KS_SINGLE every slot holds one digit, handed back through the consumed counters."""
    env = GRIDS[grid_name]
    cap = 1 if "occ1" in grid_name else 0
    xs, key, want = fused_ref(oracle_mod, mode, L)
    c, o = make(L, env)
    groups = grid(L, UNCAPPED, cap=cap)[0]
    dxs, dkey = [dev(x) for x in xs], dev(key)
    for rounds, extra in BOUNDARIES:
        batch = rounds * groups + extra
        assert batch <= want.shape[0]
        assert grid(L, batch, cap=cap) == (min(groups, batch), rounds_of(rounds, extra))
        out = torch.full((batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
        run_fused(c, o, mode, dxs, dkey, out, batch)
        check(host(out), want[:batch], groups, "%s batch %d" % (grid_name, batch))


def zero_digits(groups):
    """ciphertext -> the c1 limb set to zero (None: all of c1), for 3 * groups + 1 ciphertexts: the first and the last ciphertext
    of round 0, one in the middle of round 1, the one ciphertext of round 3"""
    return {0: None, groups - 1: 3, groups + groups // 2: 0, 3 * groups: None}


def hoisted_fallback_ref(oracle_mod):
    """three rounds and one of the default grid at L = 4 (298 ciphertexts), with zero c1 digits (zero_digits), a rotation and the
    conjugation"""
    def build():
        L = 4
        B = 3 * grid(L, UNCAPPED)[0] + 1
        o = oracle_mod.Oracle(LOG_N, L)
        ct = with_edges(o, 2 * B, 41).reshape(B, 2, L, o.N)
        for k, limb in zero_digits(grid(L, UNCAPPED)[0]).items():
            if limb is None:
                ct[k, 1] = 0
            else:
                ct[k, 1, limb] = 0
        gs = [o.galois_elt(3), 2 * o.N - 1]
        keys = [o.fill_uniform(50 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(gs))]
        return ct, gs, keys, np.stack([o.rotate(ct, g, k) for g, k in zip(gs, keys)])
    return cached(("hoisted_fallback",), build)


@pytest.mark.parametrize("chunks", [1, 3])
def test_single_buffered_hoisted_rotation_fallback(make, oracle_mod, monkeypatch, chunks):
    """rotate_hoisted with DPFHE_KS_SINGLE=1, L = 4, 298 ciphertexts, four of them with zero c1 digits: those take
    ks_fused_kernel<..., FILTER>, a static assignment that skips the rounds of the others.
    chunks = 1: the default grid, 99 groups, rounds 0, 1 and 3 hold a zero-digit ciphertext and round 2 publishes nothing.
    chunks = 3: DPFHE_HOIST_CAP_MB=200 (2 MiB of shared transforms per ciphertext: chunks of 100, 100 and 98) and DPFHE_KS_OCC=1
    (33 groups; 4, 4 and 3 rounds): the zero digits fall in rounds 0 and 2 of the first chunk, round 1 of the second and the last
    round of the third."""
    L = 4
    ct, gs, keys, want = hoisted_fallback_ref(oracle_mod)
    zeros = sorted(zero_digits(grid(L, UNCAPPED)[0]))
    env = {"DPFHE_KS_SINGLE": "1"}
    if chunks > 1:
        env["DPFHE_KS_OCC"] = "1"
    c, o = make(L, env)
    B = ct.shape[0]
    if chunks == 1:
        groups = grid(L, B)[0]
        assert grid(L, B) == (groups, 4) and sorted({k // groups for k in zeros}) == [0, 1, 3]
    else:
        groups = grid(L, UNCAPPED, cap=1)[0]
        chunk = 3 * groups + 1
        monkeypatch.setenv("DPFHE_HOIST_CAP_MB", str(2 * chunk))   # read at every call; L * L * N words per ciphertext
        assert -(-B // chunk) == 3 and grid(L, chunk, cap=1) == (groups, 4)
        where = [(k // chunk, k % chunk // groups) for k in zeros]
        assert where[0] == (0, 0) and where[-1] == (2, grid(L, B - 2 * chunk, cap=1)[1] - 1), where
    out = torch.full((len(gs), B, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted(dev(ct), gs, [dev(k) for k in keys], out, B)
    got = host(out)
    for r in range(len(gs)):
        check(got[r], want[r], groups, "rotation %d" % r)


# (first ciphertext, batch) of four launches on one context: 1, 3G + 1, 2 and G ciphertexts (G = 99 groups at L = 4)
def launch_sequence(groups):
    return [(5, 1), (0, 3 * groups + 1), (2 * groups, 2), (groups, groups)]


def restarts(limit, batches):
    """whether epoch_guard restarts the round numbering before each launch (kernels.cu:1387-1397; a launch advances it by batch + 1)"""
    epoch, out = 0, []
    for b in batches:
        r = epoch + b + 1 >= limit
        epoch = (0 if r else epoch) + b + 1
        out.append(r)
    return out


@pytest.mark.parametrize("restart", [False, True])
def test_single_buffered_launches_of_different_grids(make, oracle_mod, restart):
    """one DPFHE_KS_SINGLE context, ct x ct at L = 4 on the default grid (99 groups): launches of 1, 298, 2 and 99 ciphertexts
    (grids of 1, 99, 2 and 99 groups; 1, 4, 1 and 1 rounds).  The hand-back counters are monotone across launches and each launch
    reads its base at kernel start, so a slot that a small launch left unused must still work in the next large one.  With
    restart: DPFHE_EPOCH_LIMIT=301 (3G + 3): the round numbering restarts, and the counters are cleared, before the second and the
    third launch."""
    L = 4
    (a, b), key, want = fused_ref(oracle_mod, "mul", L)
    groups = grid(L, UNCAPPED)[0]
    seq = launch_sequence(groups)
    env = {"DPFHE_KS_SINGLE": "1"}
    if restart:
        env["DPFHE_EPOCH_LIMIT"] = str(3 * groups + 3)
        assert restarts(3 * groups + 3, [n for _, n in seq]) == [False, True, True, False]
    c, o = make(L, env)
    assert [grid(L, n)[1] for _, n in seq] == [1, 4, 1, 1]
    dxs, dkey = [dev(a), dev(b)], dev(key)
    for first, n in seq:
        out = torch.full((n, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
        run_fused(c, o, "mul", dxs, dkey, out, n, first)
        check(host(out), want[first:first + n], groups, "launch of %d from %d" % (n, first))


def test_single_buffered_slots_shared_with_other_kernels(make, oracle_mod):
    """one DPFHE_KS_SINGLE context at L = 4 (99 groups of the fused kernel on the default grid): fused ct x ct launches between a
    hybrid, a grouped (K = 2) and a hoisting launch, which write the same digit slots but not the hand-back counters; the hoisting
    launch also runs the fused FILTER instance on its zero-digit ciphertexts.  Batches: fused 298 (4 rounds), hybrid 100, fused 99,
    grouped 100, hoisted 100, fused 2."""
    L, K, n = 4, 2, 100
    (a, b), key, want = fused_ref(oracle_mod, "mul", L)
    c, o = make(L, {"DPFHE_KS_SINGLE": "1"})
    groups = grid(L, UNCAPPED)[0]
    dxs, dkey = [dev(a), dev(b)], dev(key)

    def fused(first, count):
        out = torch.full((count, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
        run_fused(c, o, "mul", dxs, dkey, out, count, first)
        check(host(out), want[first:first + count], groups, "fused launch of %d from %d" % (count, first))

    fused(0, want.shape[0])
    assert grid(L, want.shape[0]) == (groups, 4)
    ha, hkey = hybrid_inputs(o, n, 61)
    hb, _ = hybrid_inputs(o, n, 63)
    hout = torch.full(ha.shape, -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin_hybrid(dev(ha), dev(hb), dev(hkey), hout, n, T)
    check(host(hout), o.ct_mul_relin_hybrid(ha, hb, hkey, T), groups, "hybrid")
    fused(groups // 2, groups)
    ga, gkey = grouped_inputs(o, K, n, 65)
    gb, _ = grouped_inputs(o, K, n, 67)
    gout = torch.full(ga.shape, -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin_grouped(K, dev(ga), dev(gb), dev(gkey), gout, n, T)
    check(host(gout), o.ct_mul_relin_grouped(K, ga, gb, gkey, T), groups, "grouped")
    ct = with_edges(o, 2 * n, 69).reshape(n, 2, L, o.N)
    ct[0, 1] = 0
    ct[50, 1, 2] = 0
    ct[n - 1, 1, 0] = 0
    g = o.galois_elt(-3)
    rkey = o.fill_uniform(70, 2 * L).reshape(L, 2, L, o.N)
    rout = torch.full((1, n, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted(dev(ct), [g], [dev(rkey)], rout, n)
    check(host(rout)[0], o.rotate(ct, g, rkey), groups, "hoisted")
    fused(want.shape[0] - 2, 2)


# ---- 3: tuning switches -----------------------------------------------------------------------------------------------------------

SWITCHES = {"pf2": {"DPFHE_KS_PF": "2"}, "occ1": {"DPFHE_KS_OCC": "1"}, "occ2": {"DPFHE_KS_OCC": "2"}, "prof": {"DPFHE_KS_PROF": "1"},
            "force_generic": {"DPFHE_FORCE_GENERIC": "1"}, "single_pf2_occ1": {"DPFHE_KS_SINGLE": "1", "DPFHE_KS_PF": "2", "DPFHE_KS_OCC": "1"},
            "gen_mixed": {}}


@pytest.mark.parametrize("switch,mode", [(s, m) for s in SWITCHES for m in ("mul", "rot")])
def test_tuning_switch(make, oracle_mod, mode, switch):
    """each switch selects another instance or grid of the fused kernel at N = 16384, L = 4; a batch of three rounds and one:
    298 ciphertexts on the default grid (99 groups), 100 under DPFHE_KS_OCC=1 (33 groups), 199 under DPFHE_KS_OCC=2 (66 groups).
    gen_mixed: the first four moduli of that basis of tests/bases.py, which select the generic kernels."""
    L = 4
    env = SWITCHES[switch]
    moduli = None
    if switch == "gen_mixed":
        moduli = bases.catalogue(oracle_mod)["gen_mixed"][:L]
        assert not all(bases.is_fast(q) for q in moduli)
    cap = int(env.get("DPFHE_KS_OCC", 0))
    xs, key, want = fused_ref(oracle_mod, mode, L, moduli)
    c, o = make(L, env, moduli)
    groups = grid(L, UNCAPPED, cap=cap)[0]
    batch = 3 * groups + 1
    assert grid(L, batch, cap=cap) == (groups, 4)
    out = torch.full((batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    run_fused(c, o, mode, [dev(x) for x in xs], dev(key), out, batch)
    check(host(out), want[:batch], groups, switch)
    if switch == "prof" and mode == "mul":
        assert c.phase_cycles().any()   # the profiling instance ran


# ---- 4: the other persistent kernels ---------------------------------------------------------------------------------------------

def occ1(make, L, moduli=None):
    return make(L, {"DPFHE_KS_OCC": "1"}, moduli)


@pytest.mark.parametrize("mode", ["mul", "rot", "keyswitch"])
def test_hybrid_kernel_over_rounds(make, mode):
    """ks_hybrid_kernel under DPFHE_KS_OCC=1, L = 5 (four ciphertext limbs and the special prime): 26 groups of 5 CTAs, two SMs
    idle; 78 ciphertexts (3 rounds) and 79 (4 rounds).  t = 65537, the bare key switch t = 0."""
    L = 5
    c, o = occ1(make, L)
    groups = grid(L, UNCAPPED, cap=1)[0]
    B = 3 * groups + 1
    a, key = hybrid_inputs(o, B, 71)
    b, _ = hybrid_inputs(o, B, 73)
    a[-1, 1] = (np.array(o.moduli[:L - 1], dtype=np.uint64) - 1)[:, None]
    if mode == "mul":
        want = o.ct_mul_relin_hybrid(a, b, key, T)
    elif mode == "rot":
        want = o.rotate_hybrid(a, o.galois_elt(3), key, T)
    else:
        d = np.ascontiguousarray(a[:, 1])
        want = np.stack(per_ct(lambda k: np.stack(o.keyswitch_hybrid(d[k], key, 0)), B))
    da, db, dkey = dev(a), dev(b), dev(key)
    dd = dev(np.ascontiguousarray(a[:, 1]))
    for batch in (B - 1, B):
        assert grid(L, batch, cap=1) == (groups, 3 if batch == B - 1 else 4)
        out = torch.full((batch, 2, L - 1, o.N), -1, dtype=torch.int64, device="cuda")
        if mode == "mul":
            c.ct_mul_relin_hybrid(da[:batch], db[:batch], dkey, out, batch, T)
        elif mode == "rot":
            c.rotate_hybrid(da[:batch], o.galois_elt(3), dkey, out, batch, T)
        else:
            c.keyswitch_hybrid(dd[:batch], dkey, out, batch, 0)
        check(host(out), want[:batch], groups, "batch %d" % batch)


@pytest.mark.parametrize("K,L", [(1, 4), (2, 7), (3, 9), (4, 12)])
def test_grouped_kernel_over_rounds(make, K, L):
    """ks_grouped_kernel under DPFHE_KS_OCC=1, groups of L CTAs (every limb of the context): K = 1, L = 4: 33 groups; K = 2,
    Lq = 5 (a ragged last digit), L = 7: 18 groups; K = 3, L = 9: 14; K = 4, L = 12: 11.  Batches 3 * groups (3 rounds) and
    3 * groups + 1 (4 rounds), ct x ct and rotation with t = 65537, the bare key switch with t = 0."""
    c, o = occ1(make, L)
    groups = grid(L, UNCAPPED, cap=1)[0]
    B = 3 * groups + 1
    a, key = grouped_inputs(o, K, B, 80 + K)
    b, _ = grouped_inputs(o, K, B, 90 + K)
    a[-1, 1] = (np.array(o.moduli[:L - K], dtype=np.uint64) - 1)[:, None]
    d = np.ascontiguousarray(a[:, 1])
    g = o.galois_elt(3)
    want = {"mul": o.ct_mul_relin_grouped(K, a, b, key, T), "rot": o.rotate_grouped(K, a, g, key, T),
            "keyswitch": np.stack(per_ct(lambda k: np.stack(o.keyswitch_grouped(K, d[k], key, 0)), B))}
    da, db, dd, dkey = dev(a), dev(b), dev(d), dev(key)
    for batch in (B - 1, B):
        assert grid(L, batch, cap=1) == (groups, 3 if batch == B - 1 else 4)
        for mode, ref in want.items():
            out = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
            if mode == "mul":
                c.ct_mul_relin_grouped(K, da[:batch], db[:batch], dkey, out, batch, T)
            elif mode == "rot":
                c.rotate_grouped(K, da[:batch], g, dkey, out, batch, T)
            else:
                c.keyswitch_grouped(K, dd[:batch], dkey, out, batch, 0)
            check(host(out), ref[:batch], groups, "%s batch %d" % (mode, batch))


def test_rescale_and_inner_product_over_rounds(make, oracle_mod):
    """ks_rescale_grouped_kernel (ct_mul_relin_rescale_grouped) and ct_dot_grouped_kernel (three pairs) under DPFHE_KS_OCC=1,
    K = 2, Lq = 5, L = 7: 18 groups; 54 ciphertexts (3 rounds) and 55 (4 rounds), against tests/mul_rescale_ref.py and
    tests/ct_dot_ref.py"""
    K, L = 2, 7
    c, o = occ1(make, L)
    oq = oracle_mod.Oracle(LOG_N, L - K, o.moduli[:L - K])
    groups = grid(L, UNCAPPED, cap=1)[0]
    B = 3 * groups + 1
    pool = [grouped_inputs(o, K, B, 100 + 2 * i)[0] for i in range(4)]
    key = grouped_inputs(o, K, 1, 110)[1]
    ia, ib = [0, 1, 2], [3, 3, 1]
    want_rs = mrr.mul_rescale(o, K, [pool[0]], [pool[1]], key, T)
    chunks = np.array_split(np.arange(B), min(B, os.cpu_count() or 4))
    want_dot = np.concatenate(per_ct(lambda j: ct_dot_ref.ct_dot(o, oq, K, [pool[i][chunks[j]] for i in ia], [pool[i][chunks[j]] for i in ib],
                                                                 key, T), len(chunks)))
    dpool, dkey = [dev(p) for p in pool], dev(key)
    for batch in (B - 1, B):
        assert grid(L, batch, cap=1) == (groups, 3 if batch == B - 1 else 4)
        rs = torch.full((batch, 2, L - K - 1, o.N), -1, dtype=torch.int64, device="cuda")
        c.ct_mul_relin_rescale_grouped(K, dpool[0][:batch], dpool[1][:batch], dkey, rs, batch, T)
        check(host(rs), want_rs[:batch], groups, "rescale batch %d" % batch)
        dot = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
        c.ct_dot_grouped(K, [dpool[i][:batch] for i in ia], [dpool[i][:batch] for i in ib], dkey, dot, batch, T)
        check(host(dot), want_dot[:batch], groups, "inner product batch %d" % batch)


def test_hoisting_kernels_over_rounds(make):
    """ks_hoist_kernel (rotate_hoisted, L = 4: 397 ciphertexts, 4 rounds at 4 CTAs per SM, more at fewer; one ciphertext with a zero
    digit takes the fused FILTER instance) and ks_hoistg_kernel with its round marks (rotate_hoisted_grouped, K = 2, L = 7: 226
    ciphertexts), each with a rotation and the conjugation, on the default grid"""
    L = 4
    c, o = make(L)
    B = hoist_batch(L)
    groups = grid(L, B, occ=4, occ_cap=False)[0]
    ct = with_edges(o, 2 * B, 120).reshape(B, 2, L, o.N)
    ct[B // 2, 1, 1] = 0
    gs = [o.galois_elt(3), 2 * o.N - 1]
    keys = [o.fill_uniform(121 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(2)]
    out = torch.full((2, B, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted(dev(ct), gs, [dev(k) for k in keys], out, B)
    got = host(out)
    for r in range(2):
        check(got[r], o.rotate(ct, gs[r], keys[r]), groups, "hoisted rotation %d" % r)
    del ct, got, out
    K, L = 2, 7
    c, o = make(L)
    B = hoist_batch(L)
    groups = grid(L, B, occ=4, occ_cap=False)[0]
    ct, _ = grouped_inputs(o, K, B, 130)
    dnum = o.grouped_digits(K)
    keys = np.stack([o.fill_uniform(131 + r, 2 * dnum).reshape(dnum, 2, L, o.N) for r in range(2)])
    gs = [o.galois_elt(3), 2 * o.N - 1]
    out = torch.full((2, B, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted_grouped(K, dev(ct), gs, [dev(k) for k in keys], out, B, T)
    want = o.rotate_hoisted_grouped(K, ct, gs, keys, T)
    got = host(out).reshape(want.shape)
    for r in range(2):
        check(got[r], want[r], groups, "hoisted grouped rotation %d" % r)


def test_level_kernels_over_rounds(make):
    """the level forms at l = Lq - 1 = 4 on a K = 2, L = 7 context (the level's view: groups of l + K = 6 CTAs) against the same
    calls on a context over {q_0 .. q_3, p_0, p_1}, whose results are checked against the oracle: ct_mul_relin_grouped_level and
    rotate_grouped_level under DPFHE_KS_OCC=1 (22 groups; 66 and 67 ciphertexts, 3 and 4 rounds), rotate_hoisted_grouped_level on
    the default grid (265 ciphertexts, at least 3 rounds of ks_hoistg_kernel)"""
    K, L = 2, 7
    l = L - K - 1
    c, o = occ1(make, L)
    mods = [int(q) for q in o.moduli]
    cl, ol = occ1(make, l + K, mods[:l] + mods[L - K:])
    groups = grid(l + K, UNCAPPED, cap=1)[0]
    B = 3 * groups + 1
    a, _ = grouped_inputs(ol, K, B, 140)
    b, _ = grouped_inputs(ol, K, B, 141)
    top = o.fill_uniform(142, 2 * c.grouped_digits(K)).reshape(-1, 2, L, o.N)
    low = pr.restrict_key(top, L - K, K, l)
    g = o.galois_elt(3)
    want = {"mul": ol.ct_mul_relin_grouped(K, a, b, low, T), "rot": ol.rotate_grouped(K, a, g, low, T)}
    da, db, dtop, dlow = dev(a), dev(b), dev(top), dev(low)
    for batch in (B - 1, B):
        assert grid(l + K, batch, cap=1) == (groups, 3 if batch == B - 1 else 4)
        for mode, ref in want.items():
            got, same = [torch.full((batch, 2, l, o.N), -1, dtype=torch.int64, device="cuda") for _ in range(2)]
            if mode == "mul":
                c.ct_mul_relin_grouped_level(K, l, da[:batch], db[:batch], dtop, got, batch, T)
                cl.ct_mul_relin_grouped(K, da[:batch], db[:batch], dlow, same, batch, T)
            else:
                c.rotate_grouped_level(K, l, da[:batch], g, dtop, got, batch, T)
                cl.rotate_grouped(K, da[:batch], g, dlow, same, batch, T)
            check(host(same), ref[:batch], groups, "level context %s batch %d" % (mode, batch))
            check(host(got), host(same), groups, "level %s batch %d" % (mode, batch))
    B = hoist_batch(l + K)
    groups = grid(l + K, B, occ=4, occ_cap=False)[0]
    ct, _ = grouped_inputs(ol, K, B, 150)
    gs = [g, 2 * o.N - 1]
    tops = [o.fill_uniform(151 + r, 2 * c.grouped_digits(K)).reshape(-1, 2, L, o.N) for r in range(2)]
    lows = np.stack([pr.restrict_key(k, L - K, K, l) for k in tops])
    got, same = [torch.full((2, B, 2, l, o.N), -1, dtype=torch.int64, device="cuda") for _ in range(2)]
    c.rotate_hoisted_grouped_level(K, l, dev(ct), gs, [dev(k) for k in tops], got, B, T)
    cl.rotate_hoisted_grouped(K, dev(ct), gs, [dev(k) for k in lows], same, B, T)
    want = ol.rotate_hoisted_grouped(K, ct, gs, lows, T)
    for r in range(2):
        check(host(same[r]), want[r], groups, "level context hoisted rotation %d" % r)
        check(host(got[r]), host(same[r]), groups, "level hoisted rotation %d" % r)
