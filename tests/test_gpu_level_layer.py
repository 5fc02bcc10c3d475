"""The objects of a network layer at level l on the top-level context (DESIGN.md sections 2.21 / 4.18): the hoisted rotations
(rotate_hoisted_grouped_level), the linear layer (LinearLayer.grouped(..., level=l)) and the slot sum (SlotSum.grouped(..., level=l)), bit
for bit against the same call or object on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the keys restricted to that basis
(tests/polyeval_ref.py:restrict_key), over K = 1 .. 4, every valid level with ragged last digits, every ring degree, the moduli bases of
tests/bases.py, three plaintext moduli, baby = 1 and giant = 1; several grid rounds, restarting round numbers, level applies interleaved
with top-level calls on one and two streams, the host forms over several chunks, an apply after dpfhe_context_trim, the launch counts,
the level state's device memory and the argument checks; and decryption on ONE context with ONE key set: the BGV two-layer MLP
x -> W1 x + b1 -> p -> W2 at level Lf with a slot sum at Lf, CKKS PolyEval -> level layer, and the C++ example."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ckks_polyeval_ref as cr  # noqa: E402
from bases import catalogue  # noqa: E402
from test_gpu_levels import GALOIS, SEED, T_BGV, Level, _fresh, _keys, _oracles, _release_cached_blocks, _uniform, ctxs  # noqa: E402,F401
from test_gpu_parity import dev, dp, host  # noqa: E402,F401  (dp is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stack(keys, n):
    """n keys [dnum][2][rows][N] back to back, C-contiguous (what the objects take), or None when there are none"""
    return np.ascontiguousarray(np.stack(keys[:n])) if n else None


class Objects:
    """the level objects on the top-level context v.c and the same objects on the level context v.cl, over the same random keys"""

    def __init__(self, dp, v, rng, baby, giant, radices, t):
        self.v, self.t, self.baby, self.giant, self.radices = v, t, baby, giant, radices
        K, l = v.K, v.l
        self.diags = _uniform(rng, v.mods[:l], (baby * giant, l, v.N))
        top, low = v.keys(rng, baby)   # baby-step keys, then the giant-step key
        self.layer = dp.LinearLayer.grouped(v.c, K, self.diags, baby, _stack(top, baby - 1), top[baby - 1] if giant > 1 else None, t, level=l)
        self.layer_ref = dp.LinearLayer.grouped(v.cl, K, self.diags, baby, _stack(low, baby - 1), low[baby - 1] if giant > 1 else None, t)
        n_steps = len(dp.slotsum_steps(1, radices))
        top, low = v.keys(rng, n_steps)
        self.ss = dp.SlotSum.grouped(v.c, K, 1, radices, np.ascontiguousarray(top), t, level=l)
        self.ss_ref = dp.SlotSum.grouped(v.cl, K, 1, radices, _stack(low, n_steps), t)
        self.top_keys = top   # kept for the l = Lq comparison

    def close(self):
        for o in (self.layer, self.layer_ref, self.ss, self.ss_ref):
            o.close()


def _apply_both(obj, ref, v, ct, batch, stream=None):
    got, want = v.out(batch), v.out(batch)
    obj.apply(ct, got, batch, stream)
    ref.apply(ct, want, batch, stream)
    torch.cuda.synchronize()
    return got, want


def _check_hoisted(v, rng, batch, t, n_rot):
    K, l, c, cl = v.K, v.l, v.c, v.cl
    ct = dev(v.cts(rng, 1, batch)[0])
    top, low = v.keys(rng, n_rot)
    got = torch.full((n_rot, batch, 2, l, v.N), -1, dtype=torch.int64, device="cuda")
    want, same = torch.full_like(got, -1), torch.full_like(got, -1)
    c.rotate_hoisted_grouped_level(K, l, ct, GALOIS[:n_rot], [dev(k) for k in top], got, batch, t)
    cl.rotate_hoisted_grouped(K, ct, GALOIS[:n_rot], [dev(k) for k in low], want, batch, t)
    torch.cuda.synchronize()
    assert torch.equal(got, want) and bool((got != -1).all())
    if l == v.Lq:   # the top-level call itself
        c.rotate_hoisted_grouped(K, ct, GALOIS[:n_rot], [dev(k) for k in top], same, batch, t)
        torch.cuda.synchronize()
        assert torch.equal(got, same)


def _check_objects(dp, v, rng, batch, t, baby, giant, radices):
    objs = Objects(dp, v, rng, baby, giant, radices, t)
    ct = dev(v.cts(rng, 1, batch)[0])
    for obj, ref in ((objs.layer, objs.layer_ref), (objs.ss, objs.ss_ref)):
        got, want = _apply_both(obj, ref, v, ct, batch)
        assert torch.equal(got, want), type(obj).__name__
        assert bool((got != -1).all())
    if v.l == v.Lq:   # level = Lq is the top-level object itself
        top = dp.SlotSum.grouped(v.c, v.K, 1, radices, np.ascontiguousarray(objs.top_keys), t)
        got, want = _apply_both(objs.ss, top, v, ct, batch)
        assert torch.equal(got, want)
        top.close()
    objs.close()


# (log N, L, K): K = 1 .. 4, ragged last digits (K = 2, Lq = 7; K = 3, Lq = 7), every ring degree
SHAPES = [(12, 3, 1), (12, 5, 1), (12, 9, 2), (12, 10, 3), (12, 10, 4), (13, 6, 2), (13, 8, 3), (14, 6, 2), (14, 5, 1)]
# (baby, giant) and the slot sum's radices, cycled through the cases: baby = 1 and giant = 1 among them
FORMS = [((2, 3), [2]), ((1, 3), [3, 2]), ((3, 1), [2, 2]), ((4, 2), [5])]


@pytest.mark.parametrize("log_n,L,K,l", [(n, L, K, l) for n, L, K in SHAPES for l in range(K, L - K + 1)])
def test_every_level_against_level_context(dp, ctxs, log_n, L, K, l):
    v = Level(ctxs, log_n, L, K, l)
    k = 100 * log_n + 10 * L + K + l
    rng = np.random.default_rng(k)
    t = [0, 65537, T_BGV][(L + l) % 3]
    _check_hoisted(v, rng, 3, t, 1 + 2 * (k % 2))
    (baby, giant), radices = FORMS[k % len(FORMS)]
    _check_objects(dp, v, rng, 3, t, baby, giant, radices)


@pytest.mark.parametrize("t", [0, 65537, T_BGV])
@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_bases_and_plain_moduli(dp, ctxs, oracle_mod, basis, t):
    mods = catalogue(oracle_mod)[basis][:7]
    v = Level(ctxs, 12, len(mods), 2, 3, mods)
    rng = np.random.default_rng(sum(map(ord, basis)) + t % 97)
    _check_hoisted(v, rng, 2, t, 2)
    _check_objects(dp, v, rng, 2, t, 2, 2, [3])


@pytest.mark.parametrize("log_n", [13, 14])
def test_generic_arithmetic_at_larger_degrees(dp, ctxs, oracle_mod, log_n):
    """the generic-arithmetic instances at N = 8192 and 16384 (the default basis selects the fast ones)"""
    mods = catalogue(oracle_mod)["gen_mixed"][:7]
    for K, l in ((1, 3), (2, 3)):
        v = Level(ctxs, log_n, len(mods), K, l, mods)
        rng = np.random.default_rng(log_n + K)
        _check_hoisted(v, rng, 2, T_BGV, 2)
        _check_objects(dp, v, rng, 2, T_BGV, 2, 2, [2])


def test_grid_rounds(dp, ctxs, monkeypatch):
    """one CTA per SM: three grid rounds of the level's groups in every giant step and stage"""
    L, K, l, log_n = 7, 2, 3, 12
    v = Level(ctxs, log_n, L, K, l)
    v.c = _fresh(dp, monkeypatch, {"DPFHE_KS_OCC": "1"}, log_n, L)
    batch = 3 * (torch.cuda.get_device_properties(0).multi_processor_count // (l + K))
    _check_objects(dp, v, np.random.default_rng(50), batch, 65537, 2, 3, [2, 2])
    v.c.close()


def test_round_numbering_restarts_and_interleaving(dp, ctxs, monkeypatch):
    """round numbers that restart inside level layers, level applies between top-level calls, on one stream and alternating between
    two: every result is the bits of the object applied alone"""
    L, K, log_n, batch = 7, 2, 12, 9
    v = Level(ctxs, log_n, L, K, 3)
    v.c = _fresh(dp, monkeypatch, {"DPFHE_EPOCH_LIMIT": "40"}, log_n, L)   # ~10 rounds per launch against a limit of 40
    rng = np.random.default_rng(60)
    objs = Objects(dp, v, rng, 2, 4, [2, 3], 65537)
    ct = dev(v.cts(rng, 1, batch)[0])
    want_layer, want_ss = v.out(batch), v.out(batch)
    objs.layer_ref.apply(ct, want_layer, batch)
    objs.ss_ref.apply(ct, want_ss, batch)
    top = dev(_uniform(rng, v.mods[:v.Lq], (batch, 2, v.Lq, v.N)))
    key = dev(v.keys(rng, 1)[0][0])
    want_top = torch.empty_like(top)
    v.c.rotate_grouped(K, top, GALOIS[0], key, want_top, batch, 65537)
    torch.cuda.synchronize()
    for two in (False, True):
        streams = [torch.cuda.Stream(), torch.cuda.Stream()] if two else [torch.cuda.current_stream()] * 2
        outs = []
        for k in range(4):
            with torch.cuda.stream(streams[k % 2]):
                o_layer, o_ss, o_top = v.out(batch), v.out(batch), torch.empty_like(top)
            v.c.rotate_grouped(K, top, GALOIS[0], key, o_top, batch, 65537, stream=streams[k % 2].cuda_stream)
            objs.layer.apply(ct, o_layer, batch, streams[(k + 1) % 2].cuda_stream)
            objs.ss.apply(ct, o_ss, batch, streams[k % 2].cuda_stream)
            outs.append((o_layer, o_ss, o_top))
        torch.cuda.synchronize()
        for o_layer, o_ss, o_top in outs:
            assert torch.equal(o_layer, want_layer) and torch.equal(o_ss, want_ss) and torch.equal(o_top, want_top), two
    objs.close()
    v.c.close()


def test_host_forms_and_trim(dp, ctxs, monkeypatch):
    """apply_host over several chunks; an apply after dpfhe_context_trim gives the same bits"""
    monkeypatch.setenv("DPFHE_LINEAR_CHUNK_ROUNDS", "1")
    monkeypatch.setenv("DPFHE_SLOTSUM_CHUNK", "37")
    v = Level(ctxs, 12, 7, 2, 3)
    rng = np.random.default_rng(80)
    objs = Objects(dp, v, rng, 2, 3, [2, 2], 65537)
    batch = 3 * (torch.cuda.get_device_properties(0).multi_processor_count * 3 // v.L) + 5   # three chunks and a short one
    h_ct = v.cts(rng, 1, batch)[0]
    ct = dev(h_ct)
    for obj, ref in ((objs.layer, objs.layer_ref), (objs.ss, objs.ss_ref)):
        want = v.out(batch)
        ref.apply(ct, want, batch)
        h_out = np.zeros_like(h_ct)
        obj.apply_host(h_ct, h_out)
        assert np.array_equal(h_out, host(want).reshape(h_out.shape)), type(obj).__name__
    small = 4
    for obj, ref in ((objs.layer, objs.layer_ref), (objs.ss, objs.ss_ref)):
        before, _ = _apply_both(obj, ref, v, ct, small)
        v.c._chk(v.c._l.dpfhe_context_trim(v.c._h))
        after, want = _apply_both(obj, ref, v, ct, small)
        assert torch.equal(after, before) and torch.equal(after, want), type(obj).__name__
    objs.close()


def test_launch_counts_and_device_bytes(dp, ctxs):
    """an application at level l launches what the same object launches at the top level of the level context; after the first
    object at (K, l) neither a second object nor a level call adds level tables to dpfhe_context_device_bytes"""
    L, K, l, log_n, batch = 7, 2, 3, 12, 2
    v = Level(ctxs, log_n, L, K, l)
    c, cl = v.c, v.cl
    rng = np.random.default_rng(90)
    ct = dev(v.cts(rng, 1, batch)[0])
    top, _ = v.keys(rng, 3)
    dtop = [dev(k) for k in top]
    # the key-switch rows every grouped call shares, allocated first, so that what follows is the level's alone
    ctop = dev(_uniform(rng, v.mods[:v.Lq], (batch, 2, v.Lq, v.N)))
    c.rotate_grouped(K, ctop, GALOIS[0], dtop[0], torch.empty_like(ctop), batch, 0)
    torch.cuda.synchronize()
    bytes0 = c.device_bytes()
    objs = Objects(dp, v, rng, 3, 3, [2, 3], 65537)
    bytes1 = c.device_bytes()
    ss_keys = 2 * len(dp.slotsum_steps(1, [2, 3])) * c.grouped_digits(K) * 2 * L * v.N * 8   # the slot sum's keys and companions
    tables = bytes1 - bytes0 - ss_keys
    twiddles = 2 * (l + K) * v.N * 16   # the level's forward and inverse twiddles, with its limb constants: built at creation
    assert twiddles < tables < twiddles + (1 << 16), tables
    second = dp.LinearLayer.grouped(c, K, objs.diags, 3, np.ascontiguousarray(top[:2]), top[2], 65537, level=l)
    assert c.device_bytes() == bytes1
    o = v.out(batch)
    c.rotate_grouped_level(K, l, ct, GALOIS[0], dtop[0], o, batch, 0)
    torch.cuda.synchronize()
    assert c.device_bytes() == bytes1
    for obj, ref in ((objs.layer, objs.layer_ref), (objs.ss, objs.ss_ref)):
        _apply_both(obj, ref, v, ct, batch)   # scratch of the first application
        n0, m0 = c.launch_count(), cl.launch_count()
        _apply_both(obj, ref, v, ct, batch)
        assert c.launch_count() - n0 == cl.launch_count() - m0 > 0, type(obj).__name__
    n0, m0 = c.launch_count(), cl.launch_count()
    out = torch.empty((2, batch, 2, l, v.N), dtype=torch.int64, device="cuda")
    c.rotate_hoisted_grouped_level(K, l, ct, GALOIS[:2], dtop[:2], out, batch, 0)
    cl.rotate_hoisted_grouped(K, ct, GALOIS[:2], [dev(k) for k in v.keys(rng, 2)[1]], out, batch, 0)
    torch.cuda.synchronize()
    assert c.launch_count() - n0 == cl.launch_count() - m0 == 1 + 4 * 2
    second.close()
    objs.close()


def test_argument_checks(dp, oracle_mod):
    L, K, log_n, batch = 7, 2, 12, 2
    c = dp.Context(log_n, L)
    mods = [int(q) for q in oracle_mod.Oracle(log_n, L).moduli]
    Lq, N = L - K, c.N
    rng = np.random.default_rng(91)
    dnum = c.grouped_digits(K)
    keys = _uniform(rng, mods, (3, dnum, 2, L, N))
    diags3 = _uniform(rng, mods[:3], (4, 3, N))
    lib = c._l
    u64 = C.c_uint64 * 1
    for level, msg in ((1, "level 1"), (Lq + 1, "level %d" % (Lq + 1))):
        h = C.c_void_p()
        d = _uniform(rng, mods[:min(level, Lq)], (4, level, N))
        rc = lib.dpfhe_linear_create_grouped_level(c._h, K, level, d.ctypes.data, 4, 2, keys.ctypes.data, keys[2].ctypes.data, 0, C.byref(h))
        assert rc != 0 and not h.value and msg in lib.dpfhe_last_error().decode()
        rs = (C.c_uint * 1)(2)
        rc = lib.dpfhe_slotsum_create_grouped_level(c._h, K, level, 1, rs, 1, keys.ctypes.data, 0, C.byref(h))
        assert rc != 0 and not h.value and msg in lib.dpfhe_last_error().decode()
        ct = torch.zeros((batch, 2, level, N), dtype=torch.int64, device="cuda")
        out = torch.full((1, batch, 2, level, N), -7, dtype=torch.int64, device="cuda")
        with pytest.raises(dp.DpfheError) as e:
            c.rotate_hoisted_grouped_level(K, level, ct, GALOIS[:1], [dev(keys[0])], out, batch, 0)
        assert msg in str(e.value) and bool((out == -7).all())
    h = C.c_void_p()
    assert lib.dpfhe_linear_create_grouped_level(c._h, K, 3, None, 4, 2, keys.ctypes.data, keys[2].ctypes.data, 0, C.byref(h)) != 0 and not h.value
    assert lib.dpfhe_linear_create_grouped_level(c._h, K, 3, diags3.ctypes.data, 4, 2, None, keys[2].ctypes.data, 0, C.byref(h)) != 0
    assert not h.value
    assert lib.dpfhe_slotsum_create_grouped_level(c._h, K, 3, 1, (C.c_uint * 1)(2), 1, None, 0, C.byref(h)) != 0 and not h.value
    assert lib.dpfhe_linear_create_grouped_level(c._h, K, 3, diags3.ctypes.data, 4, 3, keys.ctypes.data, keys[2].ctypes.data, 0,
                                                 C.byref(h)) != 0 and not h.value   # 4 diagonals, baby 3
    assert lib.dpfhe_linear_create_grouped_level(c._h, K, 3, diags3.ctypes.data, 4, 2, keys.ctypes.data, keys[2].ctypes.data, mods[-1],
                                                 C.byref(h)) != 0 and not h.value   # t above a special prime
    ct = dev(_uniform(rng, mods[:3], (batch, 2, 3, N)))
    with pytest.raises(dp.DpfheError):   # the output overlaps the input
        c.rotate_hoisted_grouped_level(K, 3, ct, GALOIS[:1], [dev(keys[0])], ct, batch, 0)
    with pytest.raises(dp.DpfheError):   # a null key
        c._chk(lib.dpfhe_rotate_hoisted_grouped_level(c._h, K, 3, ct.data_ptr(), 1, u64(GALOIS[0]), (C.c_void_p * 1)(None),
                                                      ct.data_ptr() + 4096, batch, 0, None))
    layer = dp.LinearLayer.grouped(c, K, diags3, 2, np.ascontiguousarray(keys[:1]), keys[2], 0, level=3)
    with pytest.raises(dp.DpfheError):   # apply: the output overlaps the input
        layer.apply(ct, ct, batch)
    n0 = c.launch_count()   # an empty batch is fine and launches nothing
    layer.apply(ct, torch.empty_like(ct), 0)
    c.rotate_hoisted_grouped_level(K, 3, ct, GALOIS[:1], [dev(keys[0])], torch.empty_like(ct), 0, 0)
    assert c.launch_count() == n0
    layer.close()
    c.close()


# ---- decryption on ONE context with ONE key set -----------------------------------------------------------------------------------
def _bsgs_diagonals(W, baby, half):
    """the slots of the diagonals of an M x M matrix W as dpfhe_linear takes them: diagonal d holds W[i][(i + d) % M] in slot
    i + (d // baby) * baby (mod N/2) of the first row; the input must repeat its M slots at M .. 2M - 1"""
    M = W.shape[0]
    out = np.zeros((M, 2 * half), dtype=np.int64)
    for d in range(M):
        for i in range(M):
            out[d, (i + (d // baby) * baby) % half] = W[i, (i + d) % M]
    return out


def _margin_bits(low, mods, sk, ct):
    """decrypts ct on the prefix context `low` and returns log2(Q / 2) - log2(max |phase|), the phase centred mod Q = q_0 .. q_{l-1}:
    how many bits the noise could still grow before decryption fails"""
    B, l, N = ct.shape[0], low.L, low.N
    ph = torch.empty((B, l, N), dtype=torch.int64, device="cuda")
    low.decrypt(sk[:l].contiguous(), ct.contiguous(), 2, ph, B)
    low.ntt_inv(ph, B)
    torch.cuda.synchronize()
    r = host(ph).astype(object)
    mods = mods[:l]
    Q = 1
    for q in mods:
        Q *= q
    x = 0
    for i, q in enumerate(mods):
        Qi = Q // q
        x = x + r[:, i, :] * (Qi * pow(Qi, -1, q))
    x = x % Q
    x = np.where(x > Q // 2, x - Q, x)
    worst = max(int(abs(v)) for v in x.reshape(-1))
    return (Q // 2).bit_length() - max(worst, 1).bit_length()


def test_bgv_two_layer_mlp_and_slot_sum(dp, ctxs):
    """x -> W1 x + b1 -> p -> W2 at level Lf, with one context and one set of top-level keys, slot for slot mod t; then a slot sum at
    Lf.  Prints the phase margin after each stage (DESIGN.md section 2.21 records it)."""
    K, Lq, log_n, t, DIM, BABY, B = 2, 4, 13, 65537, 16, 4, 2
    coeffs = [3, -2, 1]   # 3 - 2x + x^2: one squaring, Lf = Lq - 1
    L = Lq + K
    c, o = ctxs(log_n, L)
    mods = [int(q) for q in o.moduli]
    N, half = c.N, c.N // 2
    sk, evk = _keys(c, K, t)
    steps = [1, 2, 3, 4]
    gk = torch.empty((len(steps), c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, t, sk, [c.galois_elt(s) for s in steps], bytes(range(2, 34)), gk)
    hk = host(gk).reshape(gk.shape)
    pe = dp.PolyEval(c, K, t, coeffs, host(evk).reshape(evk.shape))
    Lf = pe.result_limbs
    prefix = {l: ctxs(log_n, l, mods[:l])[0] for l in (Lq, Lf)}
    rng = np.random.default_rng(31)
    W1 = rng.integers(-8, 9, size=(DIM, DIM))
    W2 = rng.integers(-8, 9, size=(DIM, DIM))
    x = rng.integers(-8, 9, size=(B, DIM))
    b1 = rng.integers(-50, 51, size=DIM)
    # layer 1 is the 2 DIM x 2 DIM matrix [W1 0; W1 0] on [x, 0]: its result repeats W1 x at DIM .. 2 DIM - 1, the layout layer 2 reads
    W1e = np.zeros((2 * DIM, 2 * DIM), dtype=np.int64)
    W1e[:DIM, :DIM] = W1
    W1e[DIM:, :DIM] = W1
    xs = np.zeros((B, N), dtype=np.int64)
    xs[:, :DIM] = x
    xs[:, 2 * DIM:3 * DIM] = x
    bs = np.zeros((1, N), dtype=np.int64)
    bs[0, :DIM] = bs[0, DIM:2 * DIM] = b1

    def encode(slots, n):
        pt = torch.empty((n, Lq, N), dtype=torch.int64, device="cuda")
        prefix[Lq].bgv_encode(torch.from_numpy(np.ascontiguousarray(slots)).cuda(), pt, n, t)
        return pt

    d1 = host(encode(_bsgs_diagonals(W1e, BABY, half), 2 * DIM)).reshape(2 * DIM, Lq, N)
    d2 = host(encode(_bsgs_diagonals(W2, BABY, half), DIM)).reshape(DIM, Lq, N)[:, :Lf].copy()   # the first Lf rows: the level's encoding
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].encrypt(t, sk[:Lq].contiguous(), SEED, 0, encode(xs, B), ct, B)
    layer1 = dp.LinearLayer.grouped(c, K, d1, BABY, np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1], t)
    layer2 = dp.LinearLayer.grouped(c, K, d2, BABY, np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1], t, level=Lf)
    y = torch.empty_like(ct)
    layer1.apply(ct, y, B)
    margins = {"W1 x": _margin_bits(prefix[Lq], mods, sk, y)}
    prefix[Lq].ct_add_plain(y, encode(bs, 1)[0], y, B)
    z = torch.empty((B, 2, Lf, N), dtype=torch.int64, device="cuda")
    pe.apply(y, z, B)
    margins["p(W1 x + b1)"] = _margin_bits(prefix[Lf], mods, sk, z)
    w = torch.empty_like(z)
    layer2.apply(z, w, B)
    margins["W2 p(.) at level %d" % Lf] = _margin_bits(prefix[Lf], mods, sk, w)

    def slots(ct):
        low = prefix[ct.shape[2]]
        ph = torch.empty((ct.shape[0], low.L, N), dtype=torch.int64, device="cuda")
        low.decrypt(sk[:low.L].contiguous(), ct.contiguous(), 2, ph, ct.shape[0])
        s = torch.empty((ct.shape[0], N), dtype=torch.int64, device="cuda")
        low.bgv_decode(ph, s, ct.shape[0], t)
        return host(s).astype(object)

    def p(v):
        return sum(int(a) * v ** k for k, a in enumerate(coeffs)) % t

    h = (x.astype(object) @ W1.T.astype(object) + b1.astype(object)) % t
    zz = np.vectorize(p, otypes=[object])(h)
    want = (zz @ W2.T.astype(object)) % t
    assert np.array_equal(slots(w)[:, :DIM], want)
    # a slot sum of 16 slots at Lf on p(W1 x + b1): slot i sums the slots i .. i + 15, all of them valid for i <= DIM
    radices = [4, 4]
    ss_steps = dp.slotsum_steps(1, radices)
    sgk = torch.empty((len(ss_steps), c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, t, sk, [c.galois_elt(s) for s in ss_steps], bytes(range(3, 35)), sgk)
    ss = dp.SlotSum.grouped(c, K, 1, radices, host(sgk).reshape(sgk.shape), t, level=Lf)
    s = torch.empty_like(z)
    ss.apply(z, s, B)
    margins["slot sum at level %d" % Lf] = _margin_bits(prefix[Lf], mods, sk, s)
    zrep = np.concatenate([zz, zz], axis=1)
    want_s = np.array([[sum(zrep[k, i:i + 16]) % t for i in range(DIM + 1)] for k in range(B)], dtype=object)
    assert np.array_equal(slots(s)[:, :DIM + 1], want_s)
    print("BGV two-layer MLP on one context, phase margins in bits: %s" % margins)
    assert min(margins.values()) >= 10, margins
    for obj in (layer1, layer2, pe, ss):
        obj.close()


def test_ckks_polyeval_then_level_layer(dp, oracle_mod):
    """PolyEval.ckks -> the layer at its result level -> mod_switch_down on the prefix context, within a tolerance derived from the
    scales"""
    import deeppowers_b200
    K, Lq, log_n, DIM, BABY, B = 2, 5, 13, 16, 4, 2
    mods = cr.ckks_chain(oracle_mod, Lq, K)
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    N, half = c.N, c.N // 2
    sk, evk = _keys(c, K, 0)
    scale = float(mods[1])
    pe = dp.PolyEval.ckks(c, K, [0.5, 0.25, 0.125], scale, host(evk).reshape(evk.shape))
    Lf = pe.result_limbs
    prefix = {l: deeppowers_b200.Context(log_n, l, mods[:l]) for l in (Lq, Lf, Lf - 1)}
    gk = torch.empty((BABY, c.grouped_digits(K), 2, Lq + K, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, 0, sk, [c.galois_elt(s) for s in range(1, BABY + 1)], bytes(range(2, 34)), gk)
    hk = host(gk).reshape(gk.shape)
    rng = np.random.default_rng(41)
    W = rng.uniform(-1, 1, (DIM, DIM))
    z = np.zeros((B, half), dtype=np.complex128)
    xv = rng.uniform(-1, 1, (B, DIM))
    z[:, :DIM] = z[:, DIM:2 * DIM] = xv
    wscale = float(mods[Lf - 1])   # the diagonals' scale: the layer's product is divided by q_{Lf-1} afterwards
    dslots = np.zeros((DIM, half), dtype=np.complex128)
    for d in range(DIM):
        for i in range(DIM):
            dslots[d, (i + (d // BABY) * BABY) % half] = W[i, (i + d) % DIM]
    dpt = torch.empty((DIM, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].ckks_encode(torch.from_numpy(dslots).cuda(), dpt, DIM, wscale)
    diags = host(dpt).reshape(DIM, Lq, N)[:, :Lf].copy()
    pts = torch.empty((B, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].ckks_encode(torch.from_numpy(z).cuda(), pts, B, scale)
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    prefix[Lq].encrypt(0, sk[:Lq].contiguous(), SEED, 0, pts, ct, B)
    y = torch.empty((B, 2, Lf, N), dtype=torch.int64, device="cuda")
    pe.apply(ct, y, B)
    layer = dp.LinearLayer.grouped(c, K, diags, BABY, np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1], 0, level=Lf)
    w = torch.empty_like(y)
    layer.apply(y, w, B)
    r = torch.empty((B, 2, Lf - 1, N), dtype=torch.int64, device="cuda")
    prefix[Lf].mod_switch_down(w, r, 2 * B, 0)
    out_scale = pe.result_scale * wscale / mods[Lf - 1]
    low = prefix[Lf - 1]
    ph = torch.empty((B, Lf - 1, N), dtype=torch.int64, device="cuda")
    low.decrypt(sk[:Lf - 1].contiguous(), r, 2, ph, B)
    out = torch.empty((B, half), dtype=torch.complex128, device="cuda")
    low.ckks_decode(ph, out, B, out_scale)
    px = 0.5 + 0.25 * xv + 0.125 * xv ** 2
    want = px @ W.T
    err = np.abs(out.cpu().numpy()[:, :DIM] - want).max()
    # the bound: the rounding of the diagonals' encoding and of the rescale, relative to the scales, times the layer's DIM terms, far
    # above the key-switching noise, which the special primes divide away
    tol = DIM * 8.0 * (N / out_scale + N / wscale + N / pe.result_scale)
    print("CKKS PolyEval -> level layer at %d limbs: scale 2^%.2f, error 2^%.2f, tolerance 2^%.2f" % (Lf, np.log2(out_scale), np.log2(err), np.log2(tol)))
    assert err < tol, (err, tol)
    layer.close()
    pe.close()
    for x in [c] + list(prefix.values()):
        x.close()


def test_cpp_example(tmp_path):
    """examples/encrypted_two_layer_mlp.cpp against libdpfhe.so alone"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    libdir = os.path.join(ROOT, "deeppowers_b200")
    exe = str(tmp_path / "encrypted_two_layer_mlp")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "encrypted_two_layer_mlp.cpp"),
                           "-L", libdir, "-ldpfhe", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert " 0 wrong" in r.stdout
