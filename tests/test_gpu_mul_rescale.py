"""Multiply-and-rescale on the GPU (DESIGN.md sections 2.19 / 4.16): dpfhe_ct_mul_relin_rescale_grouped and
dpfhe_ct_dot_rescale_grouped through the C ABI, bit-exact against the oracle restatement (tests/mul_rescale_ref.py) over K = 1 .. 4,
ragged digits, every ring degree, the moduli bases of tests/bases.py, 1 / 9 / 64 pairs, three plaintext moduli, several grid rounds
and restarting round numbers; the host form, aliasing, argument checks, launch count and scratch; and what the result decrypts to
against the composition it replaces (the product, then dpfhe_mod_switch_down): BGV slots, CKKS values, the noise, and a second level."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ckks_polyeval_ref as cr  # noqa: E402
import mul_rescale_ref as mrr  # noqa: E402
import polyeval_ref as pr  # noqa: E402
from bases import catalogue  # noqa: E402
from test_gpu_parity import ctxs, dev, dp, host  # noqa: E402,F401  (ctxs and dp are fixtures)

T_BGV = 167772161


@pytest.fixture(scope="module", autouse=True)
def _release_cached_blocks():
    """the library allocates with cudaMalloc, which cannot use blocks torch keeps cached: hand this module's back when it is done"""
    yield
    torch.cuda.empty_cache()


def _setup(ctxs, log_n, L, K, moduli=None):
    c, o = ctxs(log_n, L, moduli)
    cq, oq = ctxs(log_n, L - K, list(o.moduli[:L - K]))
    return c, o, cq, oq


def _operands(o, oq, K, n_pool, batch, seed):
    pool = oq.fill_uniform(seed, n_pool * batch * 2).reshape(n_pool, batch, 2, oq.L, oq.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    pool[0, -1, 0] = (q - 1)[:, None]
    pool[-1, 0, 1] = 0
    key = o.fill_uniform(seed + 1, 2 * o.grouped_digits(K)).reshape(-1, 2, o.L, o.N)
    return pool, key


def _pairs(n, n_pool):
    ia = [(2 * t) % n_pool for t in range(n)]
    ib = [(2 * t + 1) % n_pool for t in range(n)]
    ib[-1] = ia[-1]   # a square
    return ia, ib


def _run(c, K, dpool, ia, ib, dkey, batch, t, Lq):
    out = torch.full((batch, 2, Lq - 1, c.N), -1, dtype=torch.int64, device="cuda")
    if len(ia) == 1:
        c.ct_mul_relin_rescale_grouped(K, dpool[ia[0]], dpool[ib[0]], dkey, out, batch, t)
    else:
        c.ct_dot_rescale_grouped(K, [dpool[i] for i in ia], [dpool[i] for i in ib], dkey, out, batch, t)
    return out


# (log N, L, K, batch, pairs, t): K = 1 .. 4, ragged digits (Lq = 5, K = 2), Lq = 2 (a one-limb result), every ring degree
SHAPES = [(12, 3, 1, 3, 1, 65537), (12, 4, 1, 2, 9, 0), (13, 6, 2, 3, 1, T_BGV), (13, 7, 2, 2, 9, 65537), (14, 6, 2, 2, 64, 0),
          (12, 7, 3, 2, 1, 0), (12, 8, 4, 2, 9, T_BGV), (12, 4, 2, 3, 1, 65537), (14, 7, 2, 2, 1, 65537), (13, 8, 4, 2, 64, 65537)]


@pytest.mark.parametrize("log_n,L,K,batch,n_terms,t", SHAPES)
def test_shapes_against_restatement(ctxs, log_n, L, K, batch, n_terms, t):
    c, o, cq, oq = _setup(ctxs, log_n, L, K)
    n_pool = min(2 * n_terms, 6)
    pool, key = _operands(o, oq, K, n_pool, batch, 100 + 7 * log_n + L + K)
    ia, ib = _pairs(n_terms, n_pool)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    out = _run(c, K, dpool, ia, ib, dkey, batch, t, L - K)
    want = mrr.mul_rescale(o, K, [pool[i] for i in ia], [pool[i] for i in ib], key, t)
    assert np.array_equal(host(out).reshape(want.shape), want)
    if n_terms == 1:   # the same pair as an inner product of one term: same bits
        dot = torch.empty_like(out)
        c.ct_dot_rescale_grouped(K, [dpool[ia[0]]], [dpool[ib[0]]], dkey, dot, batch, t)
        assert torch.equal(dot, out)


@pytest.mark.parametrize("t", [0, 65537, T_BGV])
@pytest.mark.parametrize("basis", ["gen_mixed", "gen_ascending", "gen_near60", "fast_mixed", "fast_narrow"])
def test_bases_and_plain_moduli(ctxs, oracle_mod, basis, t):
    mods = catalogue(oracle_mod)[basis][:6]
    K, L, log_n, batch = 2, len(mods), 12, 2
    c, o, cq, oq = _setup(ctxs, log_n, L, K, mods)
    pool, key = _operands(o, oq, K, 2, batch, 300)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    out = _run(c, K, dpool, [0], [1], dkey, batch, t, L - K)
    want = mrr.mul_rescale(o, K, [pool[0]], [pool[1]], key, t)
    assert np.array_equal(host(out).reshape(want.shape), want)


@pytest.mark.parametrize("log_n", [13, 14])
@pytest.mark.parametrize("basis", ["gen_mixed", "gen_near60"])
def test_generic_arithmetic_at_larger_degrees(ctxs, oracle_mod, basis, log_n):
    """the generic-arithmetic instances at N = 8192 and 16384 (the default basis selects the fast ones)"""
    mods = catalogue(oracle_mod)[basis][:6]
    K, L, batch = 2, len(mods), 2
    c, o, cq, oq = _setup(ctxs, log_n, L, K, mods)
    pool, key = _operands(o, oq, K, 4, batch, 350 + log_n)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    for ia, ib, t in (([0], [1], T_BGV), ([0, 2, 1, 3, 0, 2, 1, 3, 2], [1, 3, 0, 2, 1, 3, 0, 2, 2], 0)):
        out = _run(c, K, dpool, ia, ib, dkey, batch, t, L - K)
        want = mrr.mul_rescale(o, K, [pool[i] for i in ia], [pool[i] for i in ib], key, t)
        assert np.array_equal(host(out).reshape(want.shape), want), len(ia)


def test_aliased_operands(ctxs):
    """a and b as the same buffer (a square)"""
    K, L, log_n, batch = 2, 6, 12, 3
    c, o, cq, oq = _setup(ctxs, log_n, L, K)
    pool, key = _operands(o, oq, K, 1, batch, 400)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    out = _run(c, K, dpool, [0], [0], dkey, batch, 65537, L - K)
    want = mrr.mul_rescale(o, K, [pool[0]], [pool[0]], key, 65537)
    assert np.array_equal(host(out).reshape(want.shape), want)


@pytest.mark.parametrize("rounds_extra", [0, 1])
def test_grid_rounds(oracle_mod, monkeypatch, rounds_extra):
    """one CTA per SM: a batch of exactly three grid rounds, and one past them"""
    import deeppowers_b200
    monkeypatch.setenv("DPFHE_KS_OCC", "1")
    L, K, log_n = 6, 2, 12
    c = deeppowers_b200.Context(log_n, L)
    monkeypatch.delenv("DPFHE_KS_OCC")
    o = oracle_mod.Oracle(log_n, L)
    oq = oracle_mod.Oracle(log_n, L - K, o.moduli[:L - K])
    groups = torch.cuda.get_device_properties(0).multi_processor_count // L
    batch = 3 * groups + rounds_extra
    pool, key = _operands(o, oq, K, 4, batch, 500 + rounds_extra)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    for ia, ib in (([0], [1]), ([0, 2, 1], [1, 3, 1])):
        out = _run(c, K, dpool, ia, ib, dkey, batch, 65537, L - K)
        want = mrr.mul_rescale(o, K, [pool[i] for i in ia], [pool[i] for i in ib], key, 65537)
        assert np.array_equal(host(out).reshape(want.shape), want)
    c.close()


def test_round_numbering_restarts(oracle_mod, monkeypatch):
    """a context whose flag / mailbox round numbers restart inside the calls keeps producing the same bits"""
    import deeppowers_b200
    monkeypatch.setenv("DPFHE_EPOCH_LIMIT", "40")
    c = deeppowers_b200.Context(12, 6)
    monkeypatch.delenv("DPFHE_EPOCH_LIMIT")
    o = oracle_mod.Oracle(12, 6)
    oq = oracle_mod.Oracle(12, 4, o.moduli[:4])
    K, batch = 2, 9
    pool, key = _operands(o, oq, K, 4, batch, 600)
    want = mrr.mul_rescale(o, K, [pool[0], pool[2]], [pool[1], pool[3]], key, 65537)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    for _ in range(6):   # ~10 rounds per launch against a limit of 40
        out = _run(c, K, dpool, [0, 2], [1, 3], dkey, batch, 65537, 4)
        assert np.array_equal(host(out).reshape(want.shape), want)
    c.close()


def test_host_form_launches_scratch_and_checks(ctxs, dp):
    K, L, log_n, n_terms = 2, 6, 12, 3
    c, o, cq, oq = _setup(ctxs, log_n, L, K)
    Lq, batch = L - K, 700   # the host form splits the batch into several chunks
    a = oq.fill_uniform(700, n_terms * batch * 2).reshape(n_terms, batch, 2, Lq, o.N)
    b = oq.fill_uniform(701, n_terms * batch * 2).reshape(n_terms, batch, 2, Lq, o.N)
    key = o.fill_uniform(702, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    da, db, dkey = [dev(x) for x in a], [dev(x) for x in b], dev(key)
    out = torch.full((batch, 2, Lq - 1, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin_rescale_grouped(K, da[0], db[0], dkey, out, batch, 65537)   # reserves the rows of the call
    torch.cuda.synchronize()
    bytes0, n0 = c.device_bytes(), c.launch_count()
    c.ct_mul_relin_rescale_grouped(K, da[0], db[0], dkey, out, batch, 65537)
    torch.cuda.synchronize()
    assert c.launch_count() - n0 == 2 and c.device_bytes() == bytes0
    dot = torch.empty_like(out)
    n0 = c.launch_count()
    c.ct_dot_rescale_grouped(K, da, db, dkey, dot, batch, 65537)
    torch.cuda.synchronize()
    assert c.launch_count() - n0 == 2 and c.device_bytes() == bytes0
    # the host forms over several chunks (their staging buffers are the context's, kept for later host calls)
    h_out = np.zeros((batch, 2, Lq - 1, o.N), dtype=np.uint64)
    c.ct_mul_relin_rescale_grouped_host(K, a[0], b[0], key, h_out, 65537)
    assert np.array_equal(h_out, host(out).reshape(h_out.shape))
    assert np.array_equal(h_out[:2], mrr.mul_rescale(o, K, [a[0][:2]], [b[0][:2]], key, 65537))
    out = dot
    c.ct_dot_rescale_grouped_host(K, a, b, key, h_out, 65537)
    assert np.array_equal(h_out, host(out).reshape(h_out.shape))
    assert np.array_equal(h_out[-2:], mrr.mul_rescale(o, K, [x[-2:] for x in a], [x[-2:] for x in b], key, 65537))
    # rejected calls leave the output untouched
    small = 2
    mark = torch.full((small, 2, Lq - 1, o.N), -7, dtype=torch.int64, device="cuda")
    big = torch.full((small, 2, Lq, o.N), -7, dtype=torch.int64, device="cuda")
    big_head = big.view(-1)[:mark.numel()].view(mark.shape)   # the first words of big, as an output
    bad_calls = [
        lambda: c.ct_dot_rescale_grouped(K, [], [], dkey, mark, small, 65537),
        lambda: c.ct_dot_rescale_grouped(K, da[:1] * 65, db[:1] * 65, dkey, mark, small, 65537),
        lambda: c.ct_mul_relin_rescale_grouped(0, da[0], db[0], dkey, mark, small, 65537),
        lambda: c.ct_mul_relin_rescale_grouped(4, da[0], db[0], dkey, mark, small, 65537),
        lambda: c.ct_mul_relin_rescale_grouped(K, big, db[0], dkey, big_head, small, 65537),   # output overlaps an operand
        lambda: c.ct_dot_rescale_grouped(K, da[:2], [db[0], big], dkey, big_head[:1], 1, 65537),
        lambda: c.ct_mul_relin_rescale_grouped(K, da[0], db[0], dkey, mark, small, o.moduli[-1]),
        lambda: c.ct_mul_relin_rescale_grouped(K, da[0], db[0], dkey, mark, small, o.moduli[Lq - 1]),   # t above the dropped modulus
    ]
    for k, call in enumerate(bad_calls):
        with pytest.raises(dp.DpfheError):
            call()
        assert bool((mark == -7).all()) and bool((big == -7).all()), k
    mark2 = torch.full((small, 2, 1, o.N), -7, dtype=torch.int64, device="cuda")
    for Lc, k2 in ((2, 1), (3, 2)):   # one ciphertext limb: refused by the level check (K = 1), by the special-prime check (K = 2)
        c2, _ = ctxs(log_n, Lc)
        with pytest.raises(dp.DpfheError):
            c2.ct_mul_relin_rescale_grouped(k2, mark2, mark2, dkey, mark, 1, 0)
    assert bool((mark2 == -7).all())
    c.ct_mul_relin_rescale_grouped(K, da[0], db[0], dkey, mark, 0, 65537)   # an empty batch is fine and launches nothing
    c.ct_dot_rescale_grouped(K, da, db, dkey, mark, 0, 65537)
    assert bool((mark == -7).all())


# ---- semantics at N = 8192, Lq = 4, K = 2 --------------------------------------------------------------------------------------
SEED = bytes(range(40, 72))


def _keys(c, K, t):
    L, N = c.L, c.N
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    c.generate_secret(SEED, sk)
    evk = torch.empty((c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_relin_key(K, t, sk, bytes(range(1, 33)), evk)
    return sk, evk


def _composition(c, cq, K, a, b, evk, t):
    """the calls the fused one replaces: the product at Lq limbs, then the modulus switch on a context over the ciphertext moduli"""
    B, Lq, N = a.shape[0], cq.L, cq.N
    prod = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.ct_mul_relin_grouped(K, a, b, evk, prod, B, t)
    low = torch.empty((B, 2, Lq - 1, N), dtype=torch.int64, device="cuda")
    cq.mod_switch_down(prod, low, 2 * B, t)
    return low


def _phase_max(c_low, sk, ct):
    """the largest centred coefficient of the phase c0 + c1 s (an integer below the product of c_low's moduli)"""
    B = ct.shape[0]
    ph = torch.empty((B, c_low.L, c_low.N), dtype=torch.int64, device="cuda")
    c_low.decrypt(sk[:c_low.L].contiguous(), ct.contiguous(), 2, ph, B)
    c_low.ntt_inv(ph, B)
    r = host(ph).astype(object)
    mods = [int(q) for q in c_low.moduli]
    M = 1
    for q in mods:
        M *= q
    x = 0
    for l, q in enumerate(mods):
        Ml = M // q
        x = x + r[:, l] * (Ml * pow(Ml, -1, q))
    x = x % M
    x = np.where(x > M // 2, M - x, x)
    return int(x.max())


def test_bgv_slots_noise_and_second_level(ctxs):
    K, L, log_n, t = 2, 6, 13, T_BGV
    c, o, cq, oq = _setup(ctxs, log_n, L, K)
    c3, _ = ctxs(log_n, 3, list(o.moduli[:3]))
    c2, _ = ctxs(log_n, 2, list(o.moduli[:2]))
    c5, _ = ctxs(log_n, 5, list(o.moduli[:3]) + list(o.moduli[4:]))   # {q_0 .. q_2, p_0, p_1}
    N, Lq, B = c.N, L - K, 2
    sk, evk = _keys(c, K, t)
    rng = np.random.default_rng(11)
    x = rng.integers(-200, 200, size=(B, N), dtype=np.int64)
    y = rng.integers(-200, 200, size=(B, N), dtype=np.int64)
    pts = torch.empty((2 * B, Lq, N), dtype=torch.int64, device="cuda")
    cq.bgv_encode(torch.from_numpy(np.concatenate([x, y])).cuda(), pts, 2 * B, t)
    cts = torch.empty((2 * B, 2, Lq, N), dtype=torch.int64, device="cuda")
    cq.encrypt(t, sk[:Lq].contiguous(), SEED, 0, pts, cts, 2 * B)
    a, b = cts[:B].contiguous(), cts[B:].contiguous()
    fused = torch.empty((B, 2, Lq - 1, N), dtype=torch.int64, device="cuda")
    c.ct_mul_relin_rescale_grouped(K, a, b, evk, fused, B, t)
    comp = _composition(c, cq, K, a, b, evk, t)

    def slots(ctx_low, ct):
        ph = torch.empty((ct.shape[0], ctx_low.L, N), dtype=torch.int64, device="cuda")
        ctx_low.decrypt(sk[:ctx_low.L].contiguous(), ct.contiguous(), 2, ph, ct.shape[0])
        s = torch.empty((ct.shape[0], N), dtype=torch.int64, device="cuda")
        ctx_low.bgv_decode(ph, s, ct.shape[0], t)
        return host(s)

    qbar = int(o.moduli[Lq - 1])
    want = (x * y % t) * pow(qbar, -1, t) % t
    got_f, got_c = slots(c3, fused), slots(c3, comp)
    assert np.array_equal(got_f, got_c) and np.array_equal(got_f, want.astype(np.uint64))
    n_f, n_c = _phase_max(c3, sk, fused), _phase_max(c3, sk, comp)
    print("BGV phase max: fused 2^%.2f, composition 2^%.2f" % (np.log2(n_f), np.log2(n_c)))
    assert n_f <= 4 * n_c
    # a second level: the square on {q_0 .. q_2, p_0, p_1} with the restricted key gives x^4 (y^4) on two limbs
    key3 = dev(pr.restrict_key(host(evk).reshape(-1, 2, L, N), Lq, K, 3))
    four = torch.empty((B, 2, 2, N), dtype=torch.int64, device="cuda")
    c5.ct_mul_relin_rescale_grouped(K, fused, fused, key3, four, B, t)
    q2 = int(o.moduli[2])
    want4 = pow(x * y % t, 2, None) % t * pow(qbar, -2, t) % t * pow(q2, -1, t) % t
    assert np.array_equal(slots(c2, four), want4.astype(np.uint64))


def test_ckks_values_noise_and_second_level(oracle_mod):
    import deeppowers_b200
    K, Lq, log_n, delta = 2, 4, 13, 2.0**40
    mods = cr.ckks_chain(oracle_mod, Lq, K)
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    cq = deeppowers_b200.Context(log_n, Lq, mods[:Lq])
    c3 = deeppowers_b200.Context(log_n, 3, mods[:3])
    c2 = deeppowers_b200.Context(log_n, 2, mods[:2])
    c5 = deeppowers_b200.Context(log_n, 5, mods[:3] + mods[Lq:])
    N, B = c.N, 2
    sk, evk = _keys(c, K, 0)
    rng = np.random.default_rng(12)
    z = rng.uniform(-1, 1, (2 * B, N // 2)) + 1j * rng.uniform(-1, 1, (2 * B, N // 2))
    pts = torch.empty((2 * B, Lq, N), dtype=torch.int64, device="cuda")
    cq.ckks_encode(torch.from_numpy(z).cuda(), pts, 2 * B, delta)
    cts = torch.empty((2 * B, 2, Lq, N), dtype=torch.int64, device="cuda")
    cq.encrypt(0, sk[:Lq].contiguous(), SEED, 0, pts, cts, 2 * B)
    a, b = cts[:B].contiguous(), cts[B:].contiguous()
    fused = torch.empty((B, 2, Lq - 1, N), dtype=torch.int64, device="cuda")
    c.ct_mul_relin_rescale_grouped(K, a, b, evk, fused, B, 0)
    comp = _composition(c, cq, K, a, b, evk, 0)

    def decode(ctx_low, ct, scale):
        ph = torch.empty((ct.shape[0], ctx_low.L, N), dtype=torch.int64, device="cuda")
        ctx_low.decrypt(sk[:ctx_low.L].contiguous(), ct.contiguous(), 2, ph, ct.shape[0])
        out = torch.empty((ct.shape[0], N // 2), dtype=torch.complex128, device="cuda")
        ctx_low.ckks_decode(ph, out, ct.shape[0], scale)
        return out.cpu().numpy()

    scale1 = delta * delta / mods[Lq - 1]
    want = z[:B] * z[B:]
    err_f = np.abs(decode(c3, fused, scale1) - want).max()
    err_c = np.abs(decode(c3, comp, scale1) - want).max()
    n_f, n_c = _phase_max(c3, sk, fused), _phase_max(c3, sk, comp)
    print("CKKS error: fused 2^%.2f, composition 2^%.2f; phase max fused 2^%.2f, composition 2^%.2f"
          % (np.log2(err_f), np.log2(err_c), np.log2(n_f), np.log2(n_c)))
    assert err_f < 2.0**-15   # DESIGN.md section 2.19: measured 2^-20.95 (the composition 2^-21.48)
    assert n_f <= 4 * n_c
    key3 = dev(pr.restrict_key(host(evk).reshape(-1, 2, Lq + K, N), Lq, K, 3))
    four = torch.empty((B, 2, 2, N), dtype=torch.int64, device="cuda")
    c5.ct_mul_relin_rescale_grouped(K, fused, fused, key3, four, B, 0)
    err4 = np.abs(decode(c2, four, scale1 * scale1 / mods[2]) - want * want).max()
    print("CKKS second level error 2^%.2f" % np.log2(err4))
    assert err4 < 2.0**-5   # measured 2^-10.80: the second scale is about 2^25
    for x in (c, cq, c3, c2, c5):
        x.close()
