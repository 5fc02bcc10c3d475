"""Seeded ciphertexts and switch keys on the GPU (DESIGN.md section 2.23): bit for bit against the restatement (tests/seeded_ref.py) at
N = 4096, 8192 and 16384 on the default, gen_mixed and fast_mixed bases, with t and t = 0, batches past one grid wave and item numbers
crossing 2^32; keys for K = 0 .. 4 with ragged digits and more than one launch of Galois elements; the level forms against the top-level
rows and a prefix context; the host and upload forms over several chunks; launch counts; argument checks that leave the output
untouched; expanded keys through the grouped products and rotations, and the noise of a fresh seeded ciphertext."""
import numpy as np
import pytest

import bases
import keys_ref as kr
import seeded_ref as sr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(7, 39))
T = 65537


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def _setup(oracle_mod, logn, L, basis=None):
    import deeppowers_b200 as dp
    moduli = bases.catalogue(oracle_mod)[basis][:L] if basis else None
    o = oracle_mod.Oracle(logn, L, moduli)
    return dp.Context(logn, L, o.moduli), o


@pytest.mark.parametrize("logn,L,basis,t,n,first", [(12, 2, None, T, 700, 0), (12, 6, "gen_mixed", 0, 5, (1 << 32) - 2),
                                                    (13, 4, None, T, 5, 11), (13, 6, "fast_mixed", 0, 3, 0), (14, 3, None, T, 3, (1 << 32) - 1),
                                                    (14, 6, "gen_mixed", 0, 2, 7)])
def test_encrypt_and_expand_bit_exact(oracle_mod, logn, L, basis, t, n, first):
    """c0 of dpfhe_encrypt_seeded and the ciphertexts of dpfhe_expand_ciphertexts against the restatement; n = 700 at N = 4096 spans
    several waves of the grid; item numbers first + k cross 2^32"""
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, SEED)
    a_seed = ctx.public_seed(SEED)
    assert a_seed == sr.public_seed(SEED)
    pt = o.fill_uniform(11, n)
    c0 = empty(n, L, o.N)
    ctx.encrypt_seeded(t, dev(s), SEED, first, dev(pt), c0, n)
    ct = empty(n, 2, L, o.N)
    n_launch = ctx.launch_count()
    ctx.expand_ciphertexts(a_seed, first, c0, ct, n)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == 1
    got = host(ct)
    assert np.array_equal(got[:, 0], host(c0))
    idx = range(n) if n < 50 else [0, 1, 263, 264, 527, 528, n - 1]
    for k in idx:
        assert np.array_equal(got[k], sr.encrypt_seeded(o, t, s, SEED, first + k, pt[k:k + 1])[0]), k
    ctx.close()


@pytest.mark.parametrize("K", [0, 1, 2, 3, 4])
def test_relin_keys_bit_exact(oracle_mod, K):
    """K = 3: a ragged last digit (5 ciphertext limbs in digits of 3 and 2)"""
    L = 8
    ctx, o = _setup(oracle_mod, 12, L)
    s = kr.secret(o, SEED)
    nd = ctx.key_digits(K)
    want = sr.relin_key_seeded(o, K, T, s, SEED)
    b = empty(nd, L, o.N)
    ctx.generate_relin_key_seeded(K, T, dev(s), SEED, b)
    assert np.array_equal(host(b), want[:, 0])
    keys = empty(1, nd, 2, L, o.N)
    n_launch = ctx.launch_count()
    ctx.expand_switch_keys(K, ctx.public_seed(SEED), [0], b, keys)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == 1
    assert np.array_equal(host(keys)[0], want)
    hb = np.empty((nd, L, o.N), dtype=np.uint64)
    ctx.generate_relin_key_seeded_host(K, T, s, SEED, hb)
    assert np.array_equal(hb, want[:, 0])
    ctx.close()


@pytest.mark.parametrize("logn,L,K,basis", [(12, 4, 0, None), (12, 6, 2, "gen_mixed"), (13, 4, 1, None), (14, 3, 0, None), (14, 6, 3, "fast_mixed")])
def test_galois_keys_bit_exact(oracle_mod, logn, L, K, basis):
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, SEED)
    elts = [o.galois_elt(1), o.galois_elt(-3), 2 * o.N - 1]
    nd = ctx.key_digits(K)
    want = sr.galois_keys_seeded(o, K, 0, s, SEED, elts)
    b = empty(len(elts), nd, L, o.N)
    ctx.generate_galois_keys_seeded(K, 0, dev(s), elts, SEED, b)
    assert np.array_equal(host(b), want[:, :, 0])
    keys = empty(len(elts), nd, 2, L, o.N)
    ctx.expand_switch_keys(K, ctx.public_seed(SEED), elts, b, keys)
    assert np.array_equal(host(keys), want)
    hb = np.empty((len(elts), nd, L, o.N), dtype=np.uint64)
    ctx.generate_galois_keys_seeded_host(K, 0, s, elts, SEED, hb)
    assert np.array_equal(hb, want[:, :, 0])
    ctx.close()


def test_keys_beyond_one_launch(oracle_mod):
    """70 Galois elements (KEYS_MAX_ELTS = 64 per launch) and the relinearisation key among the expanded items; upload and host forms"""
    L = 2
    ctx, o = _setup(oracle_mod, 12, L)
    s = kr.secret(o, SEED)
    elts = [o.galois_elt(k) for k in range(1, 71)]
    b = empty(len(elts), L, L, o.N)
    n_launch = ctx.launch_count()
    ctx.generate_galois_keys_seeded(0, T, dev(s), elts, SEED, b)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == 2
    rb = empty(1, L, L, o.N)
    ctx.generate_relin_key_seeded(0, T, dev(s), SEED, rb)
    items = elts + [0]
    allb = torch.cat([b, rb])
    keys = empty(len(items), L, 2, L, o.N)
    a_seed = ctx.public_seed(SEED)
    n_launch = ctx.launch_count()
    ctx.expand_switch_keys(0, a_seed, items, allb, keys)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == 2
    got = host(keys)
    for i in (0, 63, 64, 69):
        assert np.array_equal(got[i], sr.galois_keys_seeded(o, 0, T, s, SEED, [elts[i]])[0]), i
    assert np.array_equal(got[70], sr.relin_key_seeded(o, 0, T, s, SEED))
    up = empty(len(items), L, 2, L, o.N)
    ctx.upload_seeded_switch_keys(0, a_seed, items, host(allb).copy(), up)
    assert np.array_equal(host(up), got)
    hk = np.empty(got.shape, dtype=np.uint64)
    ctx.expand_switch_keys_host(0, a_seed, items, host(allb).copy(), hk)
    assert np.array_equal(hk, got)
    ctx.close()


def test_upload_and_host_forms_over_several_chunks(oracle_mod):
    """1100 ciphertexts of N = 4096, L = 2 are three chunks of the pipeline: the upload and the host encryption keep item numbers
    first_index + k across chunks and equal the device forms"""
    L, n, first = 2, 1100, (1 << 32) - 600
    ctx, o = _setup(oracle_mod, 12, L)
    s = kr.secret(o, SEED)
    pt = o.fill_uniform(12, n)
    hc0 = np.empty((n, L, o.N), dtype=np.uint64)
    ctx.encrypt_seeded_host(T, s, SEED, first, pt, hc0)
    c0 = empty(n, L, o.N)
    ctx.encrypt_seeded(T, dev(s), SEED, first, dev(pt), c0, n)
    assert np.array_equal(hc0, host(c0))
    a_seed = ctx.public_seed(SEED)
    ct = empty(n, 2, L, o.N)
    ctx.expand_ciphertexts(a_seed, first, c0, ct, n)
    up = torch.full((n, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    n_launch = ctx.launch_count()
    ctx.upload_seeded_ciphertexts(a_seed, first, hc0, up)
    assert ctx.launch_count() - n_launch >= 2
    assert torch.equal(up, ct)
    for k in (0, 599, 600, n - 1):
        assert np.array_equal(host(ct[k]), sr.encrypt_seeded(o, T, s, SEED, first + k, pt[k:k + 1])[0]), k
    ctx.close()


@pytest.mark.parametrize("logn", [12, 14])
def test_level_forms(oracle_mod, logn):
    """the level forms equal the top-level rows and the calls on a prefix context; level = L is the top-level call"""
    import deeppowers_b200 as dp
    L, n = 5, 3
    ctx, o = _setup(oracle_mod, logn, L)
    s = kr.secret(o, SEED)
    a_seed = ctx.public_seed(SEED)
    pt = o.fill_uniform(13, n)
    top = empty(n, L, o.N)
    ctx.encrypt_seeded(T, dev(s), SEED, 4, dev(pt), top, n)
    top_ct = empty(n, 2, L, o.N)
    ctx.expand_ciphertexts(a_seed, 4, top, top_ct, n)
    for l in (1, 3, L):
        ptl = np.ascontiguousarray(pt[:, :l])
        c0 = empty(n, l, o.N)
        ctx.encrypt_seeded_level(l, T, dev(s), SEED, 4, dev(ptl), c0, n)
        assert torch.equal(c0, top[:, :l]), l
        ct = empty(n, 2, l, o.N)
        ctx.expand_ciphertexts_level(l, a_seed, 4, c0, ct, n)
        assert torch.equal(ct, top_ct[:, :, :l]), l
        hc0 = np.empty((n, l, o.N), dtype=np.uint64)
        ctx.encrypt_seeded_level_host(l, T, s, SEED, 4, ptl, hc0)
        assert np.array_equal(hc0, host(c0)), l
        up = empty(n, 2, l, o.N)
        ctx.upload_seeded_ciphertexts_level(l, a_seed, 4, hc0, up)
        assert torch.equal(up, ct), l
        pre = dp.Context(logn, l, o.moduli[:l])
        pc0 = empty(n, l, o.N)
        pre.encrypt_seeded(T, dev(s[:l]), SEED, 4, dev(ptl), pc0, n)
        assert torch.equal(pc0, c0), l
        pre.close()
    ctx.close()


def test_argument_checks_leave_the_output_untouched(oracle_mod):
    import deeppowers_b200 as dp
    L = 4
    ctx, o = _setup(oracle_mod, 12, L)
    s = dev(kr.secret(o, SEED))
    pt = dev(o.fill_uniform(1, 2))
    a_seed = ctx.public_seed(SEED)
    c0 = torch.full((2, L, o.N), 7, dtype=torch.int64, device="cuda")
    ct = torch.full((2, 2, L, o.N), 7, dtype=torch.int64, device="cuda")
    keys = torch.full((2, L, 2, L, o.N), 7, dtype=torch.int64, device="cuda")
    b = torch.zeros((2, L, L, o.N), dtype=torch.int64, device="cuda")
    n_launch = ctx.launch_count()
    bad = [
        lambda: ctx.encrypt_seeded(T, s, None, 0, pt, c0, 2),
        lambda: ctx.encrypt_seeded(T, s, SEED, 0, pt, pt, 2),
        lambda: ctx.encrypt_seeded_level(L + 1, T, s, SEED, 0, pt, c0, 2),
        lambda: ctx.encrypt_seeded_level(0, T, s, SEED, 0, pt, c0, 2),
        lambda: ctx.expand_ciphertexts(None, 0, c0, ct, 2),
        lambda: ctx.expand_ciphertexts(a_seed, 0, ct[0], ct, 2),
        lambda: ctx.expand_ciphertexts(a_seed, 0, c0, int(ct.data_ptr()) + 8, 2),
        lambda: ctx.expand_switch_keys(5, a_seed, [0, 3], b, keys),
        lambda: ctx.expand_switch_keys(0, a_seed, [0, 4], b, keys),
        lambda: ctx.expand_switch_keys(0, a_seed, [0, 2 * o.N + 1], b, keys),
        lambda: ctx.expand_switch_keys(0, a_seed, [0, 3], keys, keys),
        lambda: ctx.generate_relin_key_seeded(3, T, s, SEED, keys),
        lambda: ctx.generate_galois_keys_seeded(0, T, s, [2], SEED, keys),
        lambda: ctx.generate_relin_key_seeded(0, T, s, SEED, s),
        lambda: ctx.upload_seeded_switch_keys(0, a_seed, [0, 6], np.zeros((2, L, L, o.N), dtype=np.uint64), keys),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(dp.DpfheError):
            call()
    torch.cuda.synchronize()
    assert ctx.launch_count() == n_launch
    assert bool((c0 == 7).all()) and bool((ct == 7).all()) and bool((keys == 7).all())
    ctx.close()


def _noise(o, s, ct, m):
    """the largest |phase - m| over every limb, centred"""
    ph = o.phase(s[:o.L], ct)
    worst = 0
    for l, q in enumerate(o.moduli):
        for i in range(o.N):
            v = (int(ph[l, i]) - int(m[i])) % q
            worst = max(worst, abs(v - q if v > q // 2 else v))
    return worst


@pytest.mark.parametrize("logn", [12, 13])
def test_expanded_keys_in_grouped_products_and_rotations(oracle_mod, logn):
    """seeded ciphertexts and seeded keys, expanded on the device, through ct_mul_relin_grouped, rotate_grouped and
    ct_mul_relin_rescale_grouped_level: bit for bit the same calls with the restated ciphertexts and keys; the product and the rotation
    decrypt to m1 m2 and the rotated message, and a fresh seeded ciphertext carries at most 21 t of noise"""
    L, K = 6, 2
    Lq = L - K
    ctx, o = _setup(oracle_mod, logn, L)
    oq = oracle_mod.Oracle(logn, Lq, o.moduli[:Lq])
    s = kr.secret(o, SEED)
    a_seed = ctx.public_seed(SEED)
    rng = np.random.default_rng(9)
    m = rng.integers(0, T, size=(2, o.N)).astype(np.int64)
    signed = np.where(m > T // 2, m - T, m)
    pt = np.concatenate([kr.small_eval(oq, x, 1)[None] for x in signed])
    c0 = empty(2, Lq, o.N)
    ctx.encrypt_seeded_level(Lq, T, dev(s), SEED, 0, dev(pt), c0, 2)
    ct = empty(2, 2, Lq, o.N)
    ctx.expand_ciphertexts_level(Lq, a_seed, 0, c0, ct, 2)
    nd = ctx.key_digits(K)
    rb = empty(nd, L, o.N)
    ctx.generate_relin_key_seeded(K, T, dev(s), SEED, rb)
    evk = empty(1, nd, 2, L, o.N)
    ctx.expand_switch_keys(K, a_seed, [0], rb, evk)
    g = o.galois_elt(1)
    gb = empty(1, nd, L, o.N)
    ctx.generate_galois_keys_seeded(K, T, dev(s), [g], SEED, gb)
    gk = empty(1, nd, 2, L, o.N)
    ctx.expand_switch_keys(K, a_seed, [g], gb, gk)
    want_evk, want_gk = sr.relin_key_seeded(o, K, T, s, SEED), sr.galois_keys_seeded(o, K, T, s, SEED, [g])[0]
    assert np.array_equal(host(evk)[0], want_evk) and np.array_equal(host(gk)[0], want_gk)
    prod = empty(1, 2, Lq, o.N)
    ctx.ct_mul_relin_grouped(K, ct[0:1], ct[1:2], evk[0], prod, 1, T)
    rot = empty(1, 2, Lq, o.N)
    ctx.rotate_grouped(K, ct[0:1], g, gk[0], rot, 1, T)
    resc = empty(1, 2, Lq - 1, o.N)
    ctx.ct_mul_relin_rescale_grouped_level(K, Lq, ct[0:1], ct[1:2], evk[0], resc, 1, T)
    # the same calls with the restated ciphertexts and keys
    ref_ct = sr.encrypt_seeded(oq, T, s, SEED, 0, pt)
    prod2, rot2, resc2 = empty(1, 2, Lq, o.N), empty(1, 2, Lq, o.N), empty(1, 2, Lq - 1, o.N)
    ctx.ct_mul_relin_grouped(K, dev(ref_ct[0:1]), dev(ref_ct[1:2]), dev(want_evk), prod2, 1, T)
    ctx.rotate_grouped(K, dev(ref_ct[0:1]), g, dev(want_gk), rot2, 1, T)
    ctx.ct_mul_relin_rescale_grouped_level(K, Lq, dev(ref_ct[0:1]), dev(ref_ct[1:2]), dev(want_evk), resc2, 1, T)
    torch.cuda.synchronize()
    assert torch.equal(prod, prod2) and torch.equal(rot, rot2) and torch.equal(resc, resc2)
    assert np.array_equal(host(ct), ref_ct)
    assert np.array_equal(host(prod)[0], o.ct_mul_relin_grouped(K, ref_ct[0:1], ref_ct[1:2], want_evk, T)[0])
    full = np.convolve(m[0].astype(object), m[1].astype(object))
    mm = full[:o.N].copy()
    mm[:o.N - 1] -= full[o.N:]
    mm = np.array([int(x) % T for x in mm], dtype=np.int64)
    assert np.array_equal(oq.decrypt(s[:Lq], host(prod)[0], T), mm.astype(np.uint64))
    rm = np.zeros(o.N, dtype=np.int64)
    for k in range(o.N):
        e = k * g % (2 * o.N)
        rm[e % o.N] = (m[0, k] if e < o.N else -m[0, k]) % T
    assert np.array_equal(oq.decrypt(s[:Lq], host(rot)[0], T), rm.astype(np.uint64))
    # fresh seeded ciphertexts carry at most 21 t of noise, as symmetric encryption's (DESIGN.md section 2.14)
    assert _noise(oq, s, ref_ct[0], signed[0]) <= 21 * T
    ctx.close()


@pytest.fixture(scope="module")
def contract_rows():
    import seeded_contract as scn
    return scn.build_rows()


@pytest.mark.parametrize("shape", ["N4096-L3-K0", "N8192-L6-K2-l3", "N16384-L4-K0-l2"])
def test_guard_words_of_every_call(oracle_mod, contract_rows, shape):
    """every call of dpfhe_seeded.h through the memory-contract harness: outputs equal to the restatement, guard words and operands
    unchanged, outputs pre-filled with ones and with random words"""
    import deeppowers_b200 as dp
    import seeded_contract as scn
    from memory_contract import Shape
    from test_gpu_memory_contract import Refs, run_case
    s = {"N4096-L3-K0": Shape(12, 3, 0, 3, n_rot=3), "N8192-L6-K2-l3": Shape(13, 6, 2, 2, level=3, n_rot=2),
         "N16384-L4-K0-l2": Shape(14, 4, 0, 1, level=2, n_rot=2)}[shape]
    c = dp.Context(s.log_n, s.L)
    R = Refs(oracle_mod, s.log_n, s.L)
    ran = 0
    try:
        for fn, row in sorted(contract_rows.items()):
            if scn.runs_at(fn, s):
                run_case(row, c, R, s, 17)
                ran += 1
    finally:
        torch.cuda.synchronize()
        c.close()
    assert ran >= 9


def _guarded(shape, seed):
    """a device arena of random guard words with a region of `shape` in its middle: (arena, region view, guard length)"""
    n = int(np.prod(shape))
    g = 4100                       # guard words either side (an even count: the region stays 16-byte aligned)
    arena = torch.from_numpy(np.random.default_rng(seed).integers(0, 1 << 63, size=n + 2 * g, dtype=np.int64)).cuda()
    return arena, arena[g:g + n].view(shape), g


def test_upload_waits_for_pending_work_on_its_output(oracle_mod):
    """a pinned host source and work still pending on the output: the upload's copies are ordered after the kernels queued before it on
    the legacy default stream, and after the context's previous call on another stream; the words around the output stay unchanged"""
    L, n, first = 4, 512, 21
    ctx, o = _setup(oracle_mod, 13, L)
    s = kr.secret(o, SEED)
    a_seed = ctx.public_seed(SEED)
    pt = o.fill_uniform(14, n)
    c0 = empty(n, L, o.N)
    ctx.encrypt_seeded(T, dev(s), SEED, first, dev(pt), c0, n)
    want = empty(n, 2, L, o.N)
    ctx.expand_ciphertexts(a_seed, first, c0, want, n)
    h_c0 = torch.empty((n, L, o.N), dtype=torch.int64, pin_memory=True)
    h_c0.copy_(c0)
    h_np = h_c0.numpy().view(np.uint64)
    torch.cuda.synchronize()
    arena, up, g = _guarded((n, 2, L, o.N), 5)
    before = arena.clone()
    torch.cuda.synchronize()
    for _ in range(64):            # pending writes of the output on the legacy default stream when the upload starts
        up.add_(1)
    up.fill_(-1)
    ctx.upload_seeded_ciphertexts(a_seed, first, h_np, up)
    assert torch.equal(up, want)
    assert torch.equal(arena[:g], before[:g]) and torch.equal(arena[g + up.numel():], before[g + up.numel():])
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):  # the context's previous call, on another stream, writes the output
        for _ in range(8):
            ctx.expand_ciphertexts(a_seed, first + 1, c0, up, n, stream=side)
    ctx.upload_seeded_ciphertexts(a_seed, first, h_np, up)
    torch.cuda.synchronize()
    assert torch.equal(up, want)
    ctx.close()


def test_key_uploads_over_several_chunks(oracle_mod):
    """six keys of 16 MiB (N = 16384, L = 8, per-limb digits) are two chunks of the pipeline (four keys per 64 MiB): the upload and the
    host expansion keep each key's item number across chunks, equal the device expansion and write nothing around the output"""
    L = 8
    ctx, o = _setup(oracle_mod, 14, L)
    s = kr.secret(o, SEED)
    a_seed = ctx.public_seed(SEED)
    elts = [o.galois_elt(k) for k in (1, 2, 3, -1, -2)]
    items = [0] + elts
    b = empty(len(items), L, L, o.N)
    ctx.generate_relin_key_seeded(0, T, dev(s), SEED, b[0])
    ctx.generate_galois_keys_seeded(0, T, dev(s), elts, SEED, b[1:])
    keys = empty(len(items), L, 2, L, o.N)
    ctx.expand_switch_keys(0, a_seed, items, b, keys)
    hb = host(b).copy()
    arena, up, g = _guarded((len(items), L, 2, L, o.N), 6)
    before = arena.clone()
    n_launch = ctx.launch_count()
    ctx.upload_seeded_switch_keys(0, a_seed, items, hb, up)
    assert ctx.launch_count() - n_launch == 2     # one expansion per chunk
    assert torch.equal(up, keys)
    assert torch.equal(arena[:g], before[:g]) and torch.equal(arena[g + up.numel():], before[g + up.numel():])
    hk = np.empty((len(items), L, 2, L, o.N), dtype=np.uint64)
    ctx.expand_switch_keys_host(0, a_seed, items, hb, hk)
    assert np.array_equal(hk, host(keys))
    assert np.array_equal(hk[5], sr.galois_keys_seeded(o, 0, T, s, SEED, [elts[4]])[0])
    ctx.close()


def test_host_form_argument_checks(oracle_mod):
    """the uploads and the host expansion refuse a null seed, a bad level, a bad item number and (host expansion) an output over its
    input, before any copy or launch"""
    import deeppowers_b200 as dp
    L = 4
    ctx, o = _setup(oracle_mod, 12, L)
    a_seed = ctx.public_seed(SEED)
    h_c0 = np.zeros((2, L, o.N), dtype=np.uint64)
    up = torch.full((2, 2, L, o.N), 7, dtype=torch.int64, device="cuda")
    buf = np.full((3 * L * L * o.N,), 7, dtype=np.uint64)
    hb = buf[:L * L * o.N].reshape(1, L, L, o.N)
    hk_over = buf[L * L * o.N // 2:L * L * o.N // 2 + 2 * L * L * o.N].reshape(1, L, 2, L, o.N)
    hk = np.full((1, L, 2, L, o.N), 7, dtype=np.uint64)
    n_launch = ctx.launch_count()
    bad = [
        lambda: ctx.upload_seeded_ciphertexts(None, 0, h_c0, up),
        lambda: ctx._chk(ctx._l.dpfhe_upload_seeded_ciphertexts_level(ctx._h, 0, a_seed, 0, h_c0.ctypes.data, up.data_ptr(), 2)),
        lambda: ctx.upload_seeded_ciphertexts_level(L + 1, a_seed, 0, h_c0, up),
        lambda: ctx.upload_seeded_ciphertexts(a_seed, 0, h_c0, int(up.data_ptr()) + 8),
        lambda: ctx.expand_switch_keys_host(0, None, [0], hb, hk),
        lambda: ctx.expand_switch_keys_host(0, a_seed, [6], hb, hk),
        lambda: ctx.expand_switch_keys_host(5, a_seed, [0], hb, hk),
        lambda: ctx.expand_switch_keys_host(0, a_seed, [0], hb, hk_over),
        lambda: ctx.upload_seeded_switch_keys(0, a_seed, [2 * o.N + 1], hb, up),
    ]
    for call in bad:
        with pytest.raises(dp.DpfheError):
            call()
    torch.cuda.synchronize()
    assert ctx.launch_count() == n_launch
    assert bool((up == 7).all()) and np.all(hk == 7) and np.all(buf == 7)
    ctx.close()


def test_seeded_example(tmp_path):
    """examples/encrypted_seeded.cpp: the client writes seeded ciphertexts and a seeded relinearisation key as wire kinds 7 and 8, the
    server uploads them seeded and multiplies, the client decrypts every slot product"""
    import os
    import shutil
    import subprocess
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "deeppowers_b200")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "encrypted_seeded")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), "-I", os.path.join(cuda, "include"),
                           os.path.join(root, "examples", "encrypted_seeded.cpp"), "-L", libdir, "-ldpfhe", "-L", os.path.join(cuda, "lib64"),
                           "-lcudart", "-Wl,-rpath," + libdir + ":" + os.path.join(cuda, "lib64"), "-o", exe])
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "24576 slot products, 0 wrong" in r.stdout
