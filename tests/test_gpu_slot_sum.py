"""Summed rotations and slot sums on the GPU (DESIGN.md section 2.17): dpfhe_rotate_sum_grouped bit for bit against the oracle
restatement (tests/slot_sum_ref.py) with batches over several grid rounds, SlotSum against the restatement and the stage-by-stage
composition of the primitive, the host forms, the launch count, the object's scratch, the argument checks, config 4 summed after
its 768 x 768 layer, and a CKKS sum of 64 slots."""
import numpy as np
import pytest

import slot_sum_ref as ssr
from bases import catalogue

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(140, 172))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def _inputs(o, oq, K, n_rot, batch, seed):
    ct = oq.fill_uniform(seed, 2 * batch).reshape(batch, 2, oq.L, o.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    ct[-1, 0] = (q - 1)[:, None]
    dnum = o.grouped_digits(K)
    keys = o.fill_uniform(seed + 1, n_rot * 2 * dnum).reshape(n_rot, dnum, 2, o.L, o.N)
    galois = [o.galois_elt((m + 1) * (-1) ** m) for m in range(n_rot)]
    return ct, galois, keys


# (log N, K, Lq, n_rot, batch, basis): K = 1 .. 4 with ragged last digits, n_rot = 1, 2, 7, 15, every N, a generic basis; the
# batches of 260 and 150 span several rounds of the hoisting grid and of the summed kernel's grid
CASES = [
    (12, 1, 3, 15, 3, None),
    (12, 2, 4, 7, 260, None),
    (12, 2, 5, 2, 3, None),
    (12, 3, 4, 1, 3, None),
    (12, 4, 4, 15, 2, None),
    (13, 2, 4, 15, 3, None),
    (13, 1, 3, 1, 150, None),
    (14, 2, 4, 7, 3, None),
    (14, 3, 4, 2, 2, None),
    (12, 2, 4, 7, 3, "gen_mixed"),
]


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_rotate_sum_equals_the_restatement(oracle_mod, case):
    import deeppowers_b200 as dp
    log_n, K, Lq, n_rot, batch, basis = case
    moduli = catalogue(oracle_mod)[basis][:Lq + K] if basis else None
    o = oracle_mod.Oracle(log_n, Lq + K, moduli)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    ct, galois, keys = _inputs(o, oq, K, n_rot, batch, 7 * log_n + n_rot)
    ctx = dp.Context(log_n, Lq + K, o.moduli)
    out = empty(batch, 2, Lq, o.N)
    for t in (0, 65537):
        ctx.rotate_sum_grouped(K, dev(ct), galois, [dev(k) for k in keys], out, batch, t)
        assert np.array_equal(host(out).reshape(ct.shape), ssr.rotate_sum(o, K, ct, galois, keys, t)), t
    hout = np.zeros_like(ct)
    ctx.rotate_sum_grouped_host(K, ct, galois, np.ascontiguousarray(keys), hout, 65537)
    assert np.array_equal(hout, host(out).reshape(ct.shape))
    ctx.close()


def test_one_rotation_is_hoisted_rotation_plus_add(oracle_mod):
    import deeppowers_b200 as dp
    K, Lq, B = 2, 4, 5
    o = oracle_mod.Oracle(13, Lq + K)
    oq = oracle_mod.Oracle(13, Lq, o.moduli[:Lq])
    ct, galois, keys = _inputs(o, oq, K, 1, B, 3)
    ctx, ctx_q = dp.Context(13, Lq + K), dp.Context(13, Lq, o.moduli[:Lq])
    a, r, s = dev(ct), empty(1, B, 2, Lq, o.N), empty(B, 2, Lq, o.N)
    ctx.rotate_hoisted_grouped(K, a, galois, [dev(keys[0])], r, B, 65537)
    ctx_q.poly_add(r[0], a, r[0], 2 * B)
    ctx.rotate_sum_grouped(K, a, galois, [dev(keys[0])], s, B, 65537)
    assert torch.equal(r[0], s)
    ctx.close()
    ctx_q.close()


def _slotsum_keys(o, K, stride, radices, seed):
    n = len(ssr.steps(stride, radices))
    return o.fill_uniform(seed, n * 2 * o.grouped_digits(K)).reshape(n, o.grouped_digits(K), 2, o.L, o.N)


@pytest.mark.parametrize("log_n,K,Lq,stride,radices", [(12, 2, 4, 1, [4, 4, 4]), (13, 2, 4, 3, [16, 4]), (12, 1, 3, 1, [3, 4, 4, 4, 4]),
                                                       (14, 3, 4, 2, [8, 8])])
def test_slotsum_equals_restatement_and_composition(oracle_mod, log_n, K, Lq, stride, radices):
    import deeppowers_b200 as dp
    o = oracle_mod.Oracle(log_n, Lq + K)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    B, t = 3, 65537
    ct = oq.fill_uniform(11, 2 * B).reshape(B, 2, Lq, o.N)
    gks = _slotsum_keys(o, K, stride, radices, 12)
    ctx = dp.Context(log_n, Lq + K)
    ss = dp.SlotSum.grouped(ctx, K, stride, radices, gks, t)
    out = empty(B, 2, Lq, o.N)
    n0 = ctx.launch_count()
    ss.apply(dev(ct), out, B)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 4 * len(radices)
    got = host(out).reshape(ct.shape)
    assert np.array_equal(got, ssr.slot_sum(o, K, ct, stride, radices, gks, t))
    # the stage-by-stage composition of the primitive
    cur, k = dev(ct), 0
    for st in ssr.stage_steps(stride, radices):
        nxt = empty(B, 2, Lq, o.N)
        ctx.rotate_sum_grouped(K, cur, [ctx.galois_elt(s) for s in st], [dev(g) for g in gks[k:k + len(st)]], nxt, B, t)
        cur, k = nxt, k + len(st)
    assert torch.equal(cur, out)
    ss.close()
    ctx.close()


def test_host_form_scratch_and_launches(oracle_mod, monkeypatch):
    """apply_host over several chunks gives apply's bits; the object's scratch grows with the batch and is counted in the context's
    device bytes; 4 launches per stage and chunk"""
    import deeppowers_b200 as dp
    log_n, K, Lq, stride, radices = 12, 2, 4, 1, [4, 4, 4]
    o = oracle_mod.Oracle(log_n, Lq + K)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    B = 7
    ct = oq.fill_uniform(21, 2 * B).reshape(B, 2, Lq, o.N)
    gks = _slotsum_keys(o, K, stride, radices, 22)
    ctx = dp.Context(log_n, Lq + K)
    b0 = ctx.device_bytes()
    ss = dp.SlotSum.grouped(ctx, K, stride, radices, gks, 65537)
    b1 = ctx.device_bytes()
    assert b1 - b0 >= 2 * gks.nbytes   # keys and their companions
    out = empty(B, 2, Lq, o.N)
    ss.apply(dev(ct)[:2].contiguous(), out[:2], 2)
    b2 = ctx.device_bytes()
    ss.apply(dev(ct), out, B)
    b3 = ctx.device_bytes()
    assert b3 - b2 >= (B - 2) * 2 * Lq * o.N * 8   # the intermediate batch grew with it
    want = host(out).reshape(ct.shape)
    monkeypatch.setenv("DPFHE_SLOTSUM_CHUNK", "3")
    hout = np.zeros_like(ct)
    n0 = ctx.launch_count()
    ss.apply_host(ct, hout)
    assert ctx.launch_count() - n0 == 4 * len(radices) * 3   # chunks of 3, 3 and 1
    assert np.array_equal(hout, want)
    ss.close()
    assert ctx.device_bytes() < b3
    ctx.close()


def test_argument_checks(oracle_mod):
    """every rejected argument returns DPFHE_ERR_INVALID from the C ABI itself (the Python wrappers raise DpfheError on it)"""
    import ctypes as C
    import deeppowers_b200 as dp
    DPFHE_ERR_INVALID = -1
    K, Lq, N = 2, 4, 4096
    o = oracle_mod.Oracle(12, Lq + K)
    ctx = dp.Context(12, Lq + K)
    lib = ctx._l
    dnum = ctx.key_digits(K)
    key = empty(dnum, 2, Lq + K, N)
    ct, out = empty(2, 2, Lq, N), empty(2, 2, Lq, N)
    g = ctx.galois_elt(1)

    def rotate_sum(n_special=K, galois=(g,), t=0, dst=out):
        n = len(galois)
        ge = (C.c_uint64 * max(n, 1))(*[int(x) for x in galois])
        kp = (C.c_void_p * max(n, 1))(*[key.data_ptr()] * n)
        return lib.dpfhe_rotate_sum_grouped(ctx._h, n_special, C.c_void_p(ct.data_ptr()), n, ge, kp, C.c_void_p(dst.data_ptr()), 2, int(t), None)

    bad = [dict(n_special=0), dict(n_special=4), dict(galois=[g] * 16), dict(galois=[]), dict(galois=[2]), dict(galois=[2 * N + 1]),
           dict(t=o.moduli[-1]), dict(dst=ct)]
    for b in bad:
        assert rotate_sum(**b) == DPFHE_ERR_INVALID, b
        with pytest.raises(dp.DpfheError):
            gal = b.get("galois", [g])
            ctx.rotate_sum_grouped(b.get("n_special", K), ct, gal, [key] * len(gal), b.get("dst", out), 2, b.get("t", 0))
    assert rotate_sum() == 0
    gks = np.zeros((3, dnum, 2, Lq + K, N), dtype=np.uint64)

    def create(kk, stride, radices, t=0):
        rs = (C.c_uint * max(len(radices), 1))(*radices)
        h = C.c_void_p()
        rc = lib.dpfhe_slotsum_create_grouped(ctx._h, kk, stride, rs, len(radices), C.c_void_p(gks.ctypes.data), int(t), C.byref(h))
        assert (rc == 0) == bool(h.value)
        if h.value:
            lib.dpfhe_slotsum_destroy(h)
        return rc

    for stride, radices, kk in [(1, [4], 0), (1, [4], 4), (0, [4], K), (1, [1], K), (1, [17], K), (600, [4], K), (1, [2] * 17, K), (1, [], K)]:
        assert create(kk, stride, radices) == DPFHE_ERR_INVALID, (stride, radices, kk)
        with pytest.raises(dp.DpfheError):
            dp.SlotSum.grouped(ctx, kk, stride, radices, gks, 0)
    assert create(K, 1, [4], o.moduli[-1]) == DPFHE_ERR_INVALID
    assert create(K, 1, [4]) == 0
    ss = dp.SlotSum.grouped(ctx, K, 1, [4], gks, 0)
    assert lib.dpfhe_slotsum_apply(ss._h, C.c_void_p(ct.data_ptr()), C.c_void_p(ct.data_ptr()), 2, None) == DPFHE_ERR_INVALID   # in place
    assert lib.dpfhe_slotsum_apply(None, C.c_void_p(ct.data_ptr()), C.c_void_p(out.data_ptr()), 2, None) == DPFHE_ERR_INVALID
    ss.close()
    ctx.close()


def _noise_bits(ctx_f, sk, ct):
    """bits of the largest centred coefficient of the phase of ct[0] (message + t e: the noise to within log2 t bits)"""
    Lf = ctx_f.L
    ph = empty(1, Lf, ctx_f.N)
    ctx_f.decrypt(sk[:Lf].contiguous(), ct[:1].contiguous(), 2, ph, 1)
    ctx_f.ntt_inv(ph, 1)
    res = host(ph)[0]
    Q = 1
    for q in ctx_f.moduli:
        Q *= q
    X = sum(res[l].astype(object) * ((Q // q) * pow(Q // q, -1, q)) for l, q in enumerate(ctx_f.moduli)) % Q
    return max(abs(int(v) - Q if v > Q // 2 else int(v)) for v in X).bit_length()


def test_config4_sum_after_the_layer(oracle_mod):
    """config 4 (N = 8192, 4 ciphertext limbs + 2 special primes, t = 167772161): the 768 x 768 layer for 512 prompts, then a slot
    sum with radices {3, 4, 4, 4, 4}: slot 0 of each prompt decodes to sum_i (W x)_i mod t exactly; the noise before and after is
    printed"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY, DIM, t = 13, 4, 2, 512, 32, 768, 167772161
    radices = [3, 4, 4, 4, 4]
    L = Lq + K
    torch.cuda.empty_cache()
    moduli = oracle_mod.Oracle(log_n, L).moduli
    ctx = dp.Context(log_n, L, moduli)
    N = ctx.N
    ctx_q = dp.Context(log_n, Lq, moduli[:Lq])
    seed = ctx.random_seed()
    sk = empty(L, N)
    ctx.generate_secret(seed, sk)
    steps = dp.slotsum_steps(1, radices)
    elts = [ctx.galois_elt(b) for b in range(1, BABY + 1)] + [ctx.galois_elt(s) for s in steps]
    keys = empty(len(elts), ctx.key_digits(K), 2, L, N)
    ctx.generate_galois_keys(K, t, sk, elts, seed, keys)
    kh = host(keys)
    rng = np.random.default_rng(0xC0F45)
    W = rng.integers(-127, 128, (DIM, DIM))
    X = rng.integers(-127, 128, (B, DIM))
    xs = np.zeros((B, 2, N // 2), dtype=np.int64)
    xs[:, 0, :DIM] = X
    xs[:, 0, DIM:2 * DIM] = X
    ds = np.zeros((DIM, 2, N // 2), dtype=np.int64)
    ar = np.arange(DIM)
    for d in range(DIM):
        ds[d, 0, :DIM] = W[ar, (ar + d) % DIM]
        ds[d] = np.roll(ds[d], (d // BABY) * BABY, axis=1)
    diags, xpt = empty(DIM, Lq, N), empty(B, Lq, N)
    ctx_q.bgv_encode(dev(ds), diags, DIM, t)
    ctx_q.bgv_encode(dev(xs), xpt, B, t)
    ct = empty(B, 2, Lq, N)
    ctx_q.encrypt(t, sk[:Lq].contiguous(), seed, 0, xpt, ct, B)
    layer = dp.LinearLayer.grouped(ctx, K, host(diags), BABY, np.ascontiguousarray(kh[:BABY - 1]), np.ascontiguousarray(kh[BABY - 1]), t)
    y = empty(B, 2, Lq, N)
    layer.apply(ct, y, B)
    layer.close()
    ss = dp.SlotSum.grouped(ctx, K, 1, radices, np.ascontiguousarray(kh[BABY:]), t)
    z = empty(B, 2, Lq, N)
    ss.apply(y, z, B)
    ss.close()
    ph, out = empty(B, Lq, N), empty(B, 2, N // 2)
    ctx_q.decrypt(sk[:Lq].contiguous(), z, 2, ph, B)
    ctx_q.bgv_decode(ph, out, B, t)
    got = host(out)[:, 0, 0]
    want = ((X @ W.T).sum(axis=1) % t).astype(np.uint64)
    before, after = _noise_bits(ctx_q, sk, y), _noise_bits(ctx_q, sk, z)
    print("\n[config 4 slot sum] noise %d bits after the layer, %d bits after the 768-slot sum (%d bits of modulus), %d of %d right"
          % (before, after, sum(q.bit_length() for q in moduli[:Lq]), int((got == want).sum()), B))
    assert np.array_equal(got, want)
    ctx_q.close()
    ctx.close()


CKKS_ERR_BOUND = 2.0**-18   # measured worst case 1.83e-7 = 2^-22.4 on an H100: a margin of 2^4.4 (DESIGN.md section 2.17)


def test_ckks_sum_of_64_slots(oracle_mod):
    """slots uniform in [-1, 1] at scale 2^45, N = 8192, 4 ciphertext limbs + 2 special primes, radices {4, 4, 4}: each decoded slot
    is the exact sum of its 64-slot window to within CKKS_ERR_BOUND"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, scale = 13, 4, 2, 4, 2.0**45
    radices = [4, 4, 4]
    moduli = oracle_mod.Oracle(log_n, Lq + K).moduli
    ctx = dp.Context(log_n, Lq + K, moduli)
    ctx_q = dp.Context(log_n, Lq, moduli[:Lq])
    N = ctx.N
    sk = empty(Lq + K, N)
    ctx.generate_secret(SEED, sk)
    steps = dp.slotsum_steps(1, radices)
    keys = empty(len(steps), ctx.key_digits(K), 2, Lq + K, N)
    ctx.generate_galois_keys(K, 0, sk, [ctx.galois_elt(s) for s in steps], SEED, keys)
    rng = np.random.default_rng(64)
    zs = rng.uniform(-1, 1, (B, N // 2)).astype(np.complex128)
    pt, ct = empty(B, Lq, N), empty(B, 2, Lq, N)
    ctx_q.ckks_encode(torch.from_numpy(zs).cuda(), pt, B, scale)
    ctx_q.encrypt(0, sk[:Lq].contiguous(), SEED, 0, pt, ct, B)
    ss = dp.SlotSum.grouped(ctx, K, 1, radices, host(keys), 0)
    out = empty(B, 2, Lq, N)
    ss.apply(ct, out, B)
    ph = empty(B, Lq, N)
    ctx_q.decrypt(sk[:Lq].contiguous(), out, 2, ph, B)
    dec = torch.empty((B, N // 2), dtype=torch.complex128, device="cuda")
    ctx_q.ckks_decode(ph, dec, B, scale)
    got = dec.cpu().numpy()
    want = sum(np.roll(zs, -j, axis=1) for j in range(64))
    err = float(np.max(np.abs(got - want)))
    print("\n[ckks slot sum] worst |decoded - exact| = %.3g (2^%.1f) over %d slots" % (err, np.log2(err), got.size))
    assert err < CKKS_ERR_BOUND
    ss.close()
    ctx_q.close()
    ctx.close()


def test_attention_scores_example(tmp_path):
    """examples/encrypted_attention_scores.cpp links libdpfhe.so alone (encrypt -> multiply_relin_grouped -> SlotSum -> decrypt through
    the C++ classes) and gets every score q_h . k_h right"""
    import os
    import subprocess
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()   # the example runs in a process of its own
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir, exe = os.path.join(root, "deeppowers_b200"), str(tmp_path / "encrypted_attention_scores")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "examples", "encrypted_attention_scores.cpp"), "-L", lib_dir, "-ldpfhe", "-Wl,-rpath," + lib_dir,
                           "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "64 attention scores, 0 wrong" in r.stdout
