"""Scalar linear combinations and BGV polynomial evaluation on the GPU (DESIGN.md section 2.15): ct_lincomb and ct_add_plain bit for
bit against Python integers, PolyEval bit for bit against the restatement composed on the oracle (tests/polyeval_ref.py) and its
decryption against p(slots) mod t, the host form, argument checks, the launch count, two streams, and config 4 end to end."""
import numpy as np
import pytest

import bases
import polyeval_ref as pr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(90, 122))
T = 65537   # prime, 1 mod 2N up to N = 16384
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def _moduli(oracle_mod, logn, L, basis):
    return bases.catalogue(oracle_mod)[basis][:L] if basis else oracle_mod.Oracle(logn, L).moduli


@pytest.mark.parametrize("basis", [None, "gen_mixed"])
@pytest.mark.parametrize("n_terms", [1, 7, 8, 9, 64])
def test_lincomb_bit_exact(oracle_mod, basis, n_terms):
    """the extreme coefficients, inputs at q - 1, and the output aliasing the last input"""
    import deeppowers_b200 as dp
    logn, L, B = 12, 3, 2
    moduli = _moduli(oracle_mod, logn, L, basis)
    ctx = dp.Context(logn, L, moduli)
    o = oracle_mod.Oracle(logn, L, moduli)
    rng = np.random.default_rng(n_terms)
    cts = [o.fill_uniform(100 + i, 2 * B).reshape(B, 2, L, o.N) for i in range(n_terms)]
    for l, q in enumerate(moduli):
        cts[0][:, :, l, :16] = q - 1
    special = [I64_MIN, I64_MAX, 0, 1, -1]
    coeffs = [special[i] if i < len(special) else int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64)) for i in range(n_terms)]
    for constant in (I64_MIN, -12345):
        want = pr.lincomb(moduli, cts, coeffs, constant)
        d = [dev(c) for c in cts]
        out = empty(B, 2, L, o.N)
        ctx.ct_lincomb(d, coeffs, constant, out, B)
        assert np.array_equal(host(out), want)
        ctx.ct_lincomb(d, coeffs, constant, d[-1], B)   # out = an input
        assert np.array_equal(host(d[-1]), want)
    ctx.close()


@pytest.mark.parametrize("logn,basis", [(12, None), (14, "gen_mixed")])
def test_add_plain_bit_exact(oracle_mod, logn, basis):
    import deeppowers_b200 as dp
    L, B = 4, 3
    moduli = _moduli(oracle_mod, logn, L, basis)
    ctx = dp.Context(logn, L, moduli)
    o = oracle_mod.Oracle(logn, L, moduli)
    ct = o.fill_uniform(7, 2 * B).reshape(B, 2, L, o.N)
    pt = o.fill_uniform(8, 1).reshape(L, o.N)
    out = empty(B, 2, L, o.N)
    ctx.ct_add_plain(dev(ct), dev(pt), out, B)
    assert np.array_equal(host(out), pr.lincomb(moduli, [ct], [1], 0, pt))
    ctx.close()


def _setup_chain(oracle_mod, logn, Lq, K, basis, t=T, seed=SEED):
    """the key-switching context, the contexts over the ciphertext moduli, a device secret and the grouped key of the top level"""
    import deeppowers_b200 as dp
    L = Lq + K
    moduli = _moduli(oracle_mod, logn, L, basis)
    ctx = dp.Context(logn, L, moduli)
    sk = empty(L, ctx.N)
    ctx.generate_secret(seed, sk)
    key = empty(ctx.key_digits(K), 2, L, ctx.N)
    ctx.generate_relin_key(K, t, sk, seed, key)
    return ctx, moduli, sk, host(key)


def _encrypt_slots(ctx_q, sk, z, t, seed=SEED):
    B, Lq = z.shape[0], ctx_q.L
    pt, ct = empty(B, Lq, ctx_q.N), empty(B, 2, Lq, ctx_q.N)
    ctx_q.bgv_encode(dev(z), pt, B, t)
    ctx_q.encrypt(t, sk[:Lq].contiguous(), seed, 0, pt, ct, B)
    return ct


def _noise_bits(ctx_f, sk, ct):
    """bits of the largest centred coefficient of the phase of ct[0] under the first ctx_f.L limbs of the secret (message + t e:
    the message is below t, so this is the noise to within log2 t bits; it saturates at the modulus when decryption fails)"""
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


def _decrypt_slots(ctx_f, sk, ct, t):
    B, Lf = ct.shape[0], ctx_f.L
    ph, out = empty(B, Lf, ctx_f.N), empty(B, 2, ctx_f.N // 2)
    ctx_f.decrypt(sk[:Lf].contiguous(), ct, 2, ph, B)
    ctx_f.bgv_decode(ph, out, B, t)
    return host(out)


# (log N, Lq, K, basis, coefficients): K = 1, 2 at every N, K = 3, 4 where the depth allows, a generic basis, zero coefficients
CASES = [
    (12, 4, 1, None, [3, -1, 2, 5, 0, 7, 1, -4, 9]),
    (12, 4, 2, None, [1, 2, 3, 4, 5, 6, 7, 8]),
    (13, 4, 2, None, [0, 0, 1]),
    (14, 4, 2, None, [-5, 0, 0, 11]),
    (14, 3, 1, None, [2, 0, 0, 0, 1]),
    (12, 4, 2, "gen_mixed", [4, -3, 0, 2, 0, 0, 0, 0, 1]),
    (13, 4, 2, "gen_mixed", [7, 9]),
    (12, 5, 3, None, [1, 1, 1, 1, 1]),
    (12, 5, 4, None, [0, 3, 0, 2]),
    (12, 4, 2, None, [17, 0, 0, 0, 0, 0, 0, 0]),
]


@pytest.mark.parametrize("logn,Lq,K,basis,coeffs", CASES)
def test_polyeval_bit_exact_and_decrypts(oracle_mod, logn, Lq, K, basis, coeffs):
    import deeppowers_b200 as dp
    ctx, moduli, sk, key = _setup_chain(oracle_mod, logn, Lq, K, basis)
    N, B = ctx.N, 2
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    rng = np.random.default_rng(logn * 100 + Lq * 10 + K)
    z = rng.integers(0, T, (B, 2, N // 2), dtype=np.int64)
    ct = _encrypt_slots(ctx_q, sk, z, T)
    pe = dp.PolyEval(ctx, K, T, coeffs, key)
    Lf = pe.result_limbs
    assert Lf == Lq - pr.ceil_log2(len(coeffs) - 1)
    out = empty(B, 2, Lf, N)
    n0 = ctx.launch_count()
    pe.apply(ct, out, B)
    launches = ctx.launch_count() - n0
    stats = {}
    want = pr.polyeval(pr.Chain(oracle_mod, logn, moduli, K), T, coeffs, host(ct), key, stats=stats)
    assert np.array_equal(host(out), want)
    assert launches == stats["mul"] + 2 * stats["switch"] + stats["lincomb"]
    ctx_f = dp.Context(logn, Lf, moduli[:Lf])
    assert np.array_equal(_decrypt_slots(ctx_f, sk, out, T), pr.poly_mod_t(coeffs, z, T))
    pe.close()
    for c in (ctx_f, ctx_q, ctx):
        c.close()


def test_host_form_equals_device_form(oracle_mod, monkeypatch):
    """several pipeline chunks (a chunk of 3 ciphertexts over a batch of 8), and the scratch counted in the context's device bytes"""
    import deeppowers_b200 as dp
    logn, Lq, K, B = 12, 4, 2, 8
    ctx, moduli, sk, key = _setup_chain(oracle_mod, logn, Lq, K, None)
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    z = np.random.default_rng(3).integers(0, T, (B, 2, ctx.N // 2), dtype=np.int64)
    ct = _encrypt_slots(ctx_q, sk, z, T)
    before = ctx.device_bytes()
    pe = dp.PolyEval(ctx, K, T, [1, 0, 2, 0, 3], key)
    Lf = pe.result_limbs
    out = empty(B, 2, Lf, ctx.N)
    pe.apply(ct, out, B)
    assert ctx.device_bytes() > before
    monkeypatch.setenv("DPFHE_POLYEVAL_CHUNK", "3")
    h = np.empty((B, 2, Lf, ctx.N), dtype=np.uint64)
    pe.apply_host(host(ct), h)
    assert np.array_equal(h, host(out))
    alive = ctx.device_bytes()
    pe.close()
    assert ctx.device_bytes() < alive   # destroy releases the evaluator's keys, tables and scratch
    ctx_q.close()
    ctx.close()


def test_argument_errors(oracle_mod):
    import deeppowers_b200 as dp
    logn, Lq, K = 12, 4, 2
    ctx, moduli, sk, key = _setup_chain(oracle_mod, logn, Lq, K, None)
    with pytest.raises(dp.DpfheError):
        dp.PolyEval(ctx, K, T, [1] * 10, key)            # d = 9: D = 4 > Lq - 1
    with pytest.raises(dp.DpfheError):
        dp.PolyEval(ctx, 4, T, [1, 1, 1], key)           # 2K > L
    for t in (0, 1, 1 << 31):
        with pytest.raises(dp.DpfheError):
            dp.PolyEval(ctx, K, t, [1, 1], key)
    with pytest.raises(dp.DpfheError):
        dp.PolyEval(ctx, K, T, [1] * 66, key)            # d = 65
    ctx5 = dp.Context(logn, 5, moduli[:3] + moduli[4:])  # Lq = 3, K = 2: D <= 2, so degree 5 (D = 3) is too deep
    key5 = np.zeros((2, 2, 5, ctx.N), dtype=np.uint64)
    with pytest.raises(dp.DpfheError):
        dp.PolyEval(ctx5, K, T, [1] * 6, key5)
    lib, h = ctx._l, ctx._h
    cs = (dp.evaluator.C.c_int64 * 1)(1)
    pe = dp.evaluator.C.c_void_p()
    assert lib.dpfhe_polyeval_create_grouped(h, K, T, None, 1, key.ctypes.data, dp.evaluator.C.byref(pe)) == -1
    assert lib.dpfhe_polyeval_create_grouped(h, K, T, cs, 1, None, dp.evaluator.C.byref(pe)) == -1
    assert lib.dpfhe_polyeval_apply(None, None, None, 1, None) == -1
    ctq = dp.Context(logn, Lq, moduli[:Lq])
    x = empty(1, 2, Lq, ctx.N)
    with pytest.raises(dp.DpfheError):
        ctq.ct_lincomb([x] * 65, [1] * 65, 0, x, 1)
    with pytest.raises(dp.DpfheError):
        ctq.ct_lincomb([], [], 0, x, 1)
    ptrs = (dp.evaluator.C.c_void_p * 2)(x.data_ptr(), None)
    cs2 = (dp.evaluator.C.c_int64 * 2)(1, 1)
    assert lib.dpfhe_ct_lincomb(ctq._h, 2, ptrs, cs2, 0, x.data_ptr(), 1, None) == -1
    assert lib.dpfhe_ct_add_plain(ctq._h, x.data_ptr(), None, x.data_ptr(), 1, None) == -1
    pev = dp.PolyEval(ctx, K, T, [0, 1, 1], key)
    with pytest.raises(dp.DpfheError, match="overlap"):
        pev.apply(x, x, 1)
    pev.close()
    for c in (ctq, ctx5, ctx):
        c.close()


def test_two_streams_are_ordered(oracle_mod):
    """applications of one evaluator alternating between two streams share its scratch: the library orders them"""
    import deeppowers_b200 as dp
    logn, Lq, K, B = 13, 4, 2, 64
    ctx, moduli, sk, key = _setup_chain(oracle_mod, logn, Lq, K, None)
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    rng = np.random.default_rng(8)
    cts = [_encrypt_slots(ctx_q, sk, rng.integers(0, T, (B, 2, ctx.N // 2), dtype=np.int64), T) for _ in range(2)]
    pe = dp.PolyEval(ctx, K, T, [1, 2, 3, 4], key)
    Lf = pe.result_limbs
    refs = [empty(B, 2, Lf, ctx.N) for _ in range(2)]
    for c, r in zip(cts, refs):
        pe.apply(c, r, B)
        ctx.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [empty(B, 2, Lf, ctx.N) for _ in range(2)]
    for _ in range(3):
        pe.apply(cts[0], outs[0], B, stream=s1)
        pe.apply(cts[1], outs[1], B, stream=s2)
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert np.array_equal(host(o), host(r))
    pe.close()
    ctx_q.close()
    ctx.close()


def test_config4_linear_bias_activation(oracle_mod):
    """config 4 (N = 8192, 4 ciphertext limbs + 2 special primes, t = 167772161): device keys and encryption, the 768 x 768 layer,
    ct_add_plain of an encoded bias, then PolyEval for x^2 and for a cubic: the decoded slots are p(W x + b) mod t for 512 prompts.
    The noise of each result is measured and printed; the degree-7 polynomial of the same schedule, which ends on the one 60-bit
    limb q_0, is run and measured too but not asserted: at this t its noise exceeds q_0 / 2 (DESIGN.md section 2.15)."""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY, DIM, t = 13, 4, 2, 512, 32, 768, 167772161
    L = Lq + K
    torch.cuda.empty_cache()   # the layer's 15 GiB of scratch comes from cudaMalloc, which cannot use blocks torch keeps cached
    moduli = oracle_mod.Oracle(log_n, L).moduli
    ctx = dp.Context(log_n, L, moduli)
    N = ctx.N
    ctx_q = dp.Context(log_n, Lq, moduli[:Lq])
    seed = ctx.random_seed()
    sk = empty(L, N)
    ctx.generate_secret(seed, sk)
    elts = [ctx.galois_elt(b) for b in range(1, BABY + 1)]
    keys = empty(BABY, ctx.key_digits(K), 2, L, N)
    ctx.generate_galois_keys(K, t, sk, elts, seed, keys)
    kh = host(keys)
    rk = empty(ctx.key_digits(K), 2, L, N)
    ctx.generate_relin_key(K, t, sk, seed, rk)
    rng = np.random.default_rng(0xC0F4)
    W = rng.integers(-127, 128, (DIM, DIM))
    X = rng.integers(-127, 128, (B, DIM))
    bias = rng.integers(-1000, 1000, DIM)
    xs = np.zeros((B, 2, N // 2), dtype=np.int64)
    xs[:, 0, :DIM] = X
    xs[:, 0, DIM:2 * DIM] = X
    ds = np.zeros((DIM, 2, N // 2), dtype=np.int64)
    ar = np.arange(DIM)
    for d in range(DIM):
        ds[d, 0, :DIM] = W[ar, (ar + d) % DIM]
        ds[d] = np.roll(ds[d], (d // BABY) * BABY, axis=1)
    bs = np.zeros((1, 2, N // 2), dtype=np.int64)
    bs[0, 0, :DIM] = bias
    diags, xpt, bpt = empty(DIM, Lq, N), empty(B, Lq, N), empty(1, Lq, N)
    ctx_q.bgv_encode(dev(ds), diags, DIM, t)
    ctx_q.bgv_encode(dev(xs), xpt, B, t)
    ctx_q.bgv_encode(dev(bs), bpt, 1, t)
    skq = sk[:Lq].contiguous()
    ct = empty(B, 2, Lq, N)
    ctx_q.encrypt(t, skq, seed, 0, xpt, ct, B)
    layer = dp.LinearLayer.grouped(ctx, K, host(diags), BABY, np.ascontiguousarray(kh[:BABY - 1]), np.ascontiguousarray(kh[BABY - 1]), t)
    y = empty(B, 2, Lq, N)
    layer.apply(ct, y, B)
    layer.close()              # its scratch is not needed by the activations
    ctx_q.ct_add_plain(y, bpt[0], y, B)
    pre = ((X @ W.T) + bias) % t                                  # W x + b per prompt
    for coeffs in ([0, 0, 1], [5, -3, 0, 2], [5, -3, 0, 1, 0, 0, 2, 1]):
        pe = dp.PolyEval(ctx, K, t, coeffs, host(rk))
        Lf = pe.result_limbs
        out = empty(B, 2, Lf, N)
        pe.apply(y, out, B)
        ctx_f = dp.Context(log_n, Lf, moduli[:Lf])
        got = _decrypt_slots(ctx_f, sk, out, t)[:, 0, :DIM]
        want = pr.poly_mod_t(coeffs, pre, t)
        bits = _noise_bits(ctx_f, sk, out[:1])
        print("\n[config 4] degree %d: noise %d bits at %d limbs (%d bits of modulus), %d of %d slots right"
              % (len(coeffs) - 1, bits, Lf, sum(q.bit_length() for q in moduli[:Lf]), int((got == want).sum()), got.size))
        if len(coeffs) <= 4:
            assert np.array_equal(got, want), coeffs
        pe.close()
        ctx_f.close()
    ctx_q.close()
    ctx.close()


def test_cpp_mlp_example(tmp_path):
    """examples/encrypted_mlp.cpp links libdpfhe.so alone (layer -> add_plain -> PolyEval -> decrypt through the C++ classes) and gets
    every activation right"""
    import os
    import subprocess
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()   # the example runs in a process of its own and needs device memory this one may hold cached
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir, exe = os.path.join(root, "deeppowers_b200"), str(tmp_path / "encrypted_mlp")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "examples", "encrypted_mlp.cpp"), "-L", lib_dir, "-ldpfhe", "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "256 activations at 3 limbs, 0 wrong" in r.stdout


def test_partial_overlap_and_host_add_plain(oracle_mod):
    """ct_lincomb's output may be one of its inputs but not overlap one at another offset; ct_add_plain_host equals the device form"""
    import deeppowers_b200 as dp
    logn, L, B = 12, 3, 4
    ctx = dp.Context(logn, L)
    o = oracle_mod.Oracle(logn, L, ctx.moduli)
    buf = empty(B + 1, 2, L, o.N)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.ct_lincomb([buf[:B]], [3], 0, buf[1:], B)
    ct = o.fill_uniform(3, 2 * B).reshape(B, 2, L, o.N)
    pt = o.fill_uniform(4, 1).reshape(L, o.N)
    h = np.empty_like(ct)
    ctx.ct_add_plain_host(ct, pt, h)
    assert np.array_equal(h, pr.lincomb(ctx.moduli, [ct], [1], 0, pt))
    ctx.close()
