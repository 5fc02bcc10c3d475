"""Polynomial evaluation at level l on the top-level context (DESIGN.md section 2.22): PolyEval(..., level=l) and PolyEval.ckks(...,
level=l) bit for bit against the top-level object on a context over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with the key restricted to it
(tests/polyeval_ref.py:restrict_key) and against the restatements, for K = 1 .. 4 with ragged last digits and every valid level, at
degree 1 (one lincomb at the level) and the deepest degree the level allows; level = Lq against the existing object, bits and launches;
the depth errors name the level; a BGV and a CKKS network on ONE context with ONE key set; and examples/encrypted_deep_mlp.cpp."""
import os
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ckks_polyeval_ref as cr  # noqa: E402
import polyeval_ref as pr  # noqa: E402
from test_gpu_parity import dev, dp, host  # noqa: E402,F401  (dp is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 65537
SEED = bytes(range(40, 72))
# (K, Lq): every K with a ragged last digit at the top
CHAINS = [(1, 3), (2, 5), (3, 5), (4, 6)]


@pytest.fixture
def made():
    objs = []
    torch.cuda.empty_cache()
    yield objs
    torch.cuda.synchronize()
    for o in reversed(objs):
        o.close()
    torch.cuda.empty_cache()


def _uniform(rng, mods, shape):
    out = np.empty(shape, dtype=np.uint64)
    for i, q in enumerate(mods):
        out[..., i, :] = rng.integers(0, int(q), size=out[..., i, :].shape, dtype=np.uint64)
    return out


def _relin(c, K, t):
    sk = torch.empty((c.L, c.N), dtype=torch.int64, device="cuda")
    c.generate_secret(SEED, sk)
    evk = torch.empty((c.grouped_digits(K), 2, c.L, c.N), dtype=torch.int64, device="cuda")
    c.generate_relin_key(K, t, sk, bytes(range(1, 33)), evk)
    return sk, host(evk).reshape(evk.shape)


def _max_degree(l, K, ckks):
    D = min(l - 2, l - K + 1) if ckks else min(l - 1, l - K + 1)
    return 1 << D if D >= 0 else 0


def _coeffs(rng, d, ckks):
    if ckks:
        return list(rng.uniform(-1, 1, d + 1) / (d + 1))
    return [int(v) for v in rng.integers(-1000, 1000, d + 1)]


def _check_level(dp, made, c, mods, K, Lq, l, key, coeffs, ckks, rng, batch=3, oracle=None):
    """the level object on c against the top-level object on the level context; returns the result"""
    N = c.N
    scale = float(mods[1]) if ckks else None
    low = dp.Context(c.log_n, l + K, mods[:l] + mods[Lq:])
    made.append(low)
    klow = np.ascontiguousarray(pr.restrict_key(key, Lq, K, l))
    if ckks:
        pe = dp.PolyEval.ckks(c, K, coeffs, scale, key, level=l)
        ref = dp.PolyEval.ckks(low, K, coeffs, scale, klow)
    else:
        pe = dp.PolyEval(c, K, T, coeffs, key, level=l)
        ref = dp.PolyEval(low, K, T, coeffs, klow)
    made += [pe, ref]
    assert pe.result_limbs == ref.result_limbs and pe.result_scale == ref.result_scale
    ct = dev(_uniform(rng, mods[:l], (batch, 2, l, N)))
    got = torch.full((batch, 2, pe.result_limbs, N), -1, dtype=torch.int64, device="cuda")
    want = torch.full_like(got, -1)
    n0, m0 = c.launch_count(), low.launch_count()
    pe.apply(ct, got, batch)
    ref.apply(ct, want, batch)
    torch.cuda.synchronize()
    assert torch.equal(got, want), (K, Lq, l, len(coeffs) - 1)
    assert c.launch_count() - n0 == low.launch_count() - m0
    if oracle is not None:   # the restatement of the object, on the level's chain with the restricted key
        chain = pr.Chain(oracle, c.log_n, mods[:l] + mods[Lq:], K)
        x = host(ct)
        r = cr.polyeval(chain, coeffs, scale, x, klow, scale) if ckks else pr.polyeval(chain, T, coeffs, x, klow)
        assert np.array_equal(host(got), np.asarray(r, dtype=np.uint64).reshape(host(got).shape))
    return got


@pytest.mark.parametrize("ckks", [False, True], ids=["bgv", "ckks"])
@pytest.mark.parametrize("K,Lq", CHAINS)
def test_every_level_against_level_context(dp, oracle_mod, made, K, Lq, ckks):
    import deeppowers_b200
    log_n = 12
    mods = cr.ckks_chain(oracle_mod, Lq, K) if ckks else None
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    made.append(c)
    mods = [int(q) for q in c.moduli]
    _, key = _relin(c, K, 0 if ckks else T)
    rng = np.random.default_rng(10 * K + Lq)
    for l in range(K, Lq + 1):
        degrees = sorted({d for d in (1, _max_degree(l, K, ckks)) if d >= 1 and (not ckks or l >= 2 + (d > 1))})
        if ckks and l < 2:
            degrees = []
        for d in degrees:
            _check_level(dp, made, c, mods, K, Lq, l, key, _coeffs(rng, d, ckks), ckks, rng, oracle=oracle_mod if d == degrees[-1] else None)


@pytest.mark.parametrize("ckks", [False, True], ids=["bgv", "ckks"])
def test_level_lq_is_the_top_level_object(dp, oracle_mod, made, ckks):
    import deeppowers_b200
    K, Lq, log_n = 2, 5, 13
    mods = cr.ckks_chain(oracle_mod, Lq, K) if ckks else None
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    made.append(c)
    _, key = _relin(c, K, 0 if ckks else T)
    rng = np.random.default_rng(3)
    coeffs = _coeffs(rng, 7, ckks)
    scale = float(c.moduli[1])
    mk = (lambda **kw: dp.PolyEval.ckks(c, K, coeffs, scale, key, **kw)) if ckks else (lambda **kw: dp.PolyEval(c, K, T, coeffs, key, **kw))
    top, at = mk(), mk(level=Lq)
    made += [top, at]
    ct = dev(_uniform(rng, c.moduli[:Lq], (4, 2, Lq, c.N)))
    a = torch.empty((4, 2, top.result_limbs, c.N), dtype=torch.int64, device="cuda")
    b = torch.empty_like(a)
    n0 = c.launch_count()
    top.apply(ct, a, 4)
    n1 = c.launch_count()
    at.apply(ct, b, 4)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert c.launch_count() - n1 == n1 - n0


def test_depth_errors_name_the_level(dp, made):
    import deeppowers_b200
    K, Lq = 2, 5
    c = deeppowers_b200.Context(12, Lq + K)
    made.append(c)
    _, key = _relin(c, K, T)
    for l in (0, 1, Lq + 1):
        with pytest.raises(RuntimeError, match="level %d" % l):
            dp.PolyEval(c, K, T, [1, 2], key, level=l)
    # level 3: D <= min(2, 2); degree 5 needs D = 3
    with pytest.raises(RuntimeError, match="level 3: degree 5 needs 3 levels"):
        dp.PolyEval(c, K, T, [1] * 6, key, level=3)
    # CKKS at level 3: D + 2 <= 3, degree 3 needs D = 2
    with pytest.raises(RuntimeError, match="level 3: degree 3 needs 2 levels"):
        dp.PolyEval.ckks(c, K, [0.5] * 4, 2.0 ** 40, key, level=3)
    made.append(dp.PolyEval(c, K, T, [1] * 5, key, level=3))   # D = 2: the deepest level 3 allows


def _bsgs_periodic(W, baby, half):
    """the diagonals of an M x M matrix for inputs that repeat with period M across the slot row: diagonal d holds W[i % M][(i + d) % M]
    in slot i + (d // baby) * baby (mod N/2) of the first row, so that every layer's output is the next layer's periodic input"""
    M = W.shape[0]
    out = np.zeros((M, 2 * half), dtype=np.int64)
    i = np.arange(half)
    for d in range(M):
        out[d, (i + (d // baby) * baby) % half] = W[i % M, (i % M + d) % M]
    return out


def _margin_bits(c, mods, sk, ct):
    """log2(Q / 2) - log2(max |phase|) of ct at its level l, decrypted on the top context and centred mod Q = q_0 .. q_{l-1}: how many
    bits the noise may still grow before decryption fails"""
    B, l, N = ct.shape[0], ct.shape[2], c.N
    part = torch.empty((B, l, N), dtype=torch.int64, device="cuda")
    c.decrypt_level(l, sk, ct.contiguous(), 2, part, B)
    ph = torch.zeros((B, c.L, N), dtype=torch.int64, device="cuda")
    ph[:, :l] = part
    c.ntt_inv(ph, B)   # row by row: the first l rows are the prefix's coefficients
    torch.cuda.synchronize()
    r = host(ph)[:, :l].astype(object)
    low = [int(q) for q in mods[:l]]
    Q = 1
    for q in low:
        Q *= q
    x = 0
    for i, q in enumerate(low):
        Qi = Q // q
        x = x + r[:, i, :] * (Qi * pow(Qi, -1, q))
    x = x % Q
    x = np.where(x > Q // 2, x - Q, x)
    worst = max(int(abs(v)) for v in x.reshape(-1))
    return (Q // 2).bit_length() - max(worst, 1).bit_length()


def test_bgv_deep_network_on_one_context(dp, made):
    """W1 -> + b1 -> p -> W2 at Lf1 -> + b2 at Lf1 -> p at Lf1 -> W3, with one context, one relinearisation key and one set of Galois
    keys; encoded and encrypted at Lq, decrypted and decoded at the result's level, slot for slot the exact result mod t.  Prints the
    phase margin after each stage (DESIGN.md section 2.22 records it)."""
    import deeppowers_b200
    K, Lq, log_n, t, DIM, BABY, B = 2, 5, 13, 65537, 16, 4, 2
    coeffs = [3, -2, 1]
    L = Lq + K
    c = deeppowers_b200.Context(log_n, L)
    made.append(c)
    mods = [int(q) for q in c.moduli]
    N, half = c.N, c.N // 2
    sk, evk = _relin(c, K, t)
    gk = torch.empty((BABY, c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, t, sk, [c.galois_elt(s) for s in range(1, BABY + 1)], bytes(range(2, 34)), gk)
    hk = host(gk).reshape(gk.shape)
    kb, kg = np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1]
    rng = np.random.default_rng(51)
    W = [rng.integers(-8, 9, size=(DIM, DIM)) for _ in range(3)]
    x = rng.integers(-8, 9, size=(B, DIM))
    b1, b2 = rng.integers(-50, 51, size=DIM), rng.integers(-50, 51, size=DIM)
    i = np.arange(half)

    def periodic(v):
        s = np.zeros((v.shape[0], N), dtype=np.int64)
        s[:, :half] = v[:, i % DIM]
        return s

    def encode(slots, level):
        pt = torch.empty((slots.shape[0], level, N), dtype=torch.int64, device="cuda")
        c.bgv_encode_level(level, torch.from_numpy(np.ascontiguousarray(slots)).cuda(), pt, slots.shape[0], t)
        return pt

    pe1 = dp.PolyEval(c, K, t, coeffs, evk)
    Lf1 = pe1.result_limbs
    pe2 = dp.PolyEval(c, K, t, coeffs, evk, level=Lf1)
    Lf2 = pe2.result_limbs
    layers = [dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[0], BABY, half), Lq)).reshape(DIM, Lq, N), BABY, kb, kg, t),
              dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[1], BABY, half), Lf1)).reshape(DIM, Lf1, N), BABY, kb, kg, t, level=Lf1),
              dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[2], BABY, half), Lf2)).reshape(DIM, Lf2, N), BABY, kb, kg, t, level=Lf2)]
    made += [pe1, pe2] + layers
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.encrypt_level(Lq, t, sk, SEED, 0, encode(periodic(x), Lq), ct, B)
    margins = {"x at %d" % Lq: _margin_bits(c, mods, sk, ct)}
    y1 = torch.empty_like(ct)
    layers[0].apply(ct, y1, B)
    c.ct_add_plain_level(Lq, y1, encode(periodic(b1[None]), Lq)[0], y1, B)
    margins["W1 x + b1"] = _margin_bits(c, mods, sk, y1)
    h1 = torch.empty((B, 2, Lf1, N), dtype=torch.int64, device="cuda")
    pe1.apply(y1, h1, B)
    margins["p(.) at %d" % Lf1] = _margin_bits(c, mods, sk, h1)
    y2 = torch.empty_like(h1)
    layers[1].apply(h1, y2, B)
    c.ct_add_plain_level(Lf1, y2, encode(periodic(b2[None]), Lf1)[0], y2, B)
    margins["W2 h + b2 at %d" % Lf1] = _margin_bits(c, mods, sk, y2)
    h2 = torch.empty((B, 2, Lf2, N), dtype=torch.int64, device="cuda")
    pe2.apply(y2, h2, B)
    margins["p(.) at %d" % Lf2] = _margin_bits(c, mods, sk, h2)
    y3 = torch.empty_like(h2)
    layers[2].apply(h2, y3, B)
    margins["W3 h at %d" % Lf2] = _margin_bits(c, mods, sk, y3)
    ph = torch.empty((B, Lf2, N), dtype=torch.int64, device="cuda")
    c.decrypt_level(Lf2, sk, y3, 2, ph, B)
    out = torch.empty((B, N), dtype=torch.int64, device="cuda")
    c.bgv_decode_level(Lf2, ph, out, B, t)

    def p(v):
        return sum(int(a) * v ** k for k, a in enumerate(coeffs)) % t

    act = np.vectorize(p, otypes=[object])
    o = lambda a: a.astype(object)
    h = act((o(x) @ o(W[0]).T + o(b1)) % t)
    h = act((h @ o(W[1]).T + o(b2)) % t)
    want = (h @ o(W[2]).T) % t
    got = host(out)[:, :DIM].astype(object)
    print("BGV three-layer network on one context (Lq = %d, K = %d, N = %d), phase margins in bits: %s" % (Lq, K, N, margins))
    assert np.array_equal(got, want)
    assert min(margins.values()) >= 10, margins


def test_ckks_chain_on_one_context(dp, oracle_mod, made):
    """W1 -> mod_switch_down_level -> CkksPolyEval at that level -> W2 at its result level -> mod_switch_down_level -> decode_level, on
    one context, within a tolerance derived from the scales"""
    import deeppowers_b200
    K, Lq, log_n, DIM, BABY, B = 2, 6, 13, 16, 4, 2
    mods = cr.ckks_chain(oracle_mod, Lq, K)
    c = deeppowers_b200.Context(log_n, Lq + K, mods)
    made.append(c)
    N, half = c.N, c.N // 2
    sk, evk = _relin(c, K, 0)
    gk = torch.empty((BABY, c.grouped_digits(K), 2, Lq + K, N), dtype=torch.int64, device="cuda")
    c.generate_galois_keys(K, 0, sk, [c.galois_elt(s) for s in range(1, BABY + 1)], bytes(range(2, 34)), gk)
    hk = host(gk).reshape(gk.shape)
    kb, kg = np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1]
    rng = np.random.default_rng(43)
    W1, W2 = rng.uniform(-1, 1, (DIM, DIM)) / DIM, rng.uniform(-1, 1, (DIM, DIM)) / DIM
    xv = rng.uniform(-1, 1, (B, DIM))
    i = np.arange(half)
    scale = float(mods[1])

    def diags(W, level, wscale):
        d = np.zeros((DIM, half), dtype=np.complex128)
        for k in range(DIM):
            d[k, (i + (k // BABY) * BABY) % half] = W[i % DIM, (i % DIM + k) % DIM]
        pt = torch.empty((DIM, level, N), dtype=torch.int64, device="cuda")
        c.ckks_encode_level(level, torch.from_numpy(d).cuda(), pt, DIM, wscale)
        return host(pt).reshape(DIM, level, N)

    z = np.zeros((B, half), dtype=np.complex128)
    z[:] = xv[:, i % DIM]
    pts = torch.empty((B, Lq, N), dtype=torch.int64, device="cuda")
    c.ckks_encode_level(Lq, torch.from_numpy(z).cuda(), pts, B, scale)
    ct = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.encrypt_level(Lq, 0, sk, SEED, 0, pts, ct, B)
    w1scale = float(mods[Lq - 1])   # the product is divided by q_{Lq-1} afterwards: the scale stays `scale`
    layer1 = dp.LinearLayer.grouped(c, K, diags(W1, Lq, w1scale), BABY, kb, kg, 0)
    made.append(layer1)
    y = torch.empty_like(ct)
    layer1.apply(ct, y, B)
    l1 = Lq - 1
    r1 = torch.empty((B, 2, l1, N), dtype=torch.int64, device="cuda")
    c.mod_switch_down_level(Lq, y, r1, 2 * B, 0)
    s1 = scale * w1scale / mods[Lq - 1]
    pe = dp.PolyEval.ckks(c, K, [0.5, 0.25, 0.125], s1, evk, level=l1)
    made.append(pe)
    Lf = pe.result_limbs
    h = torch.empty((B, 2, Lf, N), dtype=torch.int64, device="cuda")
    pe.apply(r1, h, B)
    w2scale = float(mods[Lf - 1])
    layer2 = dp.LinearLayer.grouped(c, K, diags(W2, Lf, w2scale), BABY, kb, kg, 0, level=Lf)
    made.append(layer2)
    w = torch.empty_like(h)
    layer2.apply(h, w, B)
    r2 = torch.empty((B, 2, Lf - 1, N), dtype=torch.int64, device="cuda")
    c.mod_switch_down_level(Lf, w, r2, 2 * B, 0)
    out_scale = pe.result_scale * w2scale / mods[Lf - 1]
    ph = torch.empty((B, Lf - 1, N), dtype=torch.int64, device="cuda")
    c.decrypt_level(Lf - 1, sk, r2, 2, ph, B)
    out = torch.empty((B, half), dtype=torch.complex128, device="cuda")
    c.ckks_decode_level(Lf - 1, ph, out, B, out_scale)
    a = xv @ W1.T
    want = (0.5 + 0.25 * a + 0.125 * a ** 2) @ W2.T
    err = np.abs(out.cpu().numpy()[:, :DIM] - want).max()
    # the rounding of each encoding and rescale relative to its scale, times the layers' DIM terms
    tol = DIM * DIM * 8.0 * (N / scale + N / w1scale + N / s1 + N / pe.result_scale + N / w2scale + N / out_scale)
    print("CKKS chain on one context: result at %d limbs, scale 2^%.2f, error 2^%.2f, tolerance 2^%.2f" %
          (Lf - 1, np.log2(out_scale), np.log2(err), np.log2(tol)))
    assert err < tol, (err, tol)


def test_deep_mlp_example(tmp_path):
    """examples/encrypted_deep_mlp.cpp: three layers on one evaluator"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    libdir = os.path.join(ROOT, "deeppowers_b200")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "encrypted_deep_mlp")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda, "include"),
                           os.path.join(ROOT, "examples", "encrypted_deep_mlp.cpp"), "-L", libdir, "-ldpfhe", "-L", os.path.join(cuda, "lib64"),
                           "-lcudart", "-Wl,-rpath," + libdir + ":" + os.path.join(cuda, "lib64"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert " 0 wrong" in r.stdout
