"""Public keys and public-key encryption on the GPU (DESIGN.md section 2.14): bit for bit against the restatement (tests/public_key_ref.py),
reproducibility, host forms, one launch per call, the restriction to the ciphertext moduli, BGV and CKKS round trips, argument checks,
config 4's prompts encrypted under the public key through the linear layer and PolyEval, and the C++ example."""
import os
import subprocess

import numpy as np
import pytest

import bases
import keys_ref as kr
import public_key_ref as pkr
import polyeval_ref as pr
from test_gpu_polyeval import _decrypt_slots, _noise_bits
from test_public_key_cpu import NOISE_BOUND

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

OWNER = bytes(range(7, 39))
ENCRYPTOR = bytes(range(140, 172))
T_BGV = 65537


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


@pytest.mark.parametrize("logn,L,basis", [(12, 3, None), (13, 4, None), (14, 3, None), (12, 6, "gen_mixed"), (14, 6, "gen_mixed")])
def test_public_key_bit_exact(oracle_mod, logn, L, basis):
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, OWNER)
    for t in (T_BGV, 0):
        want = pkr.public_keygen(o, t, s, OWNER)
        pk = empty(2, L, o.N)
        ctx.public_keygen(t, dev(s), OWNER, pk)
        assert np.array_equal(host(pk), want), t
        h = np.empty((2, L, o.N), dtype=np.uint64)
        ctx.public_keygen_host(t, s, OWNER, h)
        assert np.array_equal(h, want), t
    ctx.close()


# (log N, limbs, basis, t, n, first_index): n = 700 at N = 4096 spans several waves of the grid and crosses 2^32 in the item number
ENC_CASES = [(12, 2, None, T_BGV, 700, (1 << 32) - 350), (12, 6, "gen_mixed", 0, 5, 1000), (13, 4, None, T_BGV, 5, (1 << 40) + 3),
             (13, 6, "fast_mixed", 0, 3, 1000), (14, 3, None, T_BGV, 3, (1 << 33) + 1), (14, 6, "gen_mixed", 0, 2, 1000)]


@pytest.mark.parametrize("logn,L,basis,t,n,first", ENC_CASES)
def test_encrypt_public_bit_exact(oracle_mod, logn, L, basis, t, n, first):
    ctx, o = _setup(oracle_mod, logn, L, basis)
    pk = pkr.public_keygen(o, t, kr.secret(o, OWNER), OWNER)
    pt = o.fill_uniform(11, n)
    ct = empty(n, 2, L, o.N)
    ctx.encrypt_public(t, dev(pk), ENCRYPTOR, first, dev(pt), ct, n)
    got = host(ct)
    idx = range(n) if n < 50 else [0, 1, 263, 349, 350, 351, 528, n - 1]
    for k in idx:
        assert np.array_equal(got[k], pkr.encrypt_public(o, t, pk, ENCRYPTOR, first + k, pt[k:k + 1])[0]), k
    ctx.close()


def test_reproducible_from_seed_and_index(oracle_mod):
    ctx, o = _setup(oracle_mod, 13, 3)
    pk = dev(pkr.public_keygen(o, T_BGV, kr.secret(o, OWNER), OWNER))
    pt = dev(o.fill_uniform(3, 4))
    a, b, c = empty(4, 2, 3, o.N), empty(1, 2, 3, o.N), empty(4, 2, 3, o.N)
    ctx.encrypt_public(T_BGV, pk, ENCRYPTOR, 20, pt, a, 4)
    ctx.encrypt_public(T_BGV, pk, ENCRYPTOR, 22, pt[2:3], b, 1)
    ctx.encrypt_public(T_BGV, pk, ctx.random_seed(), 20, pt, c, 4)
    assert np.array_equal(host(a)[2], host(b)[0])
    for k in range(4):
        assert not np.array_equal(host(a)[k, 1], host(c)[k, 1])
    ctx.close()


def test_host_forms_equal_device_forms_and_one_launch_per_call(oracle_mod):
    """encrypt_public_host over several pipeline chunks keeps item numbers first_index + k; every device call is one launch"""
    ctx, o = _setup(oracle_mod, 12, 2)
    n = 1100   # 512 ciphertexts of 128 KiB per chunk
    s = kr.secret(o, OWNER)
    pk = empty(2, 2, o.N)
    n0 = ctx.launch_count()
    ctx.public_keygen(T_BGV, dev(s), OWNER, pk)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 1
    pt = o.fill_uniform(12, n)
    ct_d = empty(n, 2, 2, o.N)
    n0 = ctx.launch_count()
    ctx.encrypt_public(T_BGV, pk, ENCRYPTOR, 5, dev(pt), ct_d, n)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 1
    ct_h = np.empty((n, 2, 2, o.N), dtype=np.uint64)
    ctx.encrypt_public_host(T_BGV, host(pk), ENCRYPTOR, 5, pt, ct_h)
    assert np.array_equal(ct_h, host(ct_d))
    ctx.close()


def test_restriction_to_the_ciphertext_moduli(oracle_mod):
    """the public key of the full context (4 + 2 limbs) cut to the first 4 rows is the one generated on the context over them, and
    encrypts there bit for bit as that one does"""
    import deeppowers_b200 as dp
    logn, L, Lq = 13, 6, 4
    ctx, o = _setup(oracle_mod, logn, L)
    cq = dp.Context(logn, Lq, o.moduli[:Lq])
    sk = empty(L, o.N)
    ctx.generate_secret(OWNER, sk)
    pk, pkq = empty(2, L, o.N), empty(2, Lq, o.N)
    ctx.public_keygen(T_BGV, sk, OWNER, pk)
    cq.public_keygen(T_BGV, sk[:Lq].contiguous(), OWNER, pkq)
    cut = pk[:, :Lq].contiguous()
    assert np.array_equal(host(cut), host(pkq))
    pt = dev(oracle_mod.Oracle(logn, Lq, o.moduli[:Lq]).fill_uniform(4, 3))
    a, b = empty(3, 2, Lq, o.N), empty(3, 2, Lq, o.N)
    cq.encrypt_public(T_BGV, cut, ENCRYPTOR, 0, pt, a, 3)
    cq.encrypt_public(T_BGV, pkq, ENCRYPTOR, 0, pt, b, 3)
    assert np.array_equal(host(a), host(b))
    ctx.close()
    cq.close()


@pytest.mark.parametrize("logn", [12, 13, 14])
def test_bgv_round_trip(oracle_mod, logn):
    """device secret and public key, slots encoded and publicly encrypted on the device, decrypted and decoded exactly; the phase
    noise stays below the bound section 2.14 gives"""
    ctx, o = _setup(oracle_mod, logn, 3)
    sk, pk = empty(3, o.N), empty(2, 3, o.N)
    ctx.generate_secret(OWNER, sk)
    ctx.public_keygen(T_BGV, sk, OWNER, pk)
    z = np.random.default_rng(logn).integers(0, T_BGV, (8, 2, o.N // 2), dtype=np.int64)
    pt, ct, ph, out = empty(8, 3, o.N), empty(8, 2, 3, o.N), empty(8, 3, o.N), empty(8, 2, o.N // 2)
    ctx.bgv_encode(dev(z), pt, 8, T_BGV)
    ctx.encrypt_public(T_BGV, pk, ctx.random_seed(), 0, pt, ct, 8)
    ctx.decrypt(sk, ct, 2, ph, 8)
    ctx.bgv_decode(ph, out, 8, T_BGV)
    assert np.array_equal(host(out), z.astype(np.uint64))
    q = np.array(o.moduli, dtype=np.uint64)[:, None]
    d = o.ntt_inv((host(ph) + (q - host(pt))) % q)[:, 0].astype(np.int64)
    q0 = int(o.moduli[0])
    noise = np.where(d > q0 // 2, d - q0, d)
    assert np.all(noise % T_BGV == 0)
    worst = int(np.abs(noise // T_BGV).max())
    print("\n[public-key encryption] N = %d: largest centred phase noise %d t over 8 ciphertexts" % (o.N, worst))
    assert worst <= NOISE_BOUND[logn]
    ctx.close()


def test_ckks_round_trip(oracle_mod):
    """t = 0 at N = 4096, scale 2^40: every slot within N * NOISE_BOUND / scale of the input (the bound of section 2.14)"""
    logn, scale = 12, 2.0**40
    ctx, o = _setup(oracle_mod, logn, 3)
    sk, pk = empty(3, o.N), empty(2, 3, o.N)
    ctx.generate_secret(OWNER, sk)
    ctx.public_keygen(0, sk, OWNER, pk)
    rng = np.random.default_rng(9)
    z = (rng.uniform(-1, 1, (4, o.N // 2)) + 1j * rng.uniform(-1, 1, (4, o.N // 2))).astype(np.complex128)
    pt, ct, ph = empty(4, 3, o.N), empty(4, 2, 3, o.N), empty(4, 3, o.N)
    ctx.ckks_encode(torch.from_numpy(z).cuda(), pt, 4, scale)
    ctx.encrypt_public(0, pk, ENCRYPTOR, 0, pt, ct, 4)
    ctx.decrypt(sk, ct, 2, ph, 4)
    out = torch.empty((4, o.N // 2), dtype=torch.complex128, device="cuda")
    ctx.ckks_decode(ph, out, 4, scale)
    err = np.abs(out.cpu().numpy() - z).max()
    assert err < o.N * NOISE_BOUND[logn] / scale + 2.0**-30, err
    ctx.close()


def test_argument_checks(oracle_mod):
    import deeppowers_b200 as dp
    ctx, o = _setup(oracle_mod, 12, 2)
    P = 2 * o.N
    sk = empty(2, o.N)
    ctx.generate_secret(OWNER, sk)
    pk, pt, ct = empty(2, 2, o.N), empty(1, 2, o.N), empty(1, 2, 2, o.N)
    ctx.public_keygen(T_BGV, sk, OWNER, pk)
    lib, h = ctx._l, ctx._h
    assert lib.dpfhe_public_keygen(h, T_BGV, sk.data_ptr(), None, pk.data_ptr(), None) == -1
    assert lib.dpfhe_public_keygen(h, T_BGV, None, OWNER, pk.data_ptr(), None) == -1
    assert lib.dpfhe_public_keygen(h, T_BGV, sk.data_ptr(), OWNER, None, None) == -1
    assert lib.dpfhe_encrypt_public(h, T_BGV, None, ENCRYPTOR, 0, pt.data_ptr(), ct.data_ptr(), 1, None) == -1
    assert lib.dpfhe_encrypt_public(h, T_BGV, pk.data_ptr(), None, 0, pt.data_ptr(), ct.data_ptr(), 1, None) == -1
    assert lib.dpfhe_encrypt_public(h, T_BGV, pk.data_ptr(), ENCRYPTOR, 0, None, ct.data_ptr(), 1, None) == -1
    assert lib.dpfhe_encrypt_public(h, T_BGV, pk.data_ptr(), ENCRYPTOR, 0, pt.data_ptr(), None, 1, None) == -1
    hpt, hct = host(pt).copy(), host(ct).copy()
    assert lib.dpfhe_encrypt_public_host(h, T_BGV, None, ENCRYPTOR, 0, hpt.ctypes.data, hct.ctypes.data, 1) == -1
    with pytest.raises(ValueError):
        ctx.encrypt_public(T_BGV, pk, b"short", 0, pt, ct, 1)
    # overlaps: the public key over the secret, ciphertexts over the public key and over the plaintexts
    buf = empty(4 * P)
    skb = buf[P:2 * P]
    ctx.generate_secret(OWNER, skb)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.public_keygen(T_BGV, skb, OWNER, buf[:2 * P])
    pkb = buf[:2 * P]
    ctx.public_keygen(T_BGV, sk, OWNER, pkb)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.encrypt_public(T_BGV, pkb, ENCRYPTOR, 0, pt, buf[P:3 * P], 1)
    big = empty(3 * P)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.encrypt_public(T_BGV, pk, ENCRYPTOR, 0, big[:P], big[P // 2:P // 2 + 2 * P], 1)
    ctx.close()


def test_config4_prompts_encrypted_under_the_public_key(oracle_mod):
    """config 4 (N = 8192, 4 ciphertext limbs + 2 special primes, t = 167772161): the key owner makes the secret, the public key, the
    Galois keys and the relinearisation key; the 512 prompts are encrypted under the public key with another seed, go through
    LinearLayer.grouped, ct_add_plain of an encoded bias and PolyEval for x^2 and a cubic, and decode to p(W x + b) mod t.  The
    noise of each result is printed (section 2.15 records it next to the symmetric figures)"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY, DIM, t = 13, 4, 2, 512, 32, 768, 167772161
    L = Lq + K
    torch.cuda.empty_cache()
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
    del keys
    rk = empty(ctx.key_digits(K), 2, L, N)
    ctx.generate_relin_key(K, t, sk, seed, rk)
    skq = sk[:Lq].contiguous()
    pk = empty(2, Lq, N)
    ctx_q.public_keygen(t, skq, seed, pk)
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
    ct = empty(B, 2, Lq, N)
    ctx_q.encrypt_public(t, pk, ctx_q.random_seed(), 0, xpt, ct, B)   # the data owner's own seed; no secret
    print("\n[config 4, public key] fresh noise %d bits" % _noise_bits(ctx_q, sk, ct[:1]))
    layer = dp.LinearLayer.grouped(ctx, K, host(diags), BABY, np.ascontiguousarray(kh[:BABY - 1]), np.ascontiguousarray(kh[BABY - 1]), t)
    del diags
    y = empty(B, 2, Lq, N)
    layer.apply(ct, y, B)
    layer.close()
    ctx_q.ct_add_plain(y, bpt[0], y, B)
    print("[config 4, public key] after the layer and bias: %d bits" % _noise_bits(ctx_q, sk, y[:1]))
    pre = ((X @ W.T) + bias) % t
    for coeffs in ([0, 0, 1], [5, -3, 0, 2]):
        pe = dp.PolyEval(ctx, K, t, coeffs, host(rk))
        Lf = pe.result_limbs
        out = empty(B, 2, Lf, N)
        pe.apply(y, out, B)
        ctx_f = dp.Context(log_n, Lf, moduli[:Lf])
        got = _decrypt_slots(ctx_f, sk, out, t)[:, 0, :DIM]
        want = pr.poly_mod_t(coeffs, pre, t)
        bits = _noise_bits(ctx_f, sk, out[:1])
        print("[config 4, public key] degree %d: noise %d bits at %d limbs (%d bits of modulus), %d of %d slots right"
              % (len(coeffs) - 1, bits, Lf, sum(q.bit_length() for q in moduli[:Lf]), int((got == want).sum()), got.size))
        assert np.array_equal(got, want), coeffs
        pe.close()
        ctx_f.close()
    ctx_q.close()
    ctx.close()


def test_cpp_public_key_example(tmp_path):
    """examples/encrypted_public.cpp links libdpfhe.so alone: a data owner encrypts with PublicEncryptor and no secret, the key owner
    decrypts the product"""
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir, exe = os.path.join(root, "deeppowers_b200"), str(tmp_path / "encrypted_public")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "examples", "encrypted_public.cpp"), "-L", lib_dir, "-ldpfhe", "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "8192 slot products, 0 wrong" in r.stdout
