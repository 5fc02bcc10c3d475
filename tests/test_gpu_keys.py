"""Key generation, encryption and decryption on the GPU (DESIGN.md section 2.14): bit for bit against the restatement
(tests/keys_ref.py), decryption against the oracle's phase, and device-generated keys and ciphertexts through the evaluator and the
slot encoders end to end."""
import numpy as np
import pytest

import bases
import keys_ref as kr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(7, 39))
T_BGV = 65537   # prime, 1 mod 2N up to N = 16384


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
def test_secret_bit_exact(oracle_mod, logn, L, basis):
    ctx, o = _setup(oracle_mod, logn, L, basis)
    sk = empty(L, o.N)
    ctx.generate_secret(SEED, sk)
    want = kr.secret(o, SEED)
    assert np.array_equal(host(sk), want)
    h = np.empty((L, o.N), dtype=np.uint64)
    ctx.generate_secret_host(SEED, h)
    assert np.array_equal(h, want)
    ctx.close()


@pytest.mark.parametrize("K", [0, 1, 2, 3, 4])
def test_relin_keys_bit_exact(oracle_mod, K):
    """K = 0: per-limb digits; K = 1 the hybrid key; K = 3 has a ragged last digit (5 ciphertext limbs in digits of 3 and 2)"""
    L = 8
    ctx, o = _setup(oracle_mod, 12, L)
    s = kr.secret(o, SEED)
    nd = ctx.key_digits(K)
    key = empty(nd, 2, L, o.N)
    ctx.generate_relin_key(K, T_BGV, dev(s), SEED, key)
    assert np.array_equal(host(key), kr.relin_key(o, K, T_BGV, s, SEED))
    ctx.close()


@pytest.mark.parametrize("logn,L,K,basis", [(12, 4, 0, None), (12, 6, 2, "gen_mixed"), (13, 4, 1, None), (14, 3, 0, None), (14, 6, 3, "fast_mixed")])
def test_galois_keys_bit_exact(oracle_mod, logn, L, K, basis):
    """several elements in one call, the conjugation among them; N = 16384 runs the CTA-pair kernel"""
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, SEED)
    elts = [o.galois_elt(1), o.galois_elt(-3), 2 * o.N - 1]
    nd = ctx.key_digits(K)
    keys = empty(len(elts), nd, 2, L, o.N)
    ctx.generate_galois_keys(K, 0, dev(s), elts, SEED, keys)
    want = kr.galois_keys(o, K, 0, s, SEED, elts)
    assert np.array_equal(host(keys), want)
    h = np.empty((len(elts), nd, 2, L, o.N), dtype=np.uint64)
    ctx.generate_galois_keys_host(K, 0, s, elts, SEED, h)
    assert np.array_equal(h, want)
    hk = np.empty((nd, 2, L, o.N), dtype=np.uint64)
    ctx.generate_relin_key_host(K, 0, s, SEED, hk)
    assert np.array_equal(hk, kr.relin_key(o, K, 0, s, SEED))
    ctx.close()


def test_galois_keys_beyond_one_launch(oracle_mod):
    """more elements than one launch carries (KEYS_MAX_ELTS = 64): the key of every element is its own"""
    ctx, o = _setup(oracle_mod, 12, 2)
    s = kr.secret(o, SEED)
    elts = [o.galois_elt(k) for k in range(1, 71)]
    keys = empty(len(elts), 2, 2, 2, o.N)
    ctx.generate_galois_keys(0, T_BGV, dev(s), elts, SEED, keys)
    got = host(keys)
    for i in (0, 63, 64, 69):
        assert np.array_equal(got[i], kr.galois_keys(o, 0, T_BGV, s, SEED, [elts[i]])[0])
    ctx.close()


@pytest.mark.parametrize("logn,L,basis,t,n", [(12, 2, None, T_BGV, 700), (12, 6, "gen_mixed", 0, 5), (13, 4, None, T_BGV, 5),
                                              (13, 6, "fast_mixed", 0, 3), (14, 3, None, T_BGV, 3), (14, 6, "gen_mixed", 0, 2)])
def test_encrypt_bit_exact(oracle_mod, logn, L, basis, t, n):
    """BGV t and CKKS t = 0; n = 700 at N = 4096 spans several waves of the grid"""
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, SEED)
    pt = o.fill_uniform(11, n)
    ct = empty(n, 2, L, o.N)
    ctx.encrypt(t, dev(s), SEED, 1000, dev(pt), ct, n)
    got = host(ct)
    idx = range(n) if n < 50 else [0, 1, 263, 264, 527, 528, n - 1]
    for k in idx:
        assert np.array_equal(got[k], kr.encrypt(o, t, s, SEED, 1000 + k, pt[k:k + 1])[0]), k
    ctx.close()


def test_host_forms_equal_device_forms(oracle_mod):
    """encrypt_host over several pipeline chunks keeps item numbers first_index + k; decrypt_host with three components"""
    ctx, o = _setup(oracle_mod, 12, 2)
    n = 1100   # 512 ciphertexts of 128 KiB per chunk
    s = kr.secret(o, SEED)
    pt = o.fill_uniform(12, n)
    ct_h = np.empty((n, 2, 2, o.N), dtype=np.uint64)
    ctx.encrypt_host(T_BGV, s, SEED, 5, pt, ct_h)
    ct_d = empty(n, 2, 2, o.N)
    ctx.encrypt(T_BGV, dev(s), SEED, 5, dev(pt), ct_d, n)
    assert np.array_equal(ct_h, host(ct_d))
    c3 = o.fill_uniform(13, 3 * n).reshape(n, 3, 2, o.N)
    pt_h = np.empty((n, 2, o.N), dtype=np.uint64)
    ctx.decrypt_host(s, c3, 3, pt_h)
    pt_d = empty(n, 2, o.N)
    ctx.decrypt(dev(s), dev(c3), 3, pt_d, n)
    assert np.array_equal(pt_h, host(pt_d))
    ctx.close()


@pytest.mark.parametrize("logn,L,basis", [(12, 3, None), (13, 6, "gen_mixed"), (14, 2, None)])
def test_decrypt_matches_the_oracle_phase(oracle_mod, logn, L, basis):
    ctx, o = _setup(oracle_mod, logn, L, basis)
    s = kr.secret(o, SEED)
    for n_comp in (2, 3):
        ct = o.fill_uniform(20 + n_comp, 3 * n_comp).reshape(3, n_comp, L, o.N)
        pt = empty(3, L, o.N)
        ctx.decrypt(dev(s), dev(ct), n_comp, pt, 3)
        got = host(pt)
        assert np.array_equal(got, kr.decrypt(o, s, ct))
        for k in range(3):
            assert np.array_equal(o.ntt_inv(got[k]), o.phase(s, ct[k]))
    ctx.close()


def _slots(rng, n, t, count):
    return rng.integers(0, t, (count, 2, n // 2), dtype=np.int64)


def test_bgv_round_trip_per_limb_and_grouped_keys(oracle_mod):
    """slots -> encode -> encrypt -> ct x ct (device and oracle) -> decrypt -> decode is the slot-wise product mod t; the same
    through ct_mul_relin_grouped (K = 2) and rotate_hoisted_grouped, all keys generated on the device"""
    import deeppowers_b200 as dp
    logn, L, K = 12, 6, 2
    ctx, o = _setup(oracle_mod, logn, L)
    n = o.N
    oq = oracle_mod.Oracle(logn, L - K, o.moduli[:L - K])
    cq = dp.Context(logn, L - K, oq.moduli)
    seed = ctx.random_seed()
    sk = empty(L, n)
    ctx.generate_secret(seed, sk)
    rng = np.random.default_rng(5)
    z = _slots(rng, n, T_BGV, 2)
    want = z[0] * z[1] % T_BGV
    # per-limb digits on the full context
    pt = empty(2, L, n)
    ctx.bgv_encode(dev(z), pt, 2, T_BGV)
    ct = empty(2, 2, L, n)
    ctx.encrypt(T_BGV, sk, seed, 0, pt, ct, 2)
    evk = empty(L, 2, L, n)
    ctx.generate_relin_key(0, T_BGV, sk, seed, evk)
    prod = empty(1, 2, L, n)
    ctx.ct_mul_relin(ct[0:1], ct[1:2], evk, prod, 1)
    oprod = o.ct_mul_relin(host(ct[0:1]), host(ct[1:2]), host(evk))
    assert np.array_equal(host(prod), oprod)
    dec, out = empty(1, L, n), empty(1, 2, n // 2)
    ctx.decrypt(sk, prod, 2, dec, 1)
    ctx.bgv_decode(dec, out, 1, T_BGV)
    assert np.array_equal(host(out)[0], want.astype(np.uint64))
    # grouped keys: ciphertexts under the first L - K moduli, encrypted and decrypted with the context over them
    ptq, ctq = empty(2, L - K, n), empty(2, 2, L - K, n)
    cq.bgv_encode(dev(z), ptq, 2, T_BGV)
    skq = sk[:L - K].contiguous()
    cq.encrypt(T_BGV, skq, seed, 2, ptq, ctq, 2)
    nd = ctx.key_digits(K)
    gevk = empty(nd, 2, L, n)
    ctx.generate_relin_key(K, T_BGV, sk, seed, gevk)
    gprod = empty(1, 2, L - K, n)
    ctx.ct_mul_relin_grouped(K, ctq[0:1], ctq[1:2], gevk, gprod, 1, T_BGV)
    assert np.array_equal(host(gprod), o.ct_mul_relin_grouped(K, host(ctq[0:1]), host(ctq[1:2]), host(gevk), T_BGV))
    decq, outq = empty(1, L - K, n), empty(1, 2, n // 2)
    cq.decrypt(skq, gprod, 2, decq, 1)
    cq.bgv_decode(decq, outq, 1, T_BGV)
    assert np.array_equal(host(outq)[0], want.astype(np.uint64))
    # hoisted rotations with grouped Galois keys: rows rolled left by k, 2N - 1 swaps them
    elts = [ctx.galois_elt(1), ctx.galois_elt(5), 2 * n - 1]
    gks = empty(len(elts), nd, 2, L, n)
    ctx.generate_galois_keys(K, T_BGV, sk, elts, seed, gks)
    rot = empty(len(elts), 1, 2, L - K, n)
    ctx.rotate_hoisted_grouped(K, ctq[0:1], elts, [gks[i] for i in range(len(elts))], rot, 1, T_BGV)
    for r, rolled in enumerate([np.roll(z[0], -1, axis=1), np.roll(z[0], -5, axis=1), z[0][::-1]]):
        cq.decrypt(skq, rot[r].contiguous(), 2, decq, 1)
        cq.bgv_decode(decq, outq, 1, T_BGV)
        assert np.array_equal(host(outq)[0], rolled.astype(np.uint64)), r
    ctx.close()
    cq.close()


def test_ckks_round_trip_grouped(oracle_mod):
    """CKKS (t = 0): encode -> encrypt -> ct_mul_relin_grouped -> mod_switch_down -> decrypt -> decode is z1 z2 within 2^-20 per
    slot.  The scale is 2^50, so that the product keeps 2^40 after the division by a 60-bit modulus (at 2^40 it would keep 2^20, and
    the rescaling noise alone is about 10^-2 per slot)"""
    import deeppowers_b200 as dp
    logn, L, K = 13, 6, 2
    ctx, o = _setup(oracle_mod, logn, L)
    n, Lq = o.N, L - K
    cq = dp.Context(logn, Lq, o.moduli[:Lq])
    cl = dp.Context(logn, Lq - 1, o.moduli[:Lq - 1])
    sk = empty(L, n)
    ctx.generate_secret(SEED, sk)
    rng = np.random.default_rng(9)
    z = (rng.uniform(-1, 1, (2, n // 2)) + 1j * rng.uniform(-1, 1, (2, n // 2))).astype(np.complex128)
    scale = 2.0**50
    pt, ct = empty(2, Lq, n), empty(2, 2, Lq, n)
    cq.ckks_encode(torch.from_numpy(z).cuda(), pt, 2, scale)
    skq = sk[:Lq].contiguous()
    cq.encrypt(0, skq, SEED, 0, pt, ct, 2)
    evk = empty(ctx.key_digits(K), 2, L, n)
    ctx.generate_relin_key(K, 0, sk, SEED, evk)
    prod, low = empty(1, 2, Lq, n), empty(2, Lq - 1, n)
    ctx.ct_mul_relin_grouped(K, ct[0:1], ct[1:2], evk, prod, 1, 0)
    cq.mod_switch_down(prod, low, 2, 0)
    dec = empty(1, Lq - 1, n)
    cl.decrypt(sk[:Lq - 1].contiguous(), low.reshape(1, 2, Lq - 1, n), 2, dec, 1)
    out = torch.empty((1, n // 2), dtype=torch.complex128, device="cuda")
    cl.ckks_decode(dec, out, 1, scale * scale / o.moduli[Lq - 1])
    err = np.abs(out.cpu().numpy()[0] - z[0] * z[1]).max()
    assert err < 2.0**-20, err
    for c in (ctx, cq, cl):
        c.close()


def test_argument_checks(oracle_mod):
    import deeppowers_b200 as dp
    ctx, o = _setup(oracle_mod, 12, 4)
    sk = empty(4, o.N)
    ctx.generate_secret(SEED, sk)
    key = empty(4, 2, 4, o.N)
    lib, h = ctx._l, ctx._h
    assert lib.dpfhe_secret_keygen(h, None, sk.data_ptr(), None) == -1
    assert lib.dpfhe_relin_keygen(h, 0, T_BGV, sk.data_ptr(), None, key.data_ptr(), None) == -1
    for K in (3, 5):   # 2K > L, K > 4
        with pytest.raises(dp.DpfheError):
            ctx.generate_relin_key(K, T_BGV, sk, SEED, key)
    for g in (2, 4, 2 * o.N + 1, 0):   # even or out of range
        with pytest.raises(dp.DpfheError):
            ctx.generate_galois_keys(0, T_BGV, sk, [g], SEED, key)
    ct, pt = empty(1, 2, 4, o.N), empty(1, 4, o.N)
    for n_comp in (1, 4):
        with pytest.raises(dp.DpfheError):
            ctx.decrypt(sk, ct, n_comp, pt, 1)
    with pytest.raises(ValueError):
        ctx.encrypt(T_BGV, sk, b"short", 0, pt, ct, 1)
    assert lib.dpfhe_random_seed(None) == -1
    assert ctx.random_seed() != ctx.random_seed()
    ctx.close()


def test_cpp_round_trip_example(tmp_path):
    """examples/encrypted_roundtrip.cpp links libdpfhe.so alone and recovers every slot product"""
    import os
    import subprocess
    import deeppowers_b200
    deeppowers_b200.load_library()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir, exe = os.path.join(root, "deeppowers_b200"), str(tmp_path / "encrypted_roundtrip")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "examples", "encrypted_roundtrip.cpp"), "-L", lib_dir, "-ldpfhe", "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "8192 slot products, 0 wrong" in r.stdout


def test_config4_layer_with_device_keys(oracle_mod):
    """config 4's 768 x 768 layer (N = 8192, 4 ciphertext limbs + 2 special primes) with every key made on the device: the secret, and
    the 31 baby-step and the giant-step Galois keys from ONE dpfhe_galois_keygen call, whose [n_elts][dnum][2][L][N] output goes into
    LinearLayer.grouped as it is; x encrypted and the result decrypted and decoded on the device: W x mod t"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY, DIM, t = 13, 4, 2, 2, 32, 768, 167772161
    L = Lq + K
    ctx, o = _setup(oracle_mod, log_n, L)
    N = o.N
    ctx_q = dp.Context(log_n, Lq, o.moduli[:Lq])
    seed = ctx.random_seed()
    sk = empty(L, N)
    ctx.generate_secret(seed, sk)
    elts = [ctx.galois_elt(b) for b in range(1, BABY + 1)]
    keys = empty(BABY, ctx.key_digits(K), 2, L, N)
    ctx.generate_galois_keys(K, t, sk, elts, seed, keys)
    kh = host(keys)
    rng = np.random.default_rng(0xD3390047)
    W = rng.integers(-127, 128, (DIM, DIM))
    X = rng.integers(-127, 128, (B, DIM))
    xs = np.zeros((B, 2, N // 2), dtype=np.int64)
    xs[:, 0, :DIM] = X
    xs[:, 0, DIM:2 * DIM] = X
    ds = np.zeros((DIM, 2, N // 2), dtype=np.int64)
    ar = np.arange(DIM)
    for d in range(DIM):
        ds[d, 0, :DIM] = W[ar, (ar + d) % DIM]
        ds[d] = np.roll(ds[d], (d // BABY) * BABY, axis=1)   # diagonal g*baby + b pre-rotated by -g*baby
    diags, xpt = empty(DIM, Lq, N), empty(B, Lq, N)
    ctx_q.bgv_encode(dev(ds), diags, DIM, t)
    ctx_q.bgv_encode(dev(xs), xpt, B, t)
    skq = sk[:Lq].contiguous()
    ct = empty(B, 2, Lq, N)
    ctx_q.encrypt(t, skq, seed, 0, xpt, ct, B)
    layer = dp.LinearLayer.grouped(ctx, K, host(diags), BABY, np.ascontiguousarray(kh[:BABY - 1]), np.ascontiguousarray(kh[BABY - 1]), t)
    out = empty(B, 2, Lq, N)
    layer.apply(ct, out, B)
    ph, y = empty(B, Lq, N), empty(B, 2, N // 2)
    ctx_q.decrypt(skq, out, 2, ph, B)
    ctx_q.bgv_decode(ph, y, B, t)
    got = host(y)[:, 0, :DIM]
    for b in range(B):
        assert np.array_equal(got[b], (W @ X[b]) % t)
    layer.close()
    ctx_q.close()
    ctx.close()


def test_outputs_overlapping_the_secret_are_rejected(oracle_mod):
    """every CTA reads whole secret rows while others write: an output over the secret would corrupt it silently"""
    import deeppowers_b200 as dp
    ctx, o = _setup(oracle_mod, 12, 2)
    P = 2 * o.N
    buf = empty(2 * 2 * P + P)                    # key [2][2][L][N] followed by nothing: the secret placed inside it
    sk = buf[P:2 * P]
    ctx.generate_secret(SEED, sk)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.generate_relin_key(0, T_BGV, sk, SEED, buf[:4 * P])
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.generate_galois_keys(0, T_BGV, sk, [3], SEED, buf[:4 * P])
    pt = empty(1, 2, o.N)
    with pytest.raises(dp.DpfheError, match="overlap"):
        ctx.encrypt(T_BGV, sk, SEED, 0, pt, buf[:2 * P], 1)
    ctx.close()
