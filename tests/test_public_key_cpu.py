"""Public keys and public-key encryption of DESIGN.md section 2.14, restated (tests/public_key_ref.py) and checked on the CPU: the extended
nonce table, the public key as an encryption of zero, the restriction to a prefix of the basis, decryption to BGV and CKKS slots, the
oracle's key switching and modulus switching on publicly encrypted ciphertexts, and the phase noise that section 2.14 records."""
import numpy as np
import pytest

import bgv_ref
import ckks_ref
import keys_ref as kr
import public_key_ref as pkr

OWNER = bytes(range(100, 132))        # the key owner's seed (secret, public key, switch keys)
ENCRYPTOR = bytes(range(200, 232))    # a data owner's seed (public-key encryption)
T_BGV = 65537
# the bound section 2.14 gives for the largest centred phase noise |e u + e0 + e1 s| (in units of t): each coefficient has standard
# deviation sqrt(14 N + 10.5) (e u and e1 s: N products of variance 10.5 * 2/3 each), about 240 / 340 / 480 at N = 4096 / 8192 /
# 16384; the bound is 8.5, 7.5 and 8.5 of those.  Measured: 1098 at N = 4096 and 1354 at N = 8192 (two ciphertexts, below)
NOISE_BOUND = {12: 2048, 13: 2560, 14: 4096}


def phase_noise(o, s, ct, pt, t):
    """the centred noise (phase - pt) / t in limb 0 for every ciphertext (t = 0: unscaled) as int64 [n][N]"""
    q = np.array(o.moduli, dtype=np.uint64)[:, None]
    d = o.ntt_inv((kr.decrypt(o, s, ct) + (q - pt)) % q)[:, 0].astype(np.int64)
    q0 = int(o.moduli[0])
    noise = np.where(d > q0 // 2, d - q0, d)
    if t:
        assert np.all(noise % t == 0)
        noise //= t
    return noise


def _table_rows(L, seed_id):
    """(seed, n0, item) of every row of the extended nonce table under one seed: secret, switch keys for K = 0 .. 4 (relinearisation
    and several Galois elements), a batch of symmetric encryptions, the public key and a batch of public-key encryptions"""
    rows = [(seed_id, kr.nonce0(kr.SECRET), 0)]
    N = 4096
    for K in range(5):
        if 2 * K > L:
            continue
        nd = (L - K + K - 1) // K if K else L
        for g in (0, 3, 5, 25, 2 * N - 1, pow(5, N // 4, 2 * N)):
            rows += [(seed_id, kr.nonce0(kr.KEY_A, K, j, l), g) for j in range(nd) for l in range(L)]
            rows += [(seed_id, kr.nonce0(kr.KEY_E, K, j), g) for j in range(nd)]
    for k in range(100):
        rows += [(seed_id, kr.nonce0(kr.ENC_A, 0, 0, l), k) for l in range(L)] + [(seed_id, kr.nonce0(kr.ENC_E), k)]
    rows += [(seed_id, kr.nonce0(pkr.PK_A, 0, 0, l), 0) for l in range(L)] + [(seed_id, kr.nonce0(pkr.PK_E), 0)]
    for k in list(range(100)) + [1 << 32, (1 << 32) + 1]:
        rows += [(seed_id, kr.nonce0(d), k) for d in (pkr.PENC_U, pkr.PENC_E0, pkr.PENC_E1)]
    return rows


def test_no_two_rows_of_the_extended_table_share_a_stream():
    """within one seed every row has its own (n0, item); and since the domains differ, that holds even when the key owner and the
    encryptor use the same seed"""
    L = 16
    rows = _table_rows(L, 0)
    assert len(rows) == len(set(rows))
    streams = {(n0, item) for _, n0, item in rows}
    assert len(streams) == len(rows)
    both = _table_rows(L, 0) + _table_rows(L, 1)
    assert len(both) == len(set(both))


@pytest.fixture(scope="module")
def o6(oracle_mod):
    return oracle_mod.Oracle(12, 6)


@pytest.mark.parametrize("t", [T_BGV, 0])
def test_public_key_is_the_encryption_of_zero_under_domains_6_and_7(o6, monkeypatch, t):
    s = kr.secret(o6, OWNER)
    pk = pkr.public_keygen(o6, t, s, OWNER)
    monkeypatch.setattr(kr, "ENC_A", pkr.PK_A)
    monkeypatch.setattr(kr, "ENC_E", pkr.PK_E)
    zero = np.zeros((1, o6.L, o6.N), dtype=np.uint64)
    assert np.array_equal(pk, kr.encrypt(o6, t, s, OWNER, 0, zero)[0])


def test_restriction_to_every_prefix(oracle_mod, o6):
    """the first l rows of both components are the public key of the context over q_0 .. q_{l-1} under the first l rows of the
    secret, and encrypt there to the first l rows of the full context's ciphertexts"""
    s = kr.secret(o6, OWNER)
    pk = pkr.public_keygen(o6, T_BGV, s, OWNER)
    pt = o6.fill_uniform(5, 2)
    ct = pkr.encrypt_public(o6, T_BGV, pk, ENCRYPTOR, 9, pt)
    for l in range(1, 7):
        ol = oracle_mod.Oracle(12, l, o6.moduli[:l])
        pkl = pkr.public_keygen(ol, T_BGV, s, OWNER)
        assert np.array_equal(pkl, pk[:, :l]), l
        assert np.array_equal(pkr.encrypt_public(ol, T_BGV, pkl, ENCRYPTOR, 9, pt[:, :l]), ct[:, :, :l]), l


def test_item_number_and_seed_select_the_ciphertext(o6):
    s = kr.secret(o6, OWNER)
    pk = pkr.public_keygen(o6, T_BGV, s, OWNER)
    pt = o6.fill_uniform(6, 3)
    batch = pkr.encrypt_public(o6, T_BGV, pk, ENCRYPTOR, (1 << 32) - 1, pt)
    for k in range(3):
        assert np.array_equal(batch[k], pkr.encrypt_public(o6, T_BGV, pk, ENCRYPTOR, (1 << 32) - 1 + k, pt[k:k + 1])[0])
    # the high word of the item number is part of the nonce: (2^32 - 1) + 1 is not item 0
    assert not np.array_equal(batch[1], pkr.encrypt_public(o6, T_BGV, pk, ENCRYPTOR, 0, pt[1:2])[0])
    assert not np.array_equal(batch[0], pkr.encrypt_public(o6, T_BGV, pk, OWNER, (1 << 32) - 1, pt[0:1])[0])


@pytest.mark.parametrize("logn", [12, 13])
def test_bgv_slots_decrypt_exactly_and_the_noise_is_bounded(oracle_mod, logn):
    """t = 65537 at N = 4096 and 8192 (four 60-bit limbs): every slot decodes exactly, and the phase noise e u + e0 + e1 s (printed:
    the figures of section 2.14) stays below NOISE_BOUND"""
    o = oracle_mod.Oracle(logn, 4)
    s = kr.secret(o, OWNER)
    pk = pkr.public_keygen(o, T_BGV, s, OWNER)
    z = np.random.default_rng(logn).integers(0, T_BGV, (2, 2, o.N // 2), dtype=np.int64)
    pt = bgv_ref.encode(o, z, T_BGV)
    ct = pkr.encrypt_public(o, T_BGV, pk, ENCRYPTOR, 0, pt)
    assert np.array_equal(bgv_ref.decode(o, kr.decrypt(o, s, ct), T_BGV), z.astype(np.uint64))
    noise = np.abs(phase_noise(o, s, ct, pt, T_BGV)).max()
    sym = kr.encrypt(o, T_BGV, s, OWNER, 0, pt)
    sym_noise = np.abs(phase_noise(o, s, sym, pt, T_BGV)).max()
    print("N = %d: public-key encryption noise %d t (%.1f bits with t), symmetric %d t" % (o.N, noise, np.log2(noise * T_BGV), sym_noise))
    assert sym_noise <= 21
    assert 21 < noise <= NOISE_BOUND[logn]


def test_ckks_slots_decrypt_within_the_noise_bound(oracle_mod):
    """t = 0: the phase is pt + e u + e0 + e1 s with every coefficient below NOISE_BOUND, so every slot moves by at most
    N * NOISE_BOUND / scale (a slot is the sum of N coefficients times roots of unity, divided by the scale), plus the decoder's
    own rounding: 4096 * 2048 / 2^40 < 2^-17"""
    logn, scale = 12, 2.0**40
    o = oracle_mod.Oracle(logn, 3)
    s = kr.secret(o, OWNER)
    pk = pkr.public_keygen(o, 0, s, OWNER)
    rng = np.random.default_rng(3)
    z = rng.uniform(-1, 1, (2, o.N // 2)) + 1j * rng.uniform(-1, 1, (2, o.N // 2))
    pt = ckks_ref.encode(o, z, scale)
    ct = pkr.encrypt_public(o, 0, pk, ENCRYPTOR, 0, pt)
    assert np.abs(phase_noise(o, s, ct, pt, 0)).max() <= NOISE_BOUND[logn]
    got = ckks_ref.decode(o, kr.decrypt(o, s, ct), scale)
    bound = o.N * NOISE_BOUND[logn] / scale
    err = np.abs(got - z).max()
    assert err < bound + 2.0**-30, (err, bound)


def test_public_ciphertexts_through_the_oracles_key_and_modulus_switching(oracle_mod):
    """BGV slots encrypted under the public key, multiplied with the oracle's ct_mul_relin_grouped (a relinearisation key of the
    same secret, K = 2) and switched down one limb: the slot-wise product mod t"""
    logn, L, K, t = 12, 6, 2, T_BGV
    o = oracle_mod.Oracle(logn, L)
    Lq = L - K
    oq = oracle_mod.Oracle(logn, Lq, o.moduli[:Lq])
    ol = oracle_mod.Oracle(logn, Lq - 1, o.moduli[:Lq - 1])
    s = kr.secret(o, OWNER)
    pk = pkr.public_keygen(oq, t, s, OWNER)
    z = np.random.default_rng(4).integers(0, t, (2, 2, o.N // 2), dtype=np.int64)
    ct = pkr.encrypt_public(oq, t, pk, ENCRYPTOR, 0, bgv_ref.encode(oq, z, t))
    evk = kr.relin_key(o, K, t, s, OWNER)
    prod = o.ct_mul_relin_grouped(K, ct[0:1], ct[1:2], evk, t)
    want = (z[0] * z[1] % t).astype(np.uint64)
    assert np.array_equal(bgv_ref.decode(oq, kr.decrypt(oq, s, prod), t)[0], want)
    low = oq.mod_switch_down(prod.reshape(2, Lq, o.N), t).reshape(1, 2, Lq - 1, o.N)
    # the switch multiplies the message by q_{Lq-1}^-1 mod t
    got = bgv_ref.decode(ol, kr.decrypt(ol, s, low), t)[0].astype(np.int64)
    assert np.array_equal(got * (int(o.moduli[Lq - 1]) % t) % t, want.astype(np.int64))
