"""The restatement of DESIGN.md section 2.14 (tests/keys_ref.c, tests/keys_ref.py) on the CPU: ChaCha20 against an independent
implementation, the samplers against Python integers, coarse statistics, stream separation, and the scheme's semantics through
the oracle's key switching."""
import json
import os
import random
import struct

import numpy as np
import pytest

import keys_ref as kr
from bases import LARGEST_GENERIC, SMALLEST_FAST_37, SMALLEST_GENERIC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = bytes(range(100, 132))
# the largest default modulus (2^60 - 96 * 2^32 + 1), the smallest generic and k 2^32 + 1 moduli, the largest generic one
MODULI = [(1 << 60) - 96 * (1 << 32) + 1, SMALLEST_GENERIC, SMALLEST_FAST_37, LARGEST_GENERIC]


def test_chacha20_matches_the_committed_known_answers():
    with open(os.path.join(ROOT, "tests", "golden", "chacha20_kat.json")) as f:
        cases = json.load(f)
    assert cases[0]["counter"] == 1 and cases[0]["key"] == bytes(range(32)).hex()
    # RFC 8439 §2.3.2: the serialized block begins 10 f1 e7 e4 d1 3b 59 15
    assert struct.pack("<2I", *cases[0]["block"][:2]).hex() == "10f1e7e4d13b5915"
    for c in cases:
        got = kr.chacha20_block(bytes.fromhex(c["key"]), c["counter"], c["nonce"])
        assert got.tolist() == c["block"], c


def test_chacha20_against_openssl():
    pytest.importorskip("cryptography")
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    rng = random.Random(7)
    for _ in range(64):
        key = bytes(rng.getrandbits(8) for _ in range(32))
        ctr, nonce = rng.getrandbits(32), [rng.getrandbits(32) for _ in range(3)]
        enc = Cipher(algorithms.ChaCha20(key, struct.pack("<I3I", ctr, *nonce)), mode=None).encryptor()
        assert kr.chacha20_block(key, ctr, nonce).tolist() == list(struct.unpack("<16I", enc.update(bytes(64))))


def _blocks(seed, n0, item, n_blocks):
    return [kr.chacha20_block(seed, b, [n0, item & 0xFFFFFFFF, item >> 32]).tolist() for b in range(n_blocks)]


def test_samplers_against_python_integers():
    n0, item = kr.nonce0(kr.KEY_E, 2, 3, 0), (1 << 40) + 5
    words = [w for blk in _blocks(SEED, n0, item, 64) for w in blk]
    assert kr.ternary(SEED, n0, item, 1024).tolist() == [(3 * w >> 32) - 1 for w in words]
    cbd = []
    for i in range(512):
        r = words[2 * i] | words[2 * i + 1] << 32
        cbd.append(bin(r & 0x1FFFFF).count("1") - bin((r >> 21) & 0x1FFFFF).count("1"))
    assert kr.cbd(SEED, n0, item, 512).tolist() == cbd
    for q in MODULI:
        want = [(words[4 * k] | words[4 * k + 1] << 32 | words[4 * k + 2] << 64 | words[4 * k + 3] << 96) % q for k in range(256)]
        assert kr.uniform(SEED, n0, item, q, 256).tolist() == want


def test_sampler_word_boundaries():
    """ternary at the word values where floor(3w / 2^32) steps, CBD at all-ones halves, the uniform reduction at hi / lo extremes"""
    third, two_thirds = -(-(1 << 32) // 3), -(-(2 << 32) // 3)
    for w, s in ((0, -1), (third - 1, -1), (third, 0), (two_thirds - 1, 0), (two_thirds, 1), ((1 << 32) - 1, 1)):
        assert (3 * w >> 32) - 1 == s
    for q in MODULI:
        for hi in (0, 1, q - 1, q, (1 << 64) - 1):
            for lo in (0, 1, q - 1, q, (1 << 64) - 1):
                assert kr.reduce128(lo, hi, q) == ((hi << 64) | lo) % q


def test_coarse_statistics():
    n = 1 << 16
    t = kr.ternary(SEED, kr.nonce0(kr.SECRET), 0, n)
    for v in (-1, 0, 1):
        assert abs(np.mean(t == v) - 1 / 3) < 0.01
    e = kr.cbd(SEED, kr.nonce0(kr.ENC_E), 9, n)
    assert abs(e.mean()) < 0.05 and abs(e.var() - 10.5) < 0.3 and np.abs(e).max() <= 21
    for q in MODULI:
        u = kr.uniform(SEED, kr.nonce0(kr.ENC_A, 0, 0, 1), 9, q, n).astype(np.float64) / int(q)
        assert u.max() < 1 and abs(u.mean() - 0.5) < 0.01 and abs(np.mean(u < 0.25) - 0.25) < 0.01


def _rows_of_keys(L, K, item):
    nd = (L - K + K - 1) // K if K else L
    rows = [(kr.nonce0(kr.KEY_A, K, j, l), item) for j in range(nd) for l in range(L)]
    return rows + [(kr.nonce0(kr.KEY_E, K, j), item) for j in range(nd)]


def test_no_two_rows_share_a_stream():
    """every row of relinearisation keys, Galois keys (several elements, the conjugation included) for K = 0 .. 4, the secret and a
    batch of encryptions has its own (nonce, item number)"""
    L, N = 16, 4096
    rows = [(kr.nonce0(kr.SECRET), 0)]
    for K in range(5):
        if 2 * K > L:
            continue
        rows += _rows_of_keys(L, K, 0)
        for g in (3, 5, 25, 2 * N - 1, pow(5, N // 4, 2 * N)):
            rows += _rows_of_keys(L, K, g)
    for k in range(100):
        rows += [(kr.nonce0(kr.ENC_A, 0, 0, l), k) for l in range(L)] + [(kr.nonce0(kr.ENC_E), k)]
    assert len(rows) == len(set(rows))


@pytest.fixture(scope="module")
def o3(oracle_mod):
    return oracle_mod.Oracle(12, 3)


def test_ciphertext_index_is_first_index_plus_k(o3):
    s = kr.secret(o3, SEED)
    pt = o3.fill_uniform(3, 4)
    batch = kr.encrypt(o3, 65537, s, SEED, 10, pt)
    for k in range(4):
        assert np.array_equal(batch[k], kr.encrypt(o3, 65537, s, SEED, 10 + k, pt[k:k + 1])[0])
    assert not np.array_equal(batch[0, 1], batch[1, 1])


def _negacyclic(a, b, t):
    n = len(a)
    full = np.convolve(a.astype(object), b.astype(object))
    r = full[:n].copy()
    r[: n - 1] -= full[n:]
    return np.array([int(x) % t for x in r], dtype=np.uint64)


@pytest.mark.parametrize("K", [0, 1, 2])
def test_restated_keys_relinearise_through_the_oracle(oracle_mod, K):
    """BGV: Enc(m1) x Enc(m2), relinearised by the oracle with a restated key, decrypts to m1 m2 mod t (semantics of the spec)"""
    t, L = 65537, 6
    o = oracle_mod.Oracle(12, L)
    oq = oracle_mod.Oracle(12, L - K, o.moduli[:L - K]) if K else o
    s = kr.secret(o, SEED)
    rng = np.random.default_rng(1)
    m = rng.integers(0, t, size=(2, o.N)).astype(np.int64)
    pt = np.stack([kr.small_eval(oq, np.where(x > t // 2, x - t, x), 1) for x in m])
    ct = kr.encrypt(oq, t, s, SEED, 0, pt)
    assert np.array_equal(oq.decrypt(s[:oq.L], ct[0], t), m[0].astype(np.uint64))
    evk = kr.relin_key(o, K, t, s, SEED)
    if K:
        prod = o.ct_mul_relin_grouped(K, ct[0:1], ct[1:2], evk, t)
    else:
        prod = o.ct_mul_relin(ct[0:1], ct[1:2], evk)
    assert np.array_equal(oq.decrypt(s[:oq.L], prod[0], t), _negacyclic(m[0], m[1], t))
    # the restated decryption is the oracle's phase in evaluation form
    assert np.array_equal(oq.ntt_inv(kr.decrypt(oq, s, prod))[0], oq.phase(s[:oq.L], prod[0]))


def test_restated_galois_key_rotates_through_the_oracle(oracle_mod):
    t, L = 65537, 4
    o = oracle_mod.Oracle(12, L)
    s = kr.secret(o, SEED)
    m = np.random.default_rng(2).integers(0, t, size=o.N).astype(np.int64)
    ct = kr.encrypt(o, t, s, SEED, 3, kr.small_eval(o, np.where(m > t // 2, m - t, m), 1)[None])
    for g in (o.galois_elt(1), 2 * o.N - 1):
        gk = kr.galois_keys(o, 0, t, s, SEED, [g])[0]
        rot = o.rotate(ct, g, gk)
        # sigma_g(m)(X) = m(X^g): coefficient k moves to k g mod 2N, negated past N
        want = np.zeros(o.N, dtype=np.int64)
        for k in range(o.N):
            e = k * g % (2 * o.N)
            want[e % o.N] = (m[k] if e < o.N else -m[k]) % t
        assert np.array_equal(o.decrypt(s, rot[0], t), want.astype(np.uint64))
