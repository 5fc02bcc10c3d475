"""Seeded ciphertexts and switch keys (DESIGN.md section 2.23) on the CPU: the restatement (tests/seeded_ref.py) tied to the pinned one
(tests/keys_ref.py), the public seed against the library, the nonce table, the separation of seeded and unseeded rows, decryption
and key switching through the oracle, and the restriction to every prefix of the moduli."""
import numpy as np
import pytest

import keys_ref as kr
import seeded_ref as sr

SEED = bytes(range(7, 39))
T = 65537


def _pt(o, m):
    """a small signed coefficient vector m as a plaintext in evaluation form [1][L][N]"""
    return kr.small_eval(o, m, 1)[None]


def test_restatement_is_keys_ref_with_the_unseeded_domains(oracle_mod):
    o = oracle_mod.Oracle(12, 4)
    s = kr.secret(o, SEED)
    pt = o.fill_uniform(3, 2)
    assert np.array_equal(sr.encrypt_with(o, T, s, SEED, SEED, kr.ENC_A, kr.ENC_E, 9, pt), kr.encrypt(o, T, s, SEED, 9, pt))
    for K in (0, 2):
        assert np.array_equal(sr.switch_key_with(o, K, T, s, SEED, SEED, kr.KEY_A, kr.KEY_E, o.poly_mul_pointwise(s, s), 0),
                              kr.relin_key(o, K, T, s, SEED))
    g = o.galois_elt(3)
    assert np.array_equal(sr.switch_key_with(o, 1, 0, s, SEED, SEED, kr.KEY_A, kr.KEY_E, np.ascontiguousarray(s[:, o.galois_perm(g)]), g),
                          kr.galois_keys(o, 1, 0, s, SEED, [g])[0])


def test_public_seed_is_the_library_s():
    import deeppowers_b200 as dp
    for seed in (SEED, bytes(32), bytes([255] * 32)):
        a = sr.public_seed(seed)
        assert len(a) == 32 and a != seed
        assert dp.public_seed(seed) == a
    with pytest.raises(ValueError):
        dp.public_seed(bytes(31))


def _n0_words():
    """the nonce words n0 of every row of domains 1 .. 15 for K = 0 .. 4, digits and limbs < 16, by domain"""
    rng = range(16)
    d = {1: {kr.nonce0(1)}, 5: {kr.nonce0(5)}, 11: {kr.nonce0(11)}, 13: {kr.nonce0(13)}}
    for dom in (2, 14):
        d[dom] = {kr.nonce0(dom, K, j, l) for K in range(5) for j in rng for l in rng}
    for dom in (3, 15):
        d[dom] = {kr.nonce0(dom, K, j) for K in range(5) for j in rng}
    for dom in (4, 6, 12):
        d[dom] = {kr.nonce0(dom, 0, 0, l) for l in rng}
    for dom in (7, 8, 9, 10):
        d[dom] = {kr.nonce0(dom)}
    return d


def test_nonce_domains_share_no_word():
    d = _n0_words()
    assert sorted(d) == list(range(1, 16))
    seen = set()
    for dom, words in d.items():
        assert not seen & words, dom
        seen |= words


def test_no_stream_is_shared_under_a_seed_and_its_public_seed():
    """(ChaCha20 key, n0, item) of every row: the key owner's rows of domains 1 .. 11, 13, 15 under its seed, the `a` rows of 12, 14
    under the public seed, items 0 .. 99 and the Galois elements; all distinct, and the two keys differ"""
    a_seed = sr.public_seed(SEED)
    assert a_seed != SEED
    rows = set()
    n = 0
    items = list(range(100)) + [8191, (1 << 32) + 3]
    for dom, words in _n0_words().items():
        key = a_seed if dom in (12, 14) else SEED
        for w in words:
            for it in (items if dom not in (1, 6, 7, 11) else [0]):
                rows.add((key, w, it))
                n += 1
    assert len(rows) == n


def test_seeded_and_unseeded_encryption_share_neither_a_nor_e(oracle_mod):
    o = oracle_mod.Oracle(12, 3)
    a_seed = sr.public_seed(SEED)
    for item in (0, 5, (1 << 32) + 1):
        a_u, a_s = kr._uniform_rows(o, SEED, kr.ENC_A, 0, 0, item), kr._uniform_rows(o, a_seed, sr.SENC_A, 0, 0, item)
        assert not np.any(a_u == a_s)
        e_u, e_s = kr.cbd(SEED, kr.nonce0(kr.ENC_E), item, o.N), kr.cbd(SEED, kr.nonce0(sr.SENC_E), item, o.N)
        assert not np.array_equal(e_u, e_s)
        b_u, b_s = kr._uniform_rows(o, SEED, kr.KEY_A, 2, 1, item), kr._uniform_rows(o, a_seed, sr.SKEY_A, 2, 1, item)
        assert not np.any(b_u == b_s)


def _centred(x, q):
    x = int(x) % q
    return x - q if x > q // 2 else x


@pytest.mark.parametrize("t", [T, 0])
def test_seeded_ciphertexts_decrypt_through_the_oracle(oracle_mod, t):
    """BGV (t = 65537): the oracle decrypts m exactly; both t: the phase minus m is t e with |e| <= 21 on every limb"""
    o = oracle_mod.Oracle(12, 3)
    s = kr.secret(o, SEED)
    rng = np.random.default_rng(4)
    m = rng.integers(-1000, 1000, size=o.N)
    ct = sr.encrypt_seeded(o, t, s, SEED, 7, _pt(o, m))
    assert np.array_equal(ct, sr.expand_ciphertexts(o, sr.public_seed(SEED), 7, ct[:, 0]))
    if t:
        assert np.array_equal(o.decrypt(s, ct[0], t), (m % t).astype(np.uint64))
    ph = o.phase(s, ct[0])
    tt = t or 1
    for l, q in enumerate(o.moduli):
        noise = np.array([_centred(int(ph[l, i]) - int(m[i]), q) for i in range(o.N)], dtype=object)
        assert all(v % tt == 0 for v in noise)
        assert max(abs(v) for v in noise) <= 21 * tt


@pytest.mark.parametrize("K", [0, 2])
def test_expanded_seeded_keys_switch_through_the_oracle(oracle_mod, K):
    """BGV: two seeded ciphertexts multiplied and relinearised by the oracle with the expanded seeded key decrypt to m1 m2 mod t; a
    rotation with an expanded seeded Galois key decrypts to the rotated message"""
    L = 6
    o = oracle_mod.Oracle(12, L)
    oq = oracle_mod.Oracle(12, L - K, o.moduli[:L - K]) if K else o
    s = kr.secret(o, SEED)
    rng = np.random.default_rng(5)
    m = rng.integers(0, T, size=(2, o.N)).astype(np.int64)
    signed = np.where(m > T // 2, m - T, m)
    ct = sr.encrypt_seeded(oq, T, s, SEED, 0, np.concatenate([_pt(oq, x) for x in signed]))
    b = sr.relin_key_seeded(o, K, T, s, SEED)[:, 0]
    evk = sr.expand_switch_keys(o, K, sr.public_seed(SEED), [0], b[None])[0]
    assert np.array_equal(evk, sr.relin_key_seeded(o, K, T, s, SEED))
    prod = o.ct_mul_relin_grouped(K, ct[0:1], ct[1:2], evk, T) if K else o.ct_mul_relin(ct[0:1], ct[1:2], evk)
    full = np.convolve(m[0].astype(object), m[1].astype(object))
    want = full[:o.N].copy()
    want[:o.N - 1] -= full[o.N:]
    assert np.array_equal(oq.decrypt(s[:oq.L], prod[0], T), np.array([int(x) % T for x in want], dtype=np.uint64))
    if K == 0:
        g = o.galois_elt(1)
        gk = sr.expand_switch_keys(o, 0, sr.public_seed(SEED), [g], sr.galois_keys_seeded(o, 0, T, s, SEED, [g])[:, :, 0])[0]
        rot = o.rotate(ct[0:1], g, gk)
        want = np.zeros(o.N, dtype=np.int64)
        for k in range(o.N):
            e = k * g % (2 * o.N)
            want[e % o.N] = (m[0, k] if e < o.N else -m[0, k]) % T
        assert np.array_equal(o.decrypt(s, rot[0], T), want.astype(np.uint64))


def test_restriction_at_every_prefix(oracle_mod):
    """the first l rows of a seeded ciphertext and of its expansion are the level-l seeded ciphertext"""
    L = 5
    o = oracle_mod.Oracle(12, L)
    s = kr.secret(o, SEED)
    pt = o.fill_uniform(8, 2)
    full = sr.encrypt_seeded(o, T, s, SEED, 3, pt)
    a_seed = sr.public_seed(SEED)
    for l in range(1, L + 1):
        ol = oracle_mod.Oracle(12, l, o.moduli[:l])
        assert np.array_equal(sr.encrypt_seeded(ol, T, s, SEED, 3, pt[:, :l]), full[:, :, :l]), l
        assert np.array_equal(sr.expand_ciphertexts(ol, a_seed, 3, full[:, 0, :l]), full[:, :, :l]), l


def test_seeded_wire_kinds_round_trip_and_refuse_forgeries(tmp_path, oracle_mod):
    """wire kinds 7 (seeded ciphertexts) and 8 (seeded switch key): a Python round trip, the C++ reader accepting both, and a forged
    prefix (wrapping item numbers, an even or too large key item), count (0 ciphertexts, more than the file holds) or K (5, 2K > L)
    refused by both readers; kind 9 stays unknown"""
    import os
    import subprocess
    from deeppowers_b200 import wire
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    o = oracle_mod.Oracle(12, 4)
    a_seed = sr.public_seed(SEED)
    c0 = o.fill_uniform(3, 2)
    good_ct, good_key = str(tmp_path / "ct.dpfhe"), str(tmp_path / "key.dpfhe")
    wire.write(good_ct, 12, 4, wire.SEEDED_CIPHERTEXTS, 2, o.moduli, np.concatenate([wire.seeded_prefix(a_seed, 7), c0.reshape(-1)]))
    b = o.fill_uniform(4, 1)[0]     # K = 2 on 4 limbs: one digit of [4][N]
    wire.write(good_key, 12, 4, wire.SEEDED_SWITCH_KEY, 2, o.moduli, np.concatenate([wire.seeded_prefix(a_seed, 2 * o.N - 1), b.reshape(-1)]))
    hdr, data = wire.read(good_ct)
    seed, first, rows = wire.split_seeded(data)
    assert hdr["kind"] == 7 and hdr["count"] == 2 and seed == a_seed and first == 7 and np.array_equal(rows.reshape(c0.shape), c0)
    hdr, data = wire.read(good_key)
    seed, item, rows = wire.split_seeded(data)
    assert hdr["kind"] == 8 and seed == a_seed and item == 2 * o.N - 1 and np.array_equal(rows.reshape(b.shape), b)

    def forged(src, name, count=None, kind=None, limbs=None, item=None):
        raw = bytearray(open(src, "rb").read())
        hdr = list(wire._HDR.unpack(bytes(raw[:160])))
        if count is not None:
            hdr[5] = count
        if kind is not None:
            hdr[3] = kind
        if limbs is not None:
            hdr[2] = limbs
        raw[:160] = wire._HDR.pack(*hdr)
        if item is not None:
            raw[160 + 32:160 + 40] = int(item).to_bytes(8, "little")
        path = str(tmp_path / name)
        open(path, "wb").write(bytes(raw))
        return path

    bad = [forged(good_ct, "wrap.dpfhe", item=(1 << 64) - 1), forged(good_ct, "zero.dpfhe", count=0), forged(good_ct, "more.dpfhe", count=3),
           forged(good_ct, "kind9.dpfhe", kind=9), forged(good_key, "even.dpfhe", item=4), forged(good_key, "big.dpfhe", item=2 * o.N + 1),
           forged(good_key, "k5.dpfhe", count=5), forged(good_key, "k3.dpfhe", count=3), forged(good_key, "k2l3.dpfhe", limbs=3)]
    for path in bad:
        with pytest.raises(ValueError):
            wire.read(path)
    src = tmp_path / "rd.cpp"
    src.write_text("""
#include "dpfhe_wire.hpp"
#include <iostream>
int main(int argc, char **argv) {
    using namespace deeppowers::api::fhe;
    int refused = 0;
    for (int i = 1; i < argc; ++i) {
        std::vector<std::uint64_t> payload;
        try { WireHeader h = read_wire_file(argv[i], payload); std::cout << "accepted " << argv[i] << " kind " << h.kind << " item " << payload[4] << "\\n"; }
        catch (const std::runtime_error &e) { ++refused; }
    }
    std::cout << "refused " << refused << "\\n";
    return 0;
}
""")
    exe = str(tmp_path / "rd")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.run([exe, good_ct, good_key] + bad, capture_output=True, text=True, check=True).stdout
    assert ("accepted %s kind 7 item 7" % good_ct) in out and ("accepted %s kind 8 item %d" % (good_key, 2 * o.N - 1)) in out, out
    assert "refused %d" % len(bad) in out, out
