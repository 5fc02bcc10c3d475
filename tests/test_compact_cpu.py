"""Compact ciphertexts of DESIGN.md section 2.24 without a GPU: the restatement (tests/compact_ref.py) against its own definition and
the scheme, and wire kind 10 in both readers."""
import os
import subprocess

import numpy as np
import pytest

import compact_ref as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 65537


@pytest.mark.parametrize("t", [0, 3, T])
def test_switch_is_lambda_x_within_its_rounding(oracle_mod, t):
    """BGV: y = lambda x (mod t) before the reduction mod 2^bits and |y - 2^bits x / q0| <= t/2 + 1; CKKS: |y - 2^bits x / q0| <= 1/2"""
    q0 = oracle_mod.Oracle(13, 1).moduli[0]
    rng = np.random.default_rng(t + 1)
    for bits in (2, 7, 31, 32, 33, cr.max_bits(13, q0)):
        if t and t >= 1 << (bits - 1):
            continue
        xs = [0, 1, q0 - 1, q0 // 2, q0 // 2 + 1] + [int(v) for v in rng.integers(0, q0, size=300, dtype=np.uint64)]
        for x in xs:
            y, y_full = cr.switch(x, q0, bits, t)
            assert 0 <= y < 1 << bits and (y_full - y) % (1 << bits) == 0
            # |y_full q0 - 2^bits x| <= bound q0, in integers
            bound2 = (t + 2) if t else 1   # twice the bound: t/2 + 1 or 1/2
            assert 2 * abs(y_full * q0 - (x << bits)) <= bound2 * q0, (bits, x)
            if t:
                assert (y_full - cr.lam(q0, bits, t) * x) % t == 0, (bits, x)


@pytest.mark.parametrize("bits", [2, 7, 31, 32, 33, 47])
def test_pack_and_unpack_round_trip(bits):
    """pack agrees with the bit stream's definition, and unpack inverts it; 64 | N makes a tile of 64 coefficients bits whole words"""
    rng = np.random.default_rng(bits)
    N = 4096
    y = rng.integers(0, 1 << bits, size=(3, N), dtype=np.uint64)
    y[0, :3] = [0, (1 << bits) - 1, 1 << (bits - 1)]
    w = cr.pack(y, bits)
    assert w.shape == (3, N * bits // 64)
    for r in range(3):
        assert np.array_equal(w[r], cr.pack_bigint(y[r], bits))
    assert np.array_equal(cr.unpack(w, bits, N), y)


def _ternary_message(rng, N, t):
    return rng.integers(0, t, size=N, dtype=np.uint64)


@pytest.mark.parametrize("log_n", [12, 13, 14])
def test_bgv_products_decrypt_exactly(oracle_mod, log_n):
    """an oracle-encrypted product at level 3, compacted at bits 40 and at the largest bits: the compact ciphertext decrypts to the
    message of the level-1 ciphertext that the modulus switches give, which is the product times (q_1 q_2)^-1 mod t; the measured
    phase stays within (2^bits / q0) |phase_1| + (N + 1)(t/2 + 1)"""
    L = 3
    o = oracle_mod.Oracle(log_n, L)
    rng = np.random.default_rng(log_n)
    s = o.keygen_secret(11)
    evk = o.keygen_relin(12, T, s)
    m1, m2 = _ternary_message(rng, o.N, T), _ternary_message(rng, o.N, T)
    ct = o.ct_mul_relin(o.encrypt(21, T, s, m1), o.encrypt(22, T, s, m2), evk)
    q0 = o.moduli[0]
    top = o.decrypt(s, ct, T).astype(object)
    x1 = ct.reshape(2, L, o.N)
    for k in range(L, 1, -1):
        x1 = oracle_mod.Oracle(log_n, k, o.moduli[:k]).mod_switch_down(x1, T)
    o1 = oracle_mod.Oracle(log_n, 1, o.moduli[:1])
    want = o1.decrypt(s[:1], x1.reshape(2, 1, o.N), T).astype(object)
    factor = pow(o.moduli[1] * o.moduli[2], -1, T)
    assert all((int(a) - int(b) * factor) % T == 0 for a, b in zip(want, top))
    ph1 = o1.phase(s[:1], x1.reshape(2, 1, o.N))[0]
    ph1_max = max(min(int(v), q0 - int(v)) for v in ph1)
    for bits in (40, cr.max_bits(log_n, q0)):
        cct = cr.compact(oracle_mod, o, L, bits, T, ct.reshape(1, 2, L, o.N))
        phi = cr.phase(o, bits, s, cct)
        bound = (1 << bits) * ph1_max / q0 + (o.N + 1) * (T / 2 + 1)
        print("BGV N=%d bits=%d: |phi| = 2^%.1f, bound 2^%.1f, 2^(bits-1) = 2^%d" % (o.N, bits, np.log2(float(np.abs(phi).max())), np.log2(bound), bits - 1))
        assert np.abs(phi).max() <= bound < 1 << (bits - 1)
        pt = cr.plaintext(o, bits, T, phi)
        got = o1.ntt_inv(pt)[0, 0]
        got = [(int(v) - q0 if int(v) > q0 // 2 else int(v)) % T for v in got]
        assert got == [int(v) for v in want]


@pytest.mark.parametrize("log_n", [12, 13, 14])
def test_ckks_products_decrypt_within_the_bound(oracle_mod, log_n):
    """CKKS: a product of two ciphertexts whose phases carry scaled messages, compacted from level 2 (limb 0 alone): the decrypted
    coefficients are the level-1 phase within (q0 / 2^bits)(N + 1)/2 + 1/2"""
    L = 2
    o = oracle_mod.Oracle(log_n, L)
    rng = np.random.default_rng(log_n + 100)
    s = o.keygen_secret(31)
    evk = o.keygen_relin(32, 1, s)
    cts = []
    for seed in (41, 42):
        m = rng.integers(-(1 << 12), 1 << 12, size=o.N)
        ct = o.encrypt(seed, 1, s, np.zeros(o.N, dtype=np.uint64))
        pt = np.array([[int(v) % q for v in m] for q in o.moduli], dtype=np.uint64)
        ct[0] = o.poly_add(ct[0], o.ntt_fwd(pt))
        cts.append(ct)
    ct = o.ct_mul_relin(cts[0], cts[1], evk)
    q0 = o.moduli[0]
    o1 = oracle_mod.Oracle(log_n, 1, o.moduli[:1])
    ph1 = [int(v) - q0 if int(v) > q0 // 2 else int(v) for v in o1.phase(s[:1], np.ascontiguousarray(ct[:, :1]))[0]]
    assert max(abs(v) for v in ph1) < q0 // 2
    for bits in (30, cr.max_bits(log_n, q0)):
        cct = cr.compact(oracle_mod, o, L, bits, 0, ct.reshape(1, 2, L, o.N))
        pt = cr.decrypt(o, bits, 0, s, cct)
        got = [int(v) - q0 if int(v) > q0 // 2 else int(v) for v in o1.ntt_inv(pt)[0, 0]]
        err = max(abs(a - b) for a, b in zip(got, ph1))
        bound = q0 / (1 << bits) * (o.N + 1) / 2 + 0.5
        print("CKKS N=%d bits=%d: max error %d, bound %.1f" % (o.N, bits, err, bound))
        assert err <= bound


def _forge(tmp_path, src, name, words=None, count=None, limbs=None, form=None, kind=None, q0=None, cut=0):
    from deeppowers_b200 import wire
    raw = bytearray(open(src, "rb").read())
    hdr = list(wire._HDR.unpack(bytes(raw[:160])))
    for i, v in ((5, count), (2, limbs), (4, form), (3, kind), (6, q0)):
        if v is not None:
            hdr[i] = v
    raw[:160] = wire._HDR.pack(*hdr)
    for i, v in (words or {}).items():
        raw[160 + 8 * i:168 + 8 * i] = int(v).to_bytes(8, "little")
    path = str(tmp_path / name)
    open(path, "wb").write(bytes(raw[:len(raw) - cut]))
    return path


def test_compact_wire_kind_round_trips_and_refuses_forgeries(tmp_path, oracle_mod):
    """wire kind 10: a Python round trip, the C++ reader accepting it, and forged prefixes (bits 0, bits too large for q0, bits that
    would wrap the range check's sum in 64 bits, an even t, t not below 2^(bits-1)), headers (two limbs, evaluation form), counts (0, one that wraps the size, more than the file holds) and a
    short payload refused by both readers; kind 9 stays unknown"""
    from deeppowers_b200 import wire
    o = oracle_mod.Oracle(12, 1)
    q0, bits = o.moduli[0], 33
    words = np.random.default_rng(3).integers(0, 1 << 63, size=(2, 2, o.N * bits // 64), dtype=np.uint64)
    good = str(tmp_path / "cct.dpfhe")
    wire.write(good, 12, 1, wire.COMPACT_CIPHERTEXTS, 2, [q0], np.concatenate([wire.compact_prefix(bits, T), words.reshape(-1)]), form=0)
    hdr, data = wire.read(good)
    assert hdr["kind"] == 10 and hdr["count"] == 2 and hdr["form"] == 0 and hdr["moduli"] == [q0]
    assert [int(v) for v in data[:2]] == [bits, T] and np.array_equal(data[2:].reshape(words.shape), words)
    with pytest.raises(ValueError):
        wire.write(str(tmp_path / "w.dpfhe"), 12, 1, wire.COMPACT_CIPHERTEXTS, 2, [q0], np.concatenate([wire.compact_prefix(bits, 4), words.reshape(-1)]), form=0)
    big = cr.max_bits(12, q0) + 1
    bad = [_forge(tmp_path, good, "bits0.dpfhe", words={0: 0}), _forge(tmp_path, good, "bitsbig.dpfhe", words={0: big}),
           _forge(tmp_path, good, "bitshuge.dpfhe", words={0: 1 << 62}),
           _forge(tmp_path, good, "bitswrap.dpfhe", words={0: (1 << 64) - 1}), _forge(tmp_path, good, "bitswrap12.dpfhe", words={0: (1 << 64) - 12}),
           _forge(tmp_path, good, "bits52.dpfhe", words={0: 64 - 12}), _forge(tmp_path, good, "teven.dpfhe", words={1: 65536}),
           _forge(tmp_path, good, "tbig.dpfhe", words={1: (1 << (bits - 1)) + 1}), _forge(tmp_path, good, "t1.dpfhe", words={1: 1}),
           _forge(tmp_path, good, "limbs.dpfhe", limbs=2), _forge(tmp_path, good, "form.dpfhe", form=1),
           _forge(tmp_path, good, "zero.dpfhe", count=0), _forge(tmp_path, good, "wrap.dpfhe", count=(1 << 64) - 1),
           _forge(tmp_path, good, "wrap2.dpfhe", count=1 << 58), _forge(tmp_path, good, "more.dpfhe", count=3),
           _forge(tmp_path, good, "short.dpfhe", cut=8), _forge(tmp_path, good, "prefix.dpfhe", cut=(len(open(good, "rb").read()) - 168)),
           _forge(tmp_path, good, "kind9.dpfhe", kind=9), _forge(tmp_path, good, "q0.dpfhe", q0=1 << 44)]
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
        try {
            WireHeader h = read_wire_file(argv[i], payload);
            std::cout << "accepted " << argv[i] << " kind " << h.kind << " bits " << payload[0] << " t " << payload[1] << " words " << payload.size() << "\\n";
            write_wire_file(std::string(argv[i]) + ".copy", h, payload.data());
        } catch (const std::runtime_error &e) { ++refused; }
    }
    std::cout << "refused " << refused << "\\n";
    return 0;
}
""")
    exe = str(tmp_path / "rd")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.run([exe, good] + bad, capture_output=True, text=True, check=True).stdout
    assert ("accepted %s kind 10 bits %d t %d words %d" % (good, bits, T, 2 + words.size)) in out, out
    assert "refused %d" % len(bad) in out, out
    assert open(good + ".copy", "rb").read() == open(good, "rb").read()
