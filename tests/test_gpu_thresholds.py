"""The kernels' data-dependent branches at their exact thresholds on the device (tests/thresholds.py crafts the inputs), bit for bit
against the oracle, which tests/test_thresholds_cpu.py pins to exact integers on the same kind of input: the centred lifts of the
division by one modulus and by P, a single zero coefficient of a hoisted digit (the fallback, also with a linear layer's prepared
key companions), the sign and the digits of Q - X in CKKS decoding, ties and the sign of zero in CKKS encoding.  Every entry point
and its host-buffer form, at N = 4096, 8192 and 16384, on the default basis and a generic one."""
import numpy as np
import pytest

import ckks_ref
import thresholds as th
from test_gpu_parity import ctxs, dev, dp, host  # noqa: E402,F401  (ctxs and dp are fixtures)
from test_thresholds_cpu import encode_groups, expected_plaintexts, hoist_galois, hoist_zero_cases

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SHAPES = [("default", 12), ("default", 13), ("default", 14), ("gen_mixed", 12), ("gen_mixed", 14)]
T = [0, 65537]


@pytest.fixture
def on(ctxs, oracle_mod):
    def get(basis, log_n, L):
        c, o = ctxs(log_n, L, th.basis_moduli(oracle_mod, basis, L))
        assert c.moduli == o.moduli
        return c, o
    return get


def empty(*shape):
    return torch.full(shape, -1, dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("basis,log_n", SHAPES)
def test_mod_switch_down(on, basis, log_n):
    L, n = (3 if basis == "default" else 6), 3
    c, o = on(basis, log_n, L)
    for t in T:
        x = th.mod_switch_input(o, n, t, 0x7E61)
        want = o.mod_switch_down(x, t)
        out = empty(n, L - 1, o.N)
        c.mod_switch_down(dev(x), out, n, t)
        assert np.array_equal(host(out).reshape(want.shape), want), t
        out_h = np.zeros_like(want)
        c.mod_switch_down_host(x, out_h, t)
        assert np.array_equal(out_h, want), t


@pytest.mark.parametrize("basis,log_n", SHAPES)
def test_hybrid_family(on, basis, log_n):
    """tau' at the threshold through the key (tests/thresholds.py hybrid_key): key switch, ct x ct, rotations by g = 1 and a real g"""
    L, batch = (4 if basis == "default" else 6), 2
    c, o = on(basis, log_n, L)
    key = th.hybrid_key(o, 0x7E62)
    for t in T:
        d = th.hybrid_digits(o, batch, t, 0x7E63)
        out = empty(batch, 2, L - 1, o.N)
        c.keyswitch_hybrid(dev(d), dev(key), out, batch, t)
        got = host(out).reshape(batch, 2, L - 1, o.N)
        for k in range(batch):
            assert np.array_equal(got[k], np.stack(o.keyswitch_hybrid(d[k], key, t))), (t, k)
        a, b = th.mul_inputs(o, d, 0x7E64)
        want = o.ct_mul_relin_hybrid(a, b, key, t)
        c.ct_mul_relin_hybrid(dev(a), dev(b), dev(key), out, batch, t)
        assert np.array_equal(host(out).reshape(want.shape), want), t
        out_h = np.zeros_like(want)
        c.ct_mul_relin_hybrid_host(a, b, key, out_h, t)
        assert np.array_equal(out_h, want), t
        for g in (1, o.galois_elt(3)):
            ct = th.rotate_inputs(o, d, g, 0x7E65)
            want = o.rotate_hybrid(ct, g, key, t)
            c.rotate_hybrid(dev(ct), g, dev(key), out, batch, t)
            assert np.array_equal(host(out).reshape(want.shape), want), (t, g)
            out_h = np.zeros_like(want)
            c.rotate_hybrid_host(ct, g, key, out_h, t)
            assert np.array_equal(out_h, want), (t, g)


@pytest.mark.parametrize("basis,log_n", SHAPES)
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_mod_down_special(on, basis, log_n, K):
    """K = 4 is the path with the per-term reduction of the lift; inputs where every y_k is above p_k/2 give its largest sum"""
    L, n = th.special_limbs(K), 2
    c, o = on(basis, log_n, L)
    for t in T:
        x = th.mod_down_input(o, K, n, t, 0x7E66 + K)
        want = o.mod_down_special(K, x, t)
        out = empty(n, L - K, o.N)
        c.mod_down_special(K, dev(x), out, n, t)
        assert np.array_equal(host(out).reshape(want.shape), want), t
        out_h = np.zeros_like(want)
        c.mod_down_special_host(K, x, out_h, t)
        assert np.array_equal(out_h, want), t


@pytest.mark.parametrize("basis,log_n", SHAPES)
@pytest.mark.parametrize("K", [1, 2, 4])
def test_grouped_family(on, basis, log_n, K):
    """y_k at the threshold through the key (tests/thresholds.py grouped_key): key switch, ct x ct, rotations, hoisted rotations"""
    L, batch, t = th.special_limbs(K), 2, 65537
    c, o = on(basis, log_n, L)
    Lq = L - K
    key = th.grouped_key(o, K, 0x7E67)
    d = th.grouped_digits_input(o, K, batch, t, 0x7E68 + K)
    out = empty(batch, 2, Lq, o.N)
    c.keyswitch_grouped(K, dev(d), dev(key), out, batch, t)
    got = host(out).reshape(batch, 2, Lq, o.N)
    for k in range(batch):
        assert np.array_equal(got[k], np.stack(o.keyswitch_grouped(K, d[k], key, t))), k
    a, b = th.mul_inputs(o, d, 0x7E69)
    want = o.ct_mul_relin_grouped(K, a, b, key, t)
    c.ct_mul_relin_grouped(K, dev(a), dev(b), dev(key), out, batch, t)
    assert np.array_equal(host(out).reshape(want.shape), want)
    out_h = np.zeros_like(want)
    c.ct_mul_relin_grouped_host(K, a, b, key, out_h, t)
    assert np.array_equal(out_h, want)
    for g in (1, o.galois_elt(-2)):
        ct = th.rotate_inputs(o, d, g, 0x7E6A)
        want = o.rotate_grouped(K, ct, g, key, t)
        c.rotate_grouped(K, dev(ct), g, dev(key), out, batch, t)
        assert np.array_equal(host(out).reshape(want.shape), want), g
        out_h = np.zeros_like(want)
        c.rotate_grouped_host(K, ct, g, key, out_h, t)
        assert np.array_equal(out_h, want), g
    ct = th.rotate_inputs(o, d, 1, 0x7E6A)                  # the hoisted mod-up reads the unpermuted c1 = d
    galois = [1, o.galois_elt(3), 2 * o.N - 1]
    want = o.rotate_hoisted_grouped(K, ct, galois, np.stack([key] * len(galois)), t)
    hout = empty(len(galois), batch, 2, Lq, o.N)
    c.rotate_hoisted_grouped(K, dev(ct), galois, [dev(key)] * len(galois), hout, batch, t)
    assert np.array_equal(host(hout).reshape(want.shape), want)


# ---------------------------------------------------------------- hoisted rotations: one zero coefficient in a digit
def _groups(L):
    """ciphertexts per round of the persistent kernels: at most four CTAs per SM, L CTAs per ciphertext"""
    return 4 * torch.cuda.get_device_properties(0).multi_processor_count // L


def _flagged(batch, G, n):
    """n ciphertext indices: the first, the last, two in the same round (G + 1, G + 2), the rest spread over the batch"""
    idx = [0, batch - 1, G + 1, G + 2]
    idx += [k for k in dict.fromkeys(np.linspace(3, batch - 2, n).astype(int).tolist()) if k not in idx][:n - len(idx)]
    assert len(set(idx)) == n
    return idx


@pytest.mark.parametrize("basis,log_n", SHAPES)
def test_rotate_hoisted_with_one_zero_coefficient(on, monkeypatch, basis, log_n):
    """every flagged ciphertext has exactly one zero in one digit t_j (positions 0, 1, N/2 - 1, N/2, N - 1, a random odd one; digits
    0, a middle one, L - 1), which some rotation negates; batches of more than three rounds; once more with a small scratch cap, so
    that flagged ciphertexts are in a middle chunk and in the last one"""
    L = 3 if basis == "default" else 6
    c, o = on(basis, log_n, L)
    combos = hoist_zero_cases(o)
    G = _groups(L)
    batch = 3 * G + 1
    idx = _flagged(batch, G, len(combos))
    zeros = dict(zip(idx, combos))
    ct = th.hoist_zero_input(o, batch, zeros, 0x7E6B)
    galois = hoist_galois(o)
    for j, pos in combos:
        assert pos == 0 or any(th.negated(o, g, pos) for g in galois), pos
    keys = [o.fill_uniform(0x7E6C + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))]
    d_ct, d_keys = dev(ct), [dev(k) for k in keys]
    out = empty(len(galois), batch, 2, L, o.N)
    c.rotate_hoisted(d_ct, galois, d_keys, out, batch)
    check = sorted(set(idx) | {k + 1 for k in idx if k + 1 < batch})
    single = empty(batch, 2, L, o.N)
    for r, g in enumerate(galois):
        assert np.array_equal(host(out[r][check]).reshape(len(check), 2, L, o.N), o.rotate(ct[check], g, keys[r])), r
        c.rotate(d_ct, g, d_keys[r], single, batch)
        assert torch.equal(out[r], single), r
    per_ct = L * L * o.N * 8
    cap_mb = max(1, (batch // 4) * per_ct >> 20)
    chunk = (cap_mb << 20) // per_ct
    n_chunks = -(-batch // chunk)
    assert n_chunks >= 3 and (batch - 1) // chunk == n_chunks - 1
    assert any(0 < k // chunk < n_chunks - 1 for k in idx)
    monkeypatch.setenv("DPFHE_HOIST_CAP_MB", str(cap_mb))
    capped = empty(len(galois), batch, 2, L, o.N)
    c.rotate_hoisted(d_ct, galois, d_keys, capped, batch)
    monkeypatch.delenv("DPFHE_HOIST_CAP_MB")
    assert torch.equal(capped, out)


def test_linear_layer_with_one_zero_coefficient(dp, oracle_mod):
    """dpfhe_linear_apply takes the hoisted fallback with the layer's prepared key companions only for an input with a zero digit
    coefficient: the device and host forms against the same baby-step/giant-step schedule composed from oracle calls"""
    log_n, L, baby, giant, batch = 12, 2, 4, 3, 5
    o = oracle_mod.Oracle(log_n, L)
    c = dp.Context(log_n, L)
    gb = [o.galois_elt(b) for b in range(1, baby)]
    hit = [p for p in range(1, o.N) if any(p * g % (2 * o.N) >= o.N for g in gb)]          # negated by some baby step
    pos = [min(p for p in hit if p % 2 == 0), min(p for p in hit if p % 2), max(hit)]
    assert all(any(th.negated(o, g, p) for g in gb) for p in pos) and pos[2] >= o.N // 2
    zeros = {0: (0, pos[0]), 2: (1, pos[1]), 4: (L - 1, pos[2])}
    ct = th.hoist_zero_input(o, batch, zeros, 0x7E6D)
    diags = o.fill_uniform(0x7E6E, baby * giant)
    gk_baby = np.stack([o.fill_uniform(0x7E6F + b, 2 * L).reshape(L, 2, L, o.N) for b in range(1, baby)])
    gk_giant = o.fill_uniform(0x7E70, 2 * L).reshape(L, 2, L, o.N)
    steps = np.stack([ct] + [o.rotate(ct, g, gk_baby[b]) for b, g in enumerate(gb)])
    inner = o.ct_mul_plain_inner(steps, diags.reshape(giant, baby, L, o.N))
    want = inner[giant - 1]
    for g in range(giant - 2, -1, -1):
        want = o.poly_add(o.rotate(want, o.galois_elt(baby), gk_giant), inner[g])
    layer = dp.LinearLayer(c, diags, baby, gk_baby, gk_giant)
    out = empty(batch, 2, L, o.N)
    layer.apply(dev(ct), out, batch)
    assert np.array_equal(host(out).reshape(want.shape), want)
    out_h = np.zeros_like(want)
    layer.apply_host(ct, out_h)
    assert np.array_equal(out_h, want)
    layer.close()
    c.close()


# ---------------------------------------------------------------- CKKS
@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("L", [1, 4, 16])
def test_ckks_decode_at_the_sign_threshold(dp, oracle_mod, log_n, L):
    """coefficients at (Q - 1)/2 and either side, with leading zero Garner digits, at k and k + N/2; device and host forms"""
    o = oracle_mod.Oracle(log_n, L)
    c = dp.Context(log_n, L)
    scale = 2.0**40
    pt = np.concatenate([th.to_eval(o, th.decode_coeffs(o.moduli, o.N, 0x7E71 + s)) for s in range(2)])
    want = ckks_ref.decode(o, pt, scale)
    out = torch.empty((2, o.N // 2), dtype=torch.complex128, device="cuda")
    c.ckks_decode(dev(pt), out, 2, scale)
    assert np.array_equal(out.cpu().numpy().view(np.uint64), want.view(np.uint64))
    z_h = np.empty((2, o.N // 2), dtype=np.complex128)
    c.ckks_decode_host(pt, z_h, scale)
    assert np.array_equal(z_h.view(np.uint64), want.view(np.uint64))
    c.close()


@pytest.mark.parametrize("basis,log_n", SHAPES)
def test_ckks_encode_ties_and_exact_reduction(dp, oracle_mod, basis, log_n):
    """rint ties to even, rint(-1/4) = -0.0 (residue 0), coefficients at +-2^53, +-(2^53 + 2), +-2^63, +-2^64 and near 2^1000"""
    L = 4
    mods = th.basis_moduli(oracle_mod, basis, L)
    o = oracle_mod.Oracle(log_n, L, mods)
    c = dp.Context(log_n, L, mods)
    for scale, z, a, b in encode_groups():
        slots = np.repeat(np.array(z, dtype=np.complex128)[:, None], o.N // 2, axis=1)
        want = ckks_ref.encode(o, slots, scale)
        assert np.array_equal(want, expected_plaintexts(o, a, b)), scale
        pt = empty(len(z), L, o.N)
        c.ckks_encode(torch.from_numpy(slots).cuda(), pt, len(z), scale)
        assert np.array_equal(host(pt).reshape(want.shape), want), scale
        pt_h = np.zeros_like(want)
        c.ckks_encode_host(slots, pt_h, scale)
        assert np.array_equal(pt_h, want), scale
    c.close()
