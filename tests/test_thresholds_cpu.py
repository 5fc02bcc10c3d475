"""The kernels' data-dependent branches at their exact thresholds, without a GPU (tests/thresholds.py crafts the inputs): the oracle
against exact Python-integer definitions, so that an off-by-one shared by the oracle and the kernels cannot hide, and the kernel
bodies, run by the host emulator in both arithmetic variants, against the oracle bit for bit.  tests/test_gpu_thresholds.py is the
device twin."""
import numpy as np
import pytest

import bases
import ckks_ref
import thresholds as th
from test_ckks_encoding_cpu import EmuCkks, _build_emu_ckks, _slot_exponents

T = [0, 65537]
BASES = ["default", "gen_mixed"]


@pytest.fixture(scope="module")
def catalogue(oracle_mod):
    return bases.catalogue(oracle_mod)


def _oracle(oracle_mod, catalogue, basis, log_n, L):
    return oracle_mod.Oracle(log_n, L, th.basis_moduli(oracle_mod, basis, L))


def _variants(o):
    """both arithmetic variants where the moduli allow the fast one"""
    return ["fast", "gen"] if all(bases.is_fast(q) for q in o.moduli) else ["gen"]


def _lower(oracle_mod, o, limbs):
    return oracle_mod.Oracle(o.logn, limbs, o.moduli[:limbs])


def _hybrid_acc(o, d, key):
    """the hybrid key switch's inner product over all L limbs, [2][L][N], from the oracle's exact transforms and products"""
    Lq = o.L - 1
    dc = th._coeff(o, d[None], Lq)[0]
    acc = np.zeros((2, o.L, o.N), dtype=np.uint64)
    for j in range(Lq):
        u = o.ntt_fwd(np.stack([dc[j] % np.uint64(q) for q in o.moduli])[None])[0]
        for c in range(2):
            acc[c] = o.poly_add(acc[c][None], o.poly_mul_pointwise(u[None], key[j, c][None]))[0]
    return acc


def _grouped_acc(o, K, d, key):
    """the grouped key switch's inner product over all L limbs, [2][L][N]: mod-up of DESIGN.md section 2.11 in Python integers"""
    Lq = o.L - K
    dc = th._coeff(o, d[None], Lq)[0]
    acc = np.zeros((2, o.L, o.N), dtype=np.uint64)
    for g in range(o.grouped_digits(K)):
        lo, hi = g * K, min(g * K + K, Lq)
        qs = o.moduli[lo:hi]
        Qg = th._prod(qs)
        ys = [[v * pow(Qg // q % q, -1, q) % q for v in th._ints(dc[j])] for j, q in zip(range(lo, hi), qs)]
        lift = [sum(y[n] * (Qg // q) for y, q in zip(ys, qs)) for n in range(o.N)]
        u = np.array([[v % q for v in lift] for q in o.moduli], dtype=np.uint64)
        u[lo:hi] = dc[lo:hi]                                 # limbs of the digit: the digit itself
        u = o.ntt_fwd(u[None])[0]
        for c in range(2):
            acc[c] = o.poly_add(acc[c][None], o.poly_mul_pointwise(u[None], key[g, c][None]))[0]
    return acc


def _check_composition(lo, d, keyswitch, a, b, mul, rots, o):
    """ct x ct and the rotations key-switch exactly the crafted digits d: (d0 + ks0, d1 + ks1) with d2 = a1 b1 = d, and
    (sigma(c0) + ks0, ks1) with sigma(c1) = d.  lo: the oracle of the ciphertext moduli."""
    tens = lo.ct_tensor(a, b)
    assert np.array_equal(tens[:, 2], d)
    for k in range(d.shape[0]):
        ks = np.stack(keyswitch(k))
        assert np.array_equal(mul[k], lo.poly_add(tens[k, :2], ks)), k
        for g, (ct, rot) in rots.items():
            perm = o.galois_perm(g)
            assert np.array_equal(rot[k, 1], ks[1]) and np.array_equal(rot[k, 0], lo.poly_add(ct[k, 0][None, :, perm], ks[:1])[0]), (g, k)


# ---------------------------------------------------------------- division by one modulus
@pytest.mark.parametrize("basis,log_n", [("default", 12), ("gen_mixed", 12), ("default", 14)])
@pytest.mark.parametrize("t", T)
def test_mod_switch_down_at_threshold(oracle_mod, make_emu, catalogue, basis, log_n, t):
    L = 3 if basis == "default" else 6
    o = _oracle(oracle_mod, catalogue, basis, log_n, L)
    x = th.mod_switch_input(o, 2, t, 0x7E51)
    want = o.mod_switch_down(x, t)
    assert np.array_equal(_lower(oracle_mod, o, L - 1).ntt_inv(want), th.exact_mod_switch(o, x, t))
    for v in _variants(o):
        assert np.array_equal(make_emu(log_n, L, o.moduli, v).mod_switch(x, t), want), v


@pytest.mark.parametrize("basis", BASES)
@pytest.mark.parametrize("t", T)
def test_hybrid_family_at_threshold(oracle_mod, make_emu, catalogue, basis, t):
    """tau' of the special accumulator at the threshold through the key: bare key switch, ct x ct, rotations (g = 1 and a real g)"""
    L, batch = (4 if basis == "default" else 6), 2
    o = _oracle(oracle_mod, catalogue, basis, 12, L)
    lo = _lower(oracle_mod, o, L - 1)
    key = th.hybrid_key(o, 0x7E52)
    d = th.hybrid_digits(o, batch, t, 0x7E53)
    for k in range(batch):
        c0, c1 = o.keyswitch_hybrid(d[k], key, t)
        assert np.array_equal(lo.ntt_inv(np.stack([c0, c1])), th.exact_mod_switch(o, _hybrid_acc(o, d[k], key), t)), k
    a, b = th.mul_inputs(o, d, 0x7E54)
    mul = o.ct_mul_relin_hybrid(a, b, key, t)
    rots = {g: th.rotate_inputs(o, d, g, 0x7E55) for g in (1, o.galois_elt(3))}
    _check_composition(lo, d, lambda k: o.keyswitch_hybrid(d[k], key, t), a, b, mul,
                       {g: (ct, o.rotate_hybrid(ct, g, key, t)) for g, ct in rots.items()}, o)
    for v in _variants(o):
        e = make_emu(12, L, o.moduli, v)
        got = e.ks_hybrid(1, d, None, key, batch, t_plain=t)
        for k in range(batch):
            assert np.array_equal(got[k], np.stack(o.keyswitch_hybrid(d[k], key, t))), (v, k)
        assert np.array_equal(e.ks_hybrid(0, a, b, key, batch, t_plain=t), mul), v
        for g, ct in rots.items():
            assert np.array_equal(e.ks_hybrid(2, ct, None, key, batch, galois=g, t_plain=t), o.rotate_hybrid(ct, g, key, t)), (v, g)


# ---------------------------------------------------------------- division by P
@pytest.mark.parametrize("basis,log_n", [("default", 12), ("gen_mixed", 12), ("default", 14)])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_mod_down_special_at_threshold(oracle_mod, make_emu, catalogue, basis, log_n, K):
    """every y_k at, below and above p_k/2, and all of them above at once (K = 4: the per-term reduction of the lift)"""
    L = th.special_limbs(K)
    o = _oracle(oracle_mod, catalogue, basis, log_n, L)
    lo = _lower(oracle_mod, o, L - K)
    for t in T:
        x = th.mod_down_input(o, K, 2, t, 0x7E56 + K)
        want = o.mod_down_special(K, x, t)
        assert np.array_equal(lo.ntt_inv(want), th.exact_mod_down(o, K, x, t)), t
        if K == 1:
            assert np.array_equal(want, o.mod_switch_down(x, t))
        for v in _variants(o):
            assert np.array_equal(make_emu(log_n, L, o.moduli, v).mod_down_special(K, x, t), want), (v, t)


@pytest.mark.parametrize("basis", BASES)
@pytest.mark.parametrize("K", [1, 2, 4])
def test_grouped_family_at_threshold(oracle_mod, make_emu, catalogue, basis, K):
    """y_k at the threshold through the key: bare key switch, ct x ct, rotations (g = 1 and a real g), hoisted rotations"""
    L, batch, t = th.special_limbs(K), 2, 65537
    o = _oracle(oracle_mod, catalogue, basis, 12, L)
    Lq = L - K
    lo = _lower(oracle_mod, o, Lq)
    key = th.grouped_key(o, K, 0x7E57)
    d = th.grouped_digits_input(o, K, batch, t, 0x7E58 + K)
    for k in range(batch):
        c0, c1 = o.keyswitch_grouped(K, d[k], key, t)
        assert np.array_equal(lo.ntt_inv(np.stack([c0, c1])), th.exact_mod_down(o, K, _grouped_acc(o, K, d[k], key), t)), k
    a, b = th.mul_inputs(o, d, 0x7E59)
    mul = o.ct_mul_relin_grouped(K, a, b, key, t)
    rots = {g: th.rotate_inputs(o, d, g, 0x7E5A) for g in (1, o.galois_elt(-2))}
    _check_composition(lo, d, lambda k: o.keyswitch_grouped(K, d[k], key, t), a, b, mul,
                       {g: (ct, o.rotate_grouped(K, ct, g, key, t)) for g, ct in rots.items()}, o)
    # hoisted: the mod-up of the unpermuted c1 = d, so with g = 1 the crafted y_k are those of the division
    ct = rots[1]
    galois = [1, o.galois_elt(3), 2 * o.N - 1]
    keys = np.stack([key] * len(galois))
    hoisted = o.rotate_hoisted_grouped(K, ct, galois, keys, t)
    assert np.array_equal(hoisted[0], o.rotate_grouped(K, ct, 1, key, t))
    for v in _variants(o):
        e = make_emu(12, L, o.moduli, v)
        got = e.ks_grouped(K, 1, d, None, key, batch, t_plain=t)
        for k in range(batch):
            assert np.array_equal(got[k], np.stack(o.keyswitch_grouped(K, d[k], key, t))), (v, k)
        assert np.array_equal(e.ks_grouped(K, 0, a, b, key, batch, t_plain=t), mul), v
        for g, c in rots.items():
            assert np.array_equal(e.ks_grouped(K, 2, c, None, key, batch, galois=g, t_plain=t), o.rotate_grouped(K, c, g, key, t)), (v, g)
        assert np.array_equal(e.rotate_hoisted_grouped(K, ct, galois, keys, t), hoisted), v


# ---------------------------------------------------------------- hoisted rotations: one zero coefficient in a digit
def hoist_zero_cases(o):
    """(digit, position) of a crafted zero: positions 0, 1, N/2 - 1, N/2, N - 1 and a random odd one, digits 0, a middle one and L - 1"""
    N, L = o.N, o.L
    odd = 2 * int(np.random.default_rng(N + L).integers(1, N // 2 - 1)) + 1
    return [(j, pos) for pos in (0, 1, N // 2 - 1, N // 2, N - 1, odd) for j in sorted({0, L // 2, L - 1})]


def hoist_galois(o):
    return [o.galois_elt(1), o.galois_elt(-1), 2 * o.N - 1]


def check_negated(o, galois, zeros):
    """every crafted zero but one at position 0 (X^0 is fixed by every sigma_g) is negated by some rotation: there, a missed flag
    gives other bits than the fallback"""
    for j, pos in zeros:
        assert pos == 0 or any(th.negated(o, g, pos) for g in galois), pos


@pytest.mark.parametrize("basis", BASES)
def test_rotate_hoisted_with_one_zero_coefficient(oracle_mod, make_emu, catalogue, basis):
    L = 3 if basis == "default" else 6
    o = _oracle(oracle_mod, catalogue, basis, 12, L)
    combos = hoist_zero_cases(o)
    batch = len(combos) + 3
    zeros = {k + 1: c for k, c in enumerate(combos)}        # ciphertext 0 and the last two have no zero
    ct = th.hoist_zero_input(o, batch, zeros, 0x7E5B)
    galois = hoist_galois(o)
    check_negated(o, galois, combos)
    keys = np.stack([o.fill_uniform(0x7E5C + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))])
    want = [o.rotate(ct, g, keys[r]) for r, g in enumerate(galois)]
    for v in _variants(o):
        got, flagged = make_emu(12, L, o.moduli, v).rotate_hoisted(ct, galois, keys)
        assert flagged == len(zeros), v
        for r in range(len(galois)):
            assert np.array_equal(got[r], want[r]), (v, r)


# ---------------------------------------------------------------- CKKS decoding: the sign of X and the digits of Q - X
@pytest.fixture(scope="module")
def emu_ckks():
    return {v: _build_emu_ckks(v) for v in ("gen", "fast")}


def _exact_slots(X, moduli, scale, n, js):
    """slots js of the decoding of coefficients X (integers mod Q): centred(X) / scale through the long-double definition"""
    Q = th._prod(moduli)
    c = np.array([float((x - Q if 2 * x > Q else x) / int(scale)) for x in X], dtype=np.longdouble)
    e = _slot_exponents(n)
    ang = np.pi * np.arange(2 * n, dtype=np.longdouble) / n
    cos_t, sin_t = np.cos(ang), np.sin(ang)
    out = []
    for j in js:
        idx = (e[j] * np.arange(n)) % (2 * n)
        out.append(complex((c * cos_t[idx]).sum(), (c * sin_t[idx]).sum()))
    return np.array(out), np.abs(c).sum()


@pytest.mark.parametrize("L", [1, 4, 16])
def test_ckks_decode_at_the_sign_threshold(oracle_mod, emu_ckks, L):
    logn, n, scale = 12, 4096, 2.0**40
    o = oracle_mod.Oracle(logn, L)
    X = th.decode_coeffs(o.moduli, n, 0x7E5D + L)
    Q = th._prod(o.moduli)
    h = (Q - 1) // 2
    assert [th.centred(v, Q) for v in (h, h + 1)] == [h, h + 1 - Q]
    pt = th.to_eval(o, X)
    got = ckks_ref.decode(o, pt, scale)[0]
    js = list(range(0, n // 2, 97)) + [n // 2 - 1]
    want, mass = _exact_slots(X, o.moduli, scale, n, js)
    assert np.all(np.abs(got[js] - want) <= 2.0**-53 * 2 * logn * mass)    # DESIGN.md 2.12's bound
    for v in ("gen", "fast"):
        emu = EmuCkks(emu_ckks[v], logn, o.moduli)
        assert np.array_equal(emu.decode(pt, scale).view(np.uint64), got[None].view(np.uint64)), v


@pytest.mark.parametrize("L", [1, 4])
def test_ckks_decode_constant_at_the_threshold(oracle_mod, emu_ckks, L):
    """one coefficient X alone: every slot is centred(X) / scale, so the sign and the digits of Q - X are seen directly"""
    logn, n, scale = 12, 4096, 2.0**40
    o = oracle_mod.Oracle(logn, L)
    Q = th._prod(o.moduli)
    vals = th.decode_values(o.moduli)
    pts = np.concatenate([th.to_eval(o, [v] + [0] * (n - 1)) for v in vals])
    got = ckks_ref.decode(o, pts, scale)
    for v, z in zip(vals, got):
        want = th.centred(v, Q) / int(scale)
        assert np.all(z.imag == 0) and np.all(np.abs(z.real - want) <= abs(want) * L * 2.0**-52), v
    for var in ("gen", "fast"):
        assert np.array_equal(EmuCkks(emu_ckks[var], logn, o.moduli).decode(pts, scale).view(np.uint64), got.view(np.uint64)), var


# ---------------------------------------------------------------- CKKS encoding: ties to even, the sign of zero, exact reduction
def encode_groups():
    """the constant-slot cases grouped by scale: [(scale, slots [n_case], coefficient 0 [n_case], coefficient N/2 [n_case])]"""
    out = {}
    for z, sc, a, b in th.constant_slot_cases():
        out.setdefault(sc, []).append((z, a, b))
    return [(sc, [c[0] for c in v], [c[1] for c in v], [c[2] for c in v]) for sc, v in out.items()]


def expected_plaintexts(o, a, b):
    """[n_case][L][N] evaluation form of a X^0 + b X^(N/2), reduced exactly"""
    res = np.zeros((len(a), o.L, o.N), dtype=np.uint64)
    for k, (x, y) in enumerate(zip(a, b)):
        for i, q in enumerate(o.moduli):
            res[k, i, 0], res[k, i, o.N // 2] = x % q, y % q
    return o.ntt_fwd(res)


@pytest.mark.parametrize("basis", ["default", "gen_mixed"])
def test_ckks_encode_ties_and_exact_reduction(oracle_mod, emu_ckks, catalogue, basis):
    logn, n, L = 12, 4096, 4
    o = _oracle(oracle_mod, catalogue, basis, logn, L)
    for scale, z, a, b in encode_groups():
        slots = np.repeat(np.array(z, dtype=np.complex128)[:, None], n // 2, axis=1)
        pt, cf = ckks_ref.encode(o, slots, scale, with_coeffs=True)
        want_cf = np.zeros((len(z), n))
        want_cf[:, 0], want_cf[:, n // 2] = [float(x) for x in a], [float(y) for y in b]
        assert np.array_equal(cf, want_cf), scale
        assert [int(x) for x in cf[:, 0]] == a and [int(y) for y in cf[:, n // 2]] == b
        assert np.array_equal(pt, expected_plaintexts(o, a, b)), scale
        for v in _variants(o):
            assert np.array_equal(EmuCkks(emu_ckks[v], logn, o.moduli).encode(slots, scale), pt), (v, scale)
