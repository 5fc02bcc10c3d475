"""The kernel bodies on the bases of tests/bases.py, through the host emulator, against the oracle bit for bit: every body at
N = 4096 and 16384 with the arithmetic variant the library picks for the basis, and the fast bases once more through the generic
variant.  tests/test_gpu_bases.py is the device twin; what only the device runs (PTX arithmetic, TMA and cluster forms, the launch
orchestration of abi.cu) is checked there."""
import numpy as np
import pytest

import bases

CASES = [(name, log_n, None) for name in bases.NAMES for log_n in (12, 14)] + \
        [(name, log_n, "gen") for name in bases.NAMES if bases.PATHS[name][0] for log_n in (12, 14)]


@pytest.fixture(scope="module")
def catalogue(oracle_mod):
    return bases.catalogue(oracle_mod)


def test_catalogue_selects_its_paths(catalogue):
    """the catalogue keeps covering what it was made to cover (bases.check_paths runs on every derivation; spelled out here)"""
    assert bases.selects(catalogue["gen_mixed"]) == (False, True, "none")
    assert bases.selects(catalogue["gen_near60"]) == (False, False, "all")
    assert bases.selects(catalogue["fast_mixed"]) == (True, True, "none")
    assert bases.selects(catalogue["fast_narrow"]) == (True, False, "none")
    assert catalogue["gen_ascending"] == sorted(catalogue["gen_mixed"])


def _edge(o, n_polys, seed):
    x = o.fill_uniform(seed, n_polys)
    q = np.array(o.moduli, dtype=np.uint64)
    x[0] = (q - 1)[:, None]
    x[-1, :, ::2] = 0
    x[-1, :, 1::2] = (q - 1)[:, None]
    return x


def _reduced(o, x, Lq):
    """ciphertexts x (with the L limbs of `o`) cut to their first Lq limbs, the first row set to q - 1"""
    y = np.ascontiguousarray(x[..., :Lq, :])
    y[0, 0] = (np.array(o.moduli[:Lq], dtype=np.uint64) - 1)[:, None]
    return y


@pytest.mark.parametrize("name,log_n,variant", CASES)
def test_bodies_on_basis(make_emu, oracle_mod, catalogue, name, log_n, variant):
    mods = catalogue[name]
    L = len(mods)
    e, o = make_emu(log_n, L, mods, variant=variant), oracle_mod.Oracle(log_n, L, mods)
    assert e.moduli == o.moduli == mods and e.psi == o.psi
    batch = 2
    # transforms (and the CTA-pair form at N = 16384)
    x = _edge(o, 2, 1)
    y = e.ntt(x)
    assert np.array_equal(y, o.ntt_fwd(x))
    assert np.array_equal(e.ntt(y, inverse=True), x)
    if log_n == 14:
        assert np.array_equal(e.ntt_pair(x), y)
        assert np.array_equal(e.ntt_pair(y, inverse=True), x)
    # fused key switching, all three modes (conjugation for the rotation)
    s = o.keygen_secret(2)
    evk = o.keygen_relin(3, 65537, s)
    a = _edge(o, 2 * batch, 4).reshape(batch, 2, L, o.N)
    b = o.fill_uniform(5, 2 * batch).reshape(batch, 2, L, o.N)
    assert np.array_equal(e.ks(0, a, b, evk, batch), o.ct_mul_relin(a, b, evk))
    d = np.ascontiguousarray(a[:, 1])
    got = e.ks(1, d, None, evk, batch)
    for k in range(batch):
        assert np.array_equal(got[k], np.stack(o.keyswitch(d[k], evk)))
    g = 2 * o.N - 1
    gk = o.keygen_galois(6, 65537, s, g)
    assert np.array_equal(e.ks(2, a, None, gk, batch, galois=g), o.rotate(a, g, gk))
    # hoisted rotations; c1 = 0 in the last ciphertext takes the fallback
    ct = a.copy()
    ct[-1, 1] = 0
    galois = [o.galois_elt(1), 2 * o.N - 1]
    keys = np.stack([o.fill_uniform(7 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))])
    hot, _ = e.rotate_hoisted(ct, galois, keys)
    for r, g in enumerate(galois):
        assert np.array_equal(hot[r], o.rotate(ct, g, keys[r])), r
    # modulus switch, plain and BGV-corrected
    for t in (0, 65537):
        assert np.array_equal(e.mod_switch(x, t), o.mod_switch_down(x, t)), t
    # one special prime: the three modes
    ah = _reduced(o, a, L - 1)
    bh = np.ascontiguousarray(b[:, :, :L - 1])
    hkey = o.fill_uniform(9, 2 * (L - 1)).reshape(L - 1, 2, L, o.N)
    assert np.array_equal(e.ks_hybrid(0, ah, bh, hkey, batch, t_plain=65537), o.ct_mul_relin_hybrid(ah, bh, hkey, 65537))
    g = o.galois_elt(-2)
    assert np.array_equal(e.ks_hybrid(2, ah, None, hkey, batch, galois=g, t_plain=65537), o.rotate_hybrid(ah, g, hkey, 65537))
    dh = np.ascontiguousarray(ah[:, 1])
    got = e.ks_hybrid(1, dh, None, hkey, batch)
    for k in range(batch):
        assert np.array_equal(got[k], np.stack(o.keyswitch_hybrid(dh[k], hkey, 0)))
    # two special primes: digits of two limbs (the last one ragged in the mod-up), the three modes, the division by P,
    # the hoisted rotations
    K = 2
    ag = _reduced(o, a, L - K)
    bg = np.ascontiguousarray(b[:, :, :L - K])
    dnum = o.grouped_digits(K)
    gkey = o.fill_uniform(10, 2 * dnum).reshape(dnum, 2, L, o.N)
    assert np.array_equal(e.ks_grouped(K, 0, ag, bg, gkey, batch, t_plain=65537), o.ct_mul_relin_grouped(K, ag, bg, gkey, 65537))
    assert np.array_equal(e.ks_grouped(K, 2, ag, None, gkey, batch, galois=g), o.rotate_grouped(K, ag, g, gkey, 0))
    dg = np.ascontiguousarray(ag[:, 1])
    got = e.ks_grouped(K, 1, dg, None, gkey, batch, t_plain=65537)
    for k in range(batch):
        assert np.array_equal(got[k], np.stack(o.keyswitch_grouped(K, dg[k], gkey, 65537)))
    for t in (0, 65537):
        assert np.array_equal(e.mod_down_special(K, x, t), o.mod_down_special(K, x, t)), t
    gkeys = np.stack([o.fill_uniform(11 + r, 2 * dnum).reshape(dnum, 2, L, o.N) for r in range(2)])
    assert np.array_equal(e.rotate_hoisted_grouped(K, ag, galois, gkeys, 65537), o.rotate_hoisted_grouped(K, ag, galois, gkeys, 65537))
    # plaintext inner products: a ragged count of baby steps, an all-(q - 1) tile
    nb, ng = 5, 2
    steps = o.fill_uniform(13, nb * 2).reshape(nb, 1, 2, L, o.N)
    pts = o.fill_uniform(14, ng * nb).reshape(ng, nb, L, o.N)
    q = np.array(mods, dtype=np.uint64)
    steps[:, 0, 0] = (q - 1)[:, None]
    pts[0] = (q - 1)[:, None]
    assert np.array_equal(e.pt_inner(steps, pts), o.ct_mul_plain_inner(steps, pts))
