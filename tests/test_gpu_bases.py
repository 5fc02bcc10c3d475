"""Every entry point on the bases of tests/bases.py, bit for bit against the oracle: the generic kernels (all three compiled
objects: main, one special prime, grouped), the fast kernels without the default basis's shortcuts, the smallest and the largest
admissible moduli.  The emulator (tests/test_bases_cpu.py) checks the kernel bodies on the same bases; what it cannot check runs
here: the device arithmetic (PTX), the TMA and cluster forms, and the orchestration of abi.cu.

Also: the persistent kernels over several rounds per group, a host-buffer entry point, a decryption of a generic-basis product,
and every runtime tuning switch (DPFHE_NTT_CFG, DPFHE_ROT_CFG, DPFHE_KS_PF, DPFHE_KS_OCC, DPFHE_KS_PROF) on the default basis and
on a generic one."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import bases  # noqa: E402
from test_gpu_grouped import grouped_inputs  # noqa: E402
from test_gpu_parity import ctxs, dev, dp, edge_polys, host, hybrid_inputs  # noqa: E402,F401  (ctxs and dp are fixtures)

L = bases.N_LIMBS
K = 2   # special primes of the grouped family: three digits of two limbs
SHAPES = [(name, log_n) for name in bases.NAMES for log_n in (12, 14)] + [("gen_mixed", 13), ("fast_mixed", 13)]


@pytest.fixture(scope="module")
def catalogue(oracle_mod):
    return bases.catalogue(oracle_mod)


@pytest.fixture
def on(ctxs, catalogue):
    def get(name, log_n):
        c, o = ctxs(log_n, L, catalogue[name])
        assert c.moduli == o.moduli == catalogue[name] and c.psi == o.psi
        return c, o
    return get


def rounds_batch(ctas_per_sm):
    """a batch that gives every group of a persistent kernel at least three rounds: the kernels run at most ctas_per_sm CTAs
    per SM (four: the context's digit slots) in groups of L CTAs, one ciphertext per group and round"""
    groups = ctas_per_sm * torch.cuda.get_device_properties(0).multi_processor_count // L
    return 3 * groups + 1


def conj(o):
    return 2 * o.N - 1


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_ntt(dp, on, monkeypatch, name, log_n):
    """forward and inverse transforms; the inverse by TMA and by thread copies at N <= 8192, the CTA pair at N = 16384"""
    c, o = on(name, log_n)
    x = edge_polys(o, 5, 0xBA5E0001)
    want = o.ntt_fwd(x)
    d = dev(x)
    c.ntt_fwd(d, 5)
    assert np.array_equal(host(d).reshape(x.shape), want)
    c.ntt_inv(d, 5)
    assert np.array_equal(host(d).reshape(x.shape), x)
    if log_n <= 13:
        monkeypatch.setenv("DPFHE_NTT_TMA", "0")
        c2 = dp.Context(log_n, L, c.moduli)
        monkeypatch.delenv("DPFHE_NTT_TMA")
        d = dev(want)
        c2.ntt_inv(d, 5)
        assert np.array_equal(host(d).reshape(x.shape), x)
        c2.close()


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_elementwise(on, name, log_n):
    c, o = on(name, log_n)
    B = 3
    a = edge_polys(o, 2 * B, 11).reshape(B, 2, L, o.N)
    b = edge_polys(o, 2 * B, 12)[::-1].copy().reshape(B, 2, L, o.N)
    da, db = dev(a), dev(b)
    out = torch.full_like(da, -1)
    c.poly_mul_pointwise(da, db, out, 2 * B)
    assert np.array_equal(host(out).reshape(a.shape), o.poly_mul_pointwise(a, b))
    d = torch.full((B, 3, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_tensor(da, db, d, B)
    assert np.array_equal(host(d).reshape(B, 3, L, o.N), o.ct_tensor(a, b))
    pt = edge_polys(o, 3, 13)[1]                       # all q - 1
    c.ct_mul_plain(da, dev(pt), out, B)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_plain(a, pt))
    f = torch.empty((3, L, o.N), dtype=torch.int64, device="cuda")
    c.fill_uniform(0xBA5E0002, f, 3, first_poly=7)
    assert np.array_equal(host(f).reshape(3, L, o.N), o.fill_uniform(0xBA5E0002, 3, first_poly=7))


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_keyswitch_family(on, name, log_n):
    """the fused key-switch kernel: ct x ct, the bare key switch, rotations including the conjugation"""
    c, o = on(name, log_n)
    batch = 3
    s = o.keygen_secret(21)
    evk = o.keygen_relin(22, 65537, s)
    a = edge_polys(o, 2 * batch, 23).reshape(batch, 2, L, o.N)
    b = o.fill_uniform(24, 2 * batch).reshape(batch, 2, L, o.N)
    out = torch.full((batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin(dev(a), dev(b), dev(evk), out, batch)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin(a, b, evk))
    d = np.ascontiguousarray(a[:, 1])
    c.keyswitch(dev(d), dev(evk), out, batch)
    want = np.stack([np.stack(o.keyswitch(d[k], evk)) for k in range(batch)])
    assert np.array_equal(host(out).reshape(want.shape), want)
    for g in (o.galois_elt(1), o.galois_elt(-3), conj(o)):
        gk = o.keygen_galois(25 + g % 7, 65537, s, g)
        c.rotate(dev(a), g, dev(gk), out, batch)
        assert np.array_equal(host(out).reshape(a.shape), o.rotate(a, g, gk)), g


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_rotate_hoisted(on, name, log_n):
    """shared digit transforms; a ciphertext with c1 = 0 and one with a zero digit take the fallback (the ordinary rotation)"""
    c, o = on(name, log_n)
    batch = 3
    ct = edge_polys(o, 2 * batch, 91).reshape(batch, 2, L, o.N)
    ct[batch - 1, 1] = 0
    ct[1, 1, L - 1] = 0
    galois = [o.galois_elt(1), o.galois_elt(-1), o.galois_elt(7), conj(o)]
    keys = [o.fill_uniform(100 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))]
    d_keys = [dev(k) for k in keys]
    out = torch.full((len(galois), batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    d_ct = dev(ct)
    c.rotate_hoisted(d_ct, galois, d_keys, out, batch)
    single = torch.empty((batch, 2, L, o.N), dtype=torch.int64, device="cuda")
    for r, g in enumerate(galois):
        assert np.array_equal(host(out[r]).reshape(ct.shape), o.rotate(ct, g, keys[r])), r
        c.rotate(d_ct, g, d_keys[r], single, batch)
        assert torch.equal(out[r], single), r


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_mod_switch_down(on, name, log_n):
    c, o = on(name, log_n)
    n = 4
    x = edge_polys(o, n, 71)
    for t in (0, 65537):
        out = torch.full((n, L - 1, o.N), -1, dtype=torch.int64, device="cuda")
        c.mod_switch_down(dev(x), out, n, t)
        assert np.array_equal(host(out).reshape(n, L - 1, o.N), o.mod_switch_down(x, t)), t


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_hybrid_family(on, name, log_n):
    """one special prime (the basis's last modulus): ct x ct, rotation, bare key switch"""
    c, o = on(name, log_n)
    batch, t = 3, 65537
    a, key = hybrid_inputs(o, batch, 81)
    b, _ = hybrid_inputs(o, batch, 83)
    out = torch.full((batch, 2, L - 1, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin_hybrid(dev(a), dev(b), dev(key), out, batch, t)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin_hybrid(a, b, key, t))
    for g in (o.galois_elt(-2), conj(o)):
        c.rotate_hybrid(dev(a), g, dev(key), out, batch, t)
        assert np.array_equal(host(out).reshape(a.shape), o.rotate_hybrid(a, g, key, t)), g
    d = np.ascontiguousarray(a[:, 1])
    c.keyswitch_hybrid(dev(d), dev(key), out, batch, 0)
    got = host(out).reshape(a.shape)
    for k in range(batch):
        c0, c1 = o.keyswitch_hybrid(d[k], key, 0)
        assert np.array_equal(got[k, 0], c0) and np.array_equal(got[k, 1], c1), k


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_grouped_family(on, name, log_n):
    """two special primes, digits of two limbs: ct x ct, rotation, bare key switch"""
    c, o = on(name, log_n)
    batch, t = 3, 65537
    a, key = grouped_inputs(o, K, batch, 81)
    b, _ = grouped_inputs(o, K, batch, 83)
    out = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin_grouped(K, dev(a), dev(b), dev(key), out, batch, t)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin_grouped(K, a, b, key, t))
    for g in (o.galois_elt(-2), conj(o)):
        c.rotate_grouped(K, dev(a), g, dev(key), out, batch, t)
        assert np.array_equal(host(out).reshape(a.shape), o.rotate_grouped(K, a, g, key, t)), g
    d = np.ascontiguousarray(a[:, 1])
    c.keyswitch_grouped(K, dev(d), dev(key), out, batch, 0)
    got = host(out).reshape(a.shape)
    for k in range(batch):
        c0, c1 = o.keyswitch_grouped(K, d[k], key, 0)
        assert np.array_equal(got[k, 0], c0) and np.array_equal(got[k, 1], c1), k


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_mod_down_special(on, name, log_n):
    c, o = on(name, log_n)
    n = 4
    x = edge_polys(o, n, 41)
    for t in (0, 65537):
        out = torch.full((n, L - K, o.N), -1, dtype=torch.int64, device="cuda")
        c.mod_down_special(K, dev(x), out, n, t)
        assert np.array_equal(host(out).reshape(n, L - K, o.N), o.mod_down_special(K, x, t)), t


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_rotate_hoisted_grouped(on, name, log_n):
    c, o = on(name, log_n)
    batch, t = 3, 65537
    ct, _ = grouped_inputs(o, K, batch, 51)
    galois = [o.galois_elt(1), o.galois_elt(-2), conj(o)]
    dnum = o.grouped_digits(K)
    keys = [o.fill_uniform(60 + r, 2 * dnum).reshape(dnum, 2, L, o.N) for r in range(len(galois))]
    out = torch.full((len(galois), batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted_grouped(K, dev(ct), galois, [dev(k) for k in keys], out, batch, t)
    want = o.rotate_hoisted_grouped(K, ct, galois, np.stack(keys), t)
    assert np.array_equal(host(out).reshape(want.shape), want)


@pytest.mark.parametrize("name,log_n", SHAPES)
def test_plain_inner_products(on, name, log_n):
    """nb = 19 baby steps (not a multiple of the 16-product flush), an all-(q - 1) plaintext tile and ciphertext row"""
    c, o = on(name, log_n)
    nb, ng, batch = 19, 3, 2
    steps = o.fill_uniform(51, nb * batch * 2).reshape(nb, batch, 2, L, o.N)
    pts = o.fill_uniform(52, ng * nb).reshape(ng, nb, L, o.N)
    q = np.array(o.moduli, dtype=np.uint64)
    steps[:, 0, 0] = (q - 1)[:, None]
    pts[0] = (q - 1)[:, None]
    pts[-1, :, :, ::3] = 0
    out = torch.full((ng, batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_mul_plain_inner(dev(steps), dev(pts), out, nb, ng, batch)
    assert np.array_equal(host(out).reshape(ng, batch, 2, L, o.N), o.ct_mul_plain_inner(steps, pts))


@pytest.mark.parametrize("family", ["fused", "hybrid", "grouped", "hoist", "hoist_grouped"])
def test_persistent_kernels_over_many_rounds(on, family):
    """every group of a persistent kernel runs at least three rounds, so the generic kernels' digit slots, flags and mailboxes
    change round parity under load (gen_mixed, N = 4096)"""
    c, o = on("gen_mixed", 12)
    batch, t = rounds_batch(4), 65537
    if family == "fused":
        a = o.fill_uniform(1, 2 * batch).reshape(batch, 2, L, o.N)
        b = o.fill_uniform(2, 2 * batch).reshape(batch, 2, L, o.N)
        key = o.fill_uniform(3, 2 * L).reshape(L, 2, L, o.N)
        out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
        c.ct_mul_relin(dev(a), dev(b), dev(key), out, batch)
        want = o.ct_mul_relin(a, b, key)
    elif family == "hybrid":
        a, key = hybrid_inputs(o, batch, 4)
        b, _ = hybrid_inputs(o, batch, 6)
        out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
        c.ct_mul_relin_hybrid(dev(a), dev(b), dev(key), out, batch, t)
        want = o.ct_mul_relin_hybrid(a, b, key, t)
    elif family == "grouped":
        a, key = grouped_inputs(o, K, batch, 8)
        b, _ = grouped_inputs(o, K, batch, 10)
        out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
        c.ct_mul_relin_grouped(K, dev(a), dev(b), dev(key), out, batch, t)
        want = o.ct_mul_relin_grouped(K, a, b, key, t)
    elif family == "hoist":
        a = o.fill_uniform(12, 2 * batch).reshape(batch, 2, L, o.N)
        a[batch // 2, 1] = 0
        g = o.galois_elt(3)
        key = o.fill_uniform(13, 2 * L).reshape(L, 2, L, o.N)
        out = torch.full((1,) + a.shape, -1, dtype=torch.int64, device="cuda")
        c.rotate_hoisted(dev(a), [g], [dev(key)], out, batch)
        want = o.rotate(a, g, key)[None]
    else:
        a, key = grouped_inputs(o, K, batch, 14)
        g = o.galois_elt(3)
        out = torch.full((1,) + a.shape, -1, dtype=torch.int64, device="cuda")
        c.rotate_hoisted_grouped(K, dev(a), [g], [dev(key)], out, batch, t)
        want = o.rotate_hoisted_grouped(K, a, [g], key[None], t)
    got = host(out).reshape(want.shape)
    bad = [k for k in range(batch) if not np.array_equal(got[..., k, :, :, :], want[..., k, :, :, :])]
    assert not bad, "ciphertexts %s of %d differ" % (bad[:8], batch)


def test_host_entry_points_on_a_generic_basis(on):
    """the host-buffer forms (staging pipeline of abi.cu) on gen_mixed"""
    c, o = on("gen_mixed", 12)
    batch = 5
    s = o.keygen_secret(31)
    evk = o.keygen_relin(32, 65537, s)
    a = edge_polys(o, 2 * batch, 33).reshape(batch, 2, L, o.N)
    b = o.fill_uniform(34, 2 * batch).reshape(batch, 2, L, o.N)
    out = np.zeros_like(a)
    c.ct_mul_relin_host(a, b, evk, out)
    assert np.array_equal(out, o.ct_mul_relin(a, b, evk))
    ga, gkey = grouped_inputs(o, K, batch, 35)
    gb, _ = grouped_inputs(o, K, batch, 37)
    gout = np.zeros_like(ga)
    c.ct_mul_relin_grouped_host(K, ga, gb, gkey, gout, 65537)
    assert np.array_equal(gout, o.ct_mul_relin_grouped(K, ga, gb, gkey, 65537))


@pytest.mark.parametrize("name", ["gen_mixed", "gen_ascending"])
def test_decrypt_generic_hybrid_product(oracle_mod, on, name):
    """Dec(GPU hybrid ct x ct) == m1 * m2 on a generic basis: the kernels against the scheme, not only against the oracle"""
    c, o = on(name, 12)
    oq = oracle_mod.Oracle(12, L - 1, o.moduli[:L - 1])
    t = 65537
    rng = np.random.default_rng(9)
    s = o.keygen_secret(71)
    sq = np.ascontiguousarray(s[:L - 1])
    m1 = rng.integers(0, t, o.N).astype(np.uint64)
    m2 = np.zeros(o.N, dtype=np.uint64)
    m2[2] = 5                                           # 5 X^2: a negacyclic shift by two, scaled by 5
    c1, c2 = oq.encrypt(72, t, sq, m1), oq.encrypt(73, t, sq, m2)
    out = torch.zeros((1, 2, L - 1, o.N), dtype=torch.int64, device="cuda")
    c.ct_mul_relin_hybrid(dev(c1[None]), dev(c2[None]), dev(o.keygen_relin_hybrid(74, t, s)), out, 1, t)
    want = np.empty_like(m1)
    want[2:] = (5 * m1[:-2]) % t
    want[:2] = (t - (5 * m1[-2:]) % t) % t
    assert np.array_equal(oq.decrypt(sq, host(out).reshape(2, L - 1, o.N).copy(), t), want)


SWITCHES = [("DPFHE_NTT_CFG", "1", 13), ("DPFHE_NTT_CFG", "2", 13), ("DPFHE_NTT_CFG", "3", 13), ("DPFHE_NTT_CFG", "1", 14),
            ("DPFHE_ROT_CFG", "1", 13), ("DPFHE_ROT_CFG", "2", 13), ("DPFHE_KS_PF", "2", 13), ("DPFHE_KS_OCC", "1", 13),
            ("DPFHE_KS_PROF", "1", 13)]


@pytest.mark.parametrize("basis", ["default", "gen_mixed"])
@pytest.mark.parametrize("var,value,log_n", SWITCHES)
def test_tuning_switch(dp, oracle_mod, catalogue, monkeypatch, var, value, log_n, basis):
    """each runtime tuning switch selects another kernel instance; every one must reproduce the oracle for what it selects"""
    mods = None if basis == "default" else catalogue[basis]
    monkeypatch.setenv(var, value)
    c = dp.Context(log_n, L, mods)
    monkeypatch.delenv(var)
    o = oracle_mod.Oracle(log_n, L, mods)
    assert c.moduli == o.moduli
    if var == "DPFHE_NTT_CFG":
        x = edge_polys(o, 5, 0xBA5E0003)
        d = dev(x)
        c.ntt_fwd(d, 5)
        assert np.array_equal(host(d).reshape(x.shape), o.ntt_fwd(x))
        c.ntt_inv(d, 5)
        assert np.array_equal(host(d).reshape(x.shape), x)
    elif var == "DPFHE_ROT_CFG":
        batch = 5                                       # odd: a ciphertext without a partner in the two-per-item layout
        ct = edge_polys(o, 2 * batch, 92).reshape(batch, 2, L, o.N)
        ct[1, 1] = 0
        galois = [o.galois_elt(1), o.galois_elt(-5), conj(o)]
        keys = [o.fill_uniform(110 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))]
        out = torch.full((len(galois), batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
        c.rotate_hoisted(dev(ct), galois, [dev(k) for k in keys], out, batch)
        for r, g in enumerate(galois):
            assert np.array_equal(host(out[r]).reshape(ct.shape), o.rotate(ct, g, keys[r])), r
    else:
        occ = var == "DPFHE_KS_OCC"
        batch = rounds_batch(1) if occ else 9
        a = o.fill_uniform(121, 2 * batch).reshape(batch, 2, L, o.N)
        b = o.fill_uniform(122, 2 * batch).reshape(batch, 2, L, o.N)
        key = o.fill_uniform(123, 2 * L).reshape(L, 2, L, o.N)
        out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
        c.ct_mul_relin(dev(a), dev(b), dev(key), out, batch)
        assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin(a, b, key))
        if var == "DPFHE_KS_PROF":
            assert c.phase_cycles().any()               # the profiling instance of the kernel ran
        if occ:                                         # the other persistent kernels under the same cap
            ha, hkey = hybrid_inputs(o, batch, 124)
            hout = torch.full(ha.shape, -1, dtype=torch.int64, device="cuda")
            c.ct_mul_relin_hybrid(dev(ha), dev(ha), dev(hkey), hout, batch, 65537)
            assert np.array_equal(host(hout).reshape(ha.shape), o.ct_mul_relin_hybrid(ha, ha, hkey, 65537))
            ga, gkey = grouped_inputs(o, K, batch, 126)
            gout = torch.full(ga.shape, -1, dtype=torch.int64, device="cuda")
            c.ct_mul_relin_grouped(K, dev(ga), dev(ga), dev(gkey), gout, batch, 65537)
            assert np.array_equal(host(gout).reshape(ga.shape), o.ct_mul_relin_grouped(K, ga, ga, gkey, 65537))
    c.close()
