"""CPU tests of the product's host logic: parameter derivation in libdpfhe.so's host code, the kernel
bodies run through the host emulator (index algebra, swizzle, twiddle layout, digit exchange order,
lazy-reduction bounds) against the oracle, and the C-ABI export list."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("log_n,L", [(12, 1), (12, 3), (13, 4), (14, 2)])
def test_host_params_match_oracle(make_emu, oracle_mod, log_n, L):
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    assert e.moduli == o.moduli and e.psi == o.psi
    for l in range(L):
        assert np.array_equal(e.root_powers(l), o.root_powers(l))
        assert np.array_equal(e.root_powers(l, inverse=True), o.inv_root_powers(l))


def test_canon_shortcut_threshold(make_emu, oracle_mod):
    """the forward transform's store loop canonicalises with ONE conditional subtraction when floor(2^64/q) == 16 (canon_near60:
    k = x >> 60 is then at most one short): moduli on either side of 2^64/17, the largest modulus the context accepts, every
    multiple of q +- 1 and the top of the 64-bit range"""
    lib = oracle_mod.lib()
    two_n = 2 << 12
    thr = 2**64 // 17
    above = thr - thr % two_n + two_n + 1
    while not lib.dpo_is_prime(above):
        above += two_n
    below = thr - thr % two_n + 1
    while not lib.dpo_is_prime(below):
        below -= two_n
    top = oracle_mod.Oracle(12, 1).moduli[0]
    assert 2**64 // above == 16 and 2**64 // below == 17 and 2**64 // top == 16
    e = make_emu(12, 3, [above, below, top], variant="gen")
    for l, q in enumerate(e.moduli):
        xs = {0, q - 1, 2**64 - 1, 2**64 - 2, 2**63, 2**60 - 1, 2**60, 2**60 + 1}
        for m in range(1, 2**64 // q + 1):
            xs.update(v for v in (m * q - 1, m * q, m * q + 1, m * 2**60 - 1, m * 2**60) if 0 <= v < 2**64)
        for x in xs:
            assert e.scalar("canon_store", l, x) == x % q, (q, x)      # takes ANY 64-bit value
            if x < 16 * q:                                               # the documented domain of canon
                assert e.scalar("canon", l, x) == x % q, (q, x)
    o = oracle_mod.Oracle(12, 3, [above, below, top])                    # and the transform itself on such a basis
    x = o.fill_uniform(9, 2)
    assert np.array_equal(e.ntt(x), o.ntt_fwd(x))


@pytest.mark.parametrize("variant,moduli", [pytest.param("gen", "60_35_bit", id="gen"), pytest.param("fast", "default", id="fast"),
                                            pytest.param("gen", "smallest", id="gen-smallest"),
                                            pytest.param("fast", "fast_mixed", id="fast-fast_mixed")])
def test_device_scalar_arithmetic_bounds(make_emu, oracle_mod, variant, moduli):
    """modarith.cuh on adversarial inputs: every lazy routine stays inside its documented range (SB = 4: the quotient
    estimates of the Shoup and Barrett products may be up to two short).  Both arithmetic variants: the generic one on a
    60-bit and a 35-bit modulus and on the smallest modulus the context accepts (34 bits: bar_shift = 32), the k * 2^32 + 1
    one on the two largest moduli of the default basis and on the fast_mixed basis of tests/bases.py (37 to 55 bits)."""
    import bases
    lib = oracle_mod.lib()
    small = (1 << 34) - (1 << 34) % (2 << 12) + 1
    while not lib.dpo_is_prime(small):
        small += 2 << 12
    defaults = oracle_mod.Oracle(12, 2).moduli
    assert all(q & 0xFFFFFFFF == 1 for q in defaults)
    mods = {"60_35_bit": [defaults[0] - 0, small], "default": defaults, "smallest": [bases.SMALLEST_GENERIC],
            "fast_mixed": bases.catalogue(oracle_mod)["fast_mixed"]}[moduli]
    e = make_emu(12, len(mods), mods, variant=variant)
    SB = 4
    rng = np.random.default_rng(2)
    for l, q in enumerate(e.moduli):
        xs = [0, 1, q - 1, q, 2 * q, 3 * q - 1, 2**64 - 1, 2**63, 16 * q - 1 if 16 * q < 2**64 else 2**64 - 1]
        xs += [int(v) for v in rng.integers(0, 2**64, 2000, dtype=np.uint64)]
        for x in xs:
            r = e.scalar("word_reduce", l, x)
            assert r % q == x % q and r < 3 * q
            if x < 16 * q:
                assert e.scalar("canon", l, x) == x % q
        vals = [0, 1, q - 1, q - 2] + [int(v) for v in rng.integers(0, q, 1500, dtype=np.uint64)]
        for a, b in zip(vals, reversed(vals)):
            assert e.scalar("mulmod", l, a, b) == (a * b) % q
            r = e.scalar("mulmod_lazy", l, a, b)
            assert r % q == (a * b) % q and r < SB * q
        # Shoup products accept ANY 64-bit multiplicand: the lazy form lands below SB*q, the exact one below 2q
        for x, w in zip(xs[:600], vals[:600]):
            r = e.scalar("shoup_lazy", l, x, w)
            assert r % q == (x * w) % q and r < SB * q
            r = e.scalar("shoup_exact", l, x, w)
            assert r % q == (x * w) % q and r < 2 * q
        for x in (2**64 - 1, 16 * q - 1 if 16 * q < 2**64 else 2**64 - 1, 2**32 - 1, 2**32, (2**32 - 1) << 32):
            for w in (q - 1, 1, 0, q // 2, (q - 1) & ~0xFFFFFFFF, 0xFFFFFFFF):
                r = e.scalar("shoup_lazy", l, x, w)
                assert r % q == (x * w) % q and r < SB * q
        # sums of up to 16 products (the plaintext inner products): z < 16 q^2 -> [0, 15q), and the split-operand fold -> [0, 3q)
        zs = [0, 16 * (q - 1) ** 2, (q - 1) ** 2, 2**64 - 1, 2**64] + [int(a) * int(b) * k for a, b, k in zip(vals[:200], vals[200:400], range(1, 201)) if k <= 16]
        for z in zs:
            r = e.scalar("barrett_long", l, z >> 64, z & (2**64 - 1))
            assert r % q == z % q and r < 15 * q
        m30 = (1 << 30) - 1
        for n_terms in (1, 7, 16):
            pairs = [(q - 1, q - 1)] * n_terms if n_terms != 7 else [(int(a), int(b)) for a, b in zip(vals[:7], vals[7:14])]
            a0 = sum((x & m30) * (y & m30) for x, y in pairs)
            a1a = sum((x & m30) * (y >> 30) for x, y in pairs)
            a1b = sum((x >> 30) * (y & m30) for x, y in pairs)
            a2 = sum((x >> 30) * (y >> 30) for x, y in pairs)
            assert max(a0, a1a, a1b, a2) < 2**64
            r = e.scalar("pti_fold", l, a0, a1a, a1b, a2)
            assert r % q == sum(x * y for x, y in pairs) % q and r < 3 * q
        # lazy operands (factor bounds multiplying to at most 4): below (SB + 1) q
        for a in (3 * q - 1, 2 * q + 5, q):
            for b in (q - 1, 1, q // 3):
                r = e.scalar("mulmod_lazy", l, a, b)
                assert r % q == (a * b) % q and r < (SB + 1) * q


@pytest.mark.parametrize("log_n,L,n_polys", [(12, 1, 1), (12, 3, 2), (13, 4, 2), (14, 2, 1)])
def test_emulated_ntt_bodies(make_emu, oracle_mod, log_n, L, n_polys):
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    x = o.fill_uniform(0xD3390001, n_polys)
    q = np.array(o.moduli, dtype=np.uint64)
    x[0, :, : o.N // 2] = (q - 1)[:, None]          # worst case for the lazy bounds
    y = e.ntt(x)
    assert np.array_equal(y, o.ntt_fwd(x))
    assert np.array_equal(e.ntt(y, inverse=True), x)
    if log_n == 14:   # the CTA-pair form (half a limb per CTA, the inverse reading the partner's half)
        assert np.array_equal(e.ntt_pair(x), y)
        assert np.array_equal(e.ntt_pair(y, inverse=True), x)


@pytest.mark.parametrize("log_n,L,batch,G", [(12, 2, 3, 2), (12, 3, 4, 9), (13, 4, 2, 8), (12, 1, 2, 1), (14, 2, 2, 4), (12, 9, 2, 9)])
def test_emulated_fused_keyswitch_bodies(make_emu, oracle_mod, log_n, L, batch, G):
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    s = o.keygen_secret(1)
    evk = o.keygen_relin(2, 65537, s)
    a = o.fill_uniform(3, 2 * batch).reshape(batch, 2, L, o.N)
    b = o.fill_uniform(4, 2 * batch).reshape(batch, 2, L, o.N)
    q = np.array(o.moduli, dtype=np.uint64)
    a[0] = (q - 1)[None, :, None]
    b[0] = (q - 1)[None, :, None]
    assert np.array_equal(e.ks(0, a, b, evk, batch, G=G), o.ct_mul_relin(a, b, evk))
    d = o.fill_uniform(5, batch)
    ref = np.stack([np.stack(o.keyswitch(d[k], evk)) for k in range(batch)])
    assert np.array_equal(e.ks(1, d, None, evk, batch, G=G), ref)
    g = o.galois_elt(-2)
    gk = o.keygen_galois(6, 65537, s, g)
    assert np.array_equal(e.ks(2, a, None, gk, batch, galois=g, G=G), o.rotate(a, g, gk))


@pytest.mark.parametrize("log_n,L,t", [(12, 3, 65537), (12, 2, 0), (13, 4, 167772161), (14, 2, 65537)])
def test_emulated_mod_switch_bodies(make_emu, oracle_mod, log_n, L, t):
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    x = o.fill_uniform(9, 3)
    q = np.array(o.moduli, dtype=np.uint64)
    x[0] = (q - 1)[:, None]
    x[1, -1] = 0
    assert np.array_equal(e.mod_switch(x, t), o.mod_switch_down(x, t))


@pytest.mark.parametrize("log_n,L,nb,ng,batch,gmax", [(12, 2, 5, 3, 2, 0), (12, 1, 33, 10, 1, 4), (13, 2, 16, 9, 1, 8)])
def test_emulated_plain_inner_products(make_emu, oracle_mod, log_n, L, nb, ng, batch, gmax):
    """BSGS inner loop: split-operand accumulation, flush every 16 products, ragged giant-step blocks, edge residues"""
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    steps = o.fill_uniform(41, nb * batch * 2).reshape(nb, batch, 2, L, o.N)
    pts = o.fill_uniform(42, ng * nb).reshape(ng, nb, L, o.N)
    q = np.array(o.moduli, dtype=np.uint64)
    steps[:, 0, 0] = (q - 1)[:, None]      # worst case for the 64-bit accumulators: every product (q-1)^2
    pts[0] = (q - 1)[:, None]
    pts[-1, :, :, ::3] = 0
    assert np.array_equal(e.pt_inner(steps, pts, gmax), o.ct_mul_plain_inner(steps, pts))


@pytest.mark.parametrize("log_n,L,batch,G", [(12, 1, 2, None), (12, 3, 4, 6), (13, 4, 3, None), (14, 2, 2, None), (12, 5, 3, None)])
def test_emulated_hoisted_rotations(make_emu, oracle_mod, log_n, L, batch, G):
    """rotations that share the digit transforms == independent rotations, bit for bit; zero digits take the fallback"""
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    ct = o.fill_uniform(61, 2 * batch).reshape(batch, 2, L, o.N)
    ct[1, 1] = 0                      # c1 = 0: every coefficient of every digit is zero
    if batch > 2:
        ct[2, 1, L - 1] = 0           # one zero digit
    ks = [1, -1, 5]
    galois = [o.galois_elt(k) for k in ks] + [2 * o.N - 1]    # plus the conjugation element
    keys = np.stack([o.fill_uniform(70 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))])
    got, flagged = e.rotate_hoisted(ct, galois, keys, G)
    assert flagged == (0 if L == 1 else (1 if batch <= 2 else 2))
    for r, g in enumerate(galois):
        assert np.array_equal(got[r], o.rotate(ct, g, keys[r])), "rotation %d" % r


def _hybrid_inputs(o, batch, seed):
    """[batch][2][L-1][N] uniform residues (with edge rows) under the first L-1 moduli, and a uniform hybrid key"""
    Lq = o.L - 1
    x = o.fill_uniform(seed, 2 * batch)[:, :Lq].reshape(batch, 2, Lq, o.N).copy()
    q = np.array(o.moduli[:Lq], dtype=np.uint64)
    x[0, 0] = (q - 1)[:, None]
    x[0, 1, :, ::2] = 0
    key = o.fill_uniform(seed + 1, 2 * Lq).reshape(Lq, 2, o.L, o.N)
    return x, key


@pytest.mark.parametrize("log_n,L,batch,t,G", [(12, 2, 2, 65537, None), (12, 4, 3, 65537, 10), (13, 5, 2, 0, None), (14, 3, 1, 65537, None),
                                               (12, 9, 2, 65537, None)])
def test_emulated_hybrid_keyswitch_bodies(make_emu, oracle_mod, log_n, L, batch, t, G):
    """special-prime key switching: the device bodies in the kernel's role order against the oracle, all three modes"""
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    a, key = _hybrid_inputs(o, batch, 21)
    b, _ = _hybrid_inputs(o, batch, 23)
    assert np.array_equal(e.ks_hybrid(0, a, b, key, batch, t_plain=t, G=G), o.ct_mul_relin_hybrid(a, b, key, t))
    g = o.galois_elt(3)
    assert np.array_equal(e.ks_hybrid(2, a, None, key, batch, galois=g, t_plain=t, G=G), o.rotate_hybrid(a, g, key, t))
    d = a[:, 1]
    got = e.ks_hybrid(1, d, None, key, batch, t_plain=t, G=G)
    for k in range(batch):
        c0, c1 = o.keyswitch_hybrid(d[k], key, t)
        assert np.array_equal(got[k, 0], c0) and np.array_equal(got[k, 1], c1)


@pytest.mark.parametrize("log_n,L,K,t", [(12, 4, 2, 65537), (13, 5, 3, 0), (14, 3, 2, 65537), (12, 6, 4, 65537), (12, 3, 1, 65537)])
def test_emulated_mod_down_special(make_emu, oracle_mod, log_n, L, K, t):
    """division by the product of the last K limbs (md_tau / md_limb kernel bodies); K = 1 is the one-limb modulus switch"""
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    x = o.fill_uniform(41, 3)
    x[0, :, ::3] = 0
    x[1] = (np.array(o.moduli, dtype=np.uint64) - 1)[:, None]
    got = e.mod_down_special(K, x, t)
    assert np.array_equal(got, o.mod_down_special(K, x, t))
    if K == 1:
        assert np.array_equal(got, e.mod_switch(x, t))


def _grouped_inputs(o, K, batch, seed):
    """[batch][2][L-K][N] uniform residues (with edge rows) under the first L-K moduli, and a uniform grouped key"""
    Lq = o.L - K
    x = o.fill_uniform(seed, 2 * batch)[:, :Lq].reshape(batch, 2, Lq, o.N).copy()
    q = np.array(o.moduli[:Lq], dtype=np.uint64)
    x[0, 0] = (q - 1)[:, None]
    x[0, 1, :, ::2] = 0
    dnum = o.grouped_digits(K)
    key = o.fill_uniform(seed + 1, 2 * dnum).reshape(dnum, 2, o.L, o.N)
    return x, key


@pytest.mark.parametrize("log_n,L,K,batch,t,G,variant", [(12, 6, 2, 3, 65537, 13, "fast"), (12, 5, 2, 2, 65537, None, "fast"), (13, 6, 2, 2, 0, None, "fast"),
                                                         (14, 4, 2, 1, 65537, None, "fast"), (12, 10, 3, 2, 65537, None, "fast"),
                                                         (12, 12, 4, 1, 0, None, "fast"), (12, 4, 1, 2, 65537, None, "fast"),
                                                         (12, 6, 2, 2, 65537, None, "gen")])
def test_emulated_grouped_keyswitch_bodies(make_emu, oracle_mod, log_n, L, K, batch, t, G, variant):
    """digits of K limbs and K special primes: the device bodies in the role order of ks_grouped_kernel against the oracle, all
    three modes (ragged last digit, three and four special primes, one special prime = the hybrid variant)"""
    e, o = make_emu(log_n, L, variant=variant), oracle_mod.Oracle(log_n, L)
    a, key = _grouped_inputs(o, K, batch, 31)
    b, _ = _grouped_inputs(o, K, batch, 33)
    assert np.array_equal(e.ks_grouped(K, 0, a, b, key, batch, t_plain=t, G=G), o.ct_mul_relin_grouped(K, a, b, key, t))
    g = o.galois_elt(3)
    assert np.array_equal(e.ks_grouped(K, 2, a, None, key, batch, galois=g, t_plain=t, G=G), o.rotate_grouped(K, a, g, key, t))
    d = a[:, 1]
    got = e.ks_grouped(K, 1, d, None, key, batch, t_plain=t, G=G)
    for k in range(batch):
        c0, c1 = o.keyswitch_grouped(K, d[k], key, t)
        assert np.array_equal(got[k, 0], c0) and np.array_equal(got[k, 1], c1)
    if K == 1:
        assert np.array_equal(e.ks_grouped(1, 0, a, b, key, batch, t_plain=t, G=G), e.ks_hybrid(0, a, b, key, batch, t_plain=t, G=G))


@pytest.mark.parametrize("log_n,L,K,batch,t", [(12, 6, 2, 3, 65537), (12, 5, 2, 2, 0), (13, 4, 1, 2, 65537), (14, 4, 2, 1, 65537), (12, 9, 3, 2, 65537)])
def test_emulated_hoisted_grouped_rotations(make_emu, oracle_mod, log_n, L, K, batch, t):
    """hoisting with grouped hybrid keys: hoistg bodies, rot_apply_grouped rows and the division by P against the oracle"""
    e, o = make_emu(log_n, L), oracle_mod.Oracle(log_n, L)
    ct, _ = _grouped_inputs(o, K, batch, 51)
    galois = [o.galois_elt(1), o.galois_elt(-2), 2 * o.N - 1]
    dnum = o.grouped_digits(K)
    keys = np.stack([o.fill_uniform(60 + r, 2 * dnum).reshape(dnum, 2, L, o.N) for r in range(len(galois))])
    assert np.array_equal(e.rotate_hoisted_grouped(K, ct, galois, keys, t), o.rotate_hoisted_grouped(K, ct, galois, keys, t))


@pytest.mark.parametrize("log_n,L", [(12, 3), (13, 4), (14, 2)])
def test_generic_variant_on_the_default_basis(make_emu, oracle_mod, log_n, L):
    """the generic kernels must also be right for k * 2^32 + 1 moduli (DPFHE_FORCE_GENERIC runs them on the default basis)"""
    e, o = make_emu(log_n, L, variant="gen"), oracle_mod.Oracle(log_n, L)
    assert e.moduli == o.moduli
    x = o.fill_uniform(31, 2)
    x[0] = (np.array(o.moduli, dtype=np.uint64) - 1)[:, None]
    y = e.ntt(x)
    assert np.array_equal(y, o.ntt_fwd(x)) and np.array_equal(e.ntt(y, inverse=True), x)
    s = o.keygen_secret(1)
    evk = o.keygen_relin(2, 65537, s)
    a = o.fill_uniform(3, 4).reshape(2, 2, L, o.N)
    b = o.fill_uniform(4, 4).reshape(2, 2, L, o.N)
    assert np.array_equal(e.ks(0, a, b, evk, 2, G=L), o.ct_mul_relin(a, b, evk))
    g = o.galois_elt(5)
    gk = o.keygen_galois(6, 65537, s, g)
    assert np.array_equal(e.ks(2, a, None, gk, 2, galois=g, G=2 * L), o.rotate(a, g, gk))
    if L >= 3:
        assert np.array_equal(e.mod_switch(x, 65537), o.mod_switch_down(x, 65537))


def test_emulated_mixed_size_moduli(make_emu, oracle_mod):
    lib = oracle_mod.lib()
    two_n = 2 << 12
    mods = []
    for start in ((1 << 59), (1 << 40), (1 << 34) + (1 << 33)):
        c = (start // two_n) * two_n + 1
        while not lib.dpo_is_prime(c):
            c -= two_n
        mods.append(c)
    e, o = make_emu(12, 3, mods), oracle_mod.Oracle(12, 3, mods)
    s = o.keygen_secret(1)
    evk = o.keygen_relin(2, 65537, s)
    a = o.fill_uniform(3, 4).reshape(2, 2, 3, o.N)
    b = o.fill_uniform(4, 4).reshape(2, 2, 3, o.N)
    assert np.array_equal(e.ks(0, a, b, evk, 2), o.ct_mul_relin(a, b, evk))


def test_abi_exports_every_declared_symbol():
    """libdpfhe.so loads (no GPU needed for that) and exports exactly what include/dpfhe.h declares."""
    import deeppowers_b200
    from deeppowers_b200 import _lib
    lib = deeppowers_b200.load_library()
    with open(os.path.join(ROOT, "include", "dpfhe.h")) as f:
        header = f.read()
    declared = set(re.findall(r"\b(dpfhe_[a-z0-9_]+)\s*\(", header))
    declared -= {"dpfhe_ctx", "dpfhe_params"}
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), "libdpfhe.so does not export %s" % name
    assert declared == set(_lib.SYMBOLS), "python binding and header disagree: %s" % (declared ^ set(_lib.SYMBOLS))
    assert lib.dpfhe_version().decode().startswith("dpfhe")


def test_no_cpu_fallback_without_gpu():
    import torch
    import deeppowers_b200 as dp
    if torch.cuda.is_available():
        pytest.skip("this check is for the GPU-less container")
    with pytest.raises(dp.DpfheError) as ei:
        dp.Context(13, 4)
    assert "no CPU fallback" in str(ei.value)


def test_product_never_touches_oracle():
    """the shipped path (deeppowers_b200/, include/) must not import, include or link anything under oracle/"""
    bad = []
    for base in ("deeppowers_b200", "include"):
        for dp_, _, files in os.walk(os.path.join(ROOT, base)):
            if "build" in dp_.split(os.sep) or "__pycache__" in dp_:
                continue
            for fn in files:
                if fn.endswith((".so", ".o", ".pyc")):
                    continue
                with open(os.path.join(dp_, fn), errors="ignore") as f:
                    txt = f.read()
                if re.search(r"(import\s+oracle|from\s+oracle|dpfhe_oracle|dpo_[a-z])", txt):
                    bad.append(os.path.join(dp_, fn))
    assert not bad, bad
