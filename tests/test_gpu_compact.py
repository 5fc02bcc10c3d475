"""Compact ciphertexts on the GPU (DESIGN.md section 2.24): compaction and decryption bit for bit against the restatement
(tests/compact_ref.py) at N = 4096, 8192 and 16384 on the default, gen_mixed and fast_mixed bases, at level 1, a middle level and the
top, with bits at both ends of its range, BGV and CKKS; the download over one and over several chunks, ordered after pending work on
its input; launch counts; argument checks that leave the output untouched; the scratch counted and trimmed; every call through the
guard-word harness.  What it means, with the library's keys and ciphertexts and tests/scheme_model.py: the BGV slots of a
multiply-and-rescale and of a polynomial evaluation at a level, exactly, the CKKS slots of a multiply-and-rescale within the derived
bound, and the measured phase against its bound (both printed)."""
import math

import numpy as np
import pytest

import bases
import compact_ref as cr
import scheme_model as sm
from ckks_polyeval_ref import ckks_chain

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(9, 41))
T = 65537


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


def _ciphertexts(o, level, n, seed):
    """n canonical level-`level` ciphertexts [n][2][level][N] (any residues: compaction is bit-exact on every input)"""
    return np.ascontiguousarray(o.fill_uniform(seed, 2 * n).reshape(n, 2, o.L, o.N)[:, :, :level])


def _launches(level, t):
    return 2 * level if t and level >= 2 else 2


@pytest.mark.parametrize("logn,L,basis,t,level,bits,n", [
    (12, 4, None, T, 4, 18, 3), (12, 4, None, 0, 1, 2, 1), (12, 6, "gen_mixed", T, 3, "max", 2), (13, 5, None, 0, 5, "max", 2),
    (13, 6, "fast_mixed", T, 1, "max", 300), (13, 3, None, T, 2, 32, 2), (13, 4, None, 3, 2, 3, 1), (14, 3, None, T, 2, "max", 1),
    (14, 6, "gen_mixed", 0, 3, 2, 2), (14, 4, "fast_mixed", T, 4, 18, 1), (14, 5, None, T, 3, 33, 1)])
def test_compaction_and_decryption_bit_exact(oracle_mod, logn, L, basis, t, level, bits, n):
    """n = 300 at N = 8192 spans several waves of the element-wise grid (checked on its first, a middle and its last ciphertext)"""
    ctx, o = _setup(oracle_mod, logn, L, basis)
    if bits == "max":
        bits = cr.max_bits(logn, o.moduli[0])
    ct = _ciphertexts(o, level, n, 5 + level)
    W = ctx.compact_words(bits)
    assert W == o.N * bits // 32
    out = empty(n, W)
    n_launch = ctx.launch_count()
    ctx.compact_ciphertexts(level, bits, t, dev(ct), out, n)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == _launches(level, t)
    got = host(out).reshape(n, 2, W // 2)
    idx = list(range(n)) if n < 8 else [0, n // 2, n - 1]
    want = cr.compact(oracle_mod, o, level, bits, t, ct[idx])
    assert np.array_equal(got[idx], want)
    sk = empty(L, o.N)
    ctx.generate_secret(SEED, sk)
    pt = empty(n, 1, o.N)
    n_launch = ctx.launch_count()
    ctx.decrypt_compact(bits, t, sk, out, pt, n)
    torch.cuda.synchronize()
    assert ctx.launch_count() - n_launch == 6
    assert np.array_equal(host(pt)[idx], cr.decrypt(o, bits, t, host(sk).reshape(L, o.N), got[idx]))
    hp = np.zeros((n, 1, o.N), dtype=np.uint64)
    ctx.decrypt_compact_host(bits, t, host(sk).copy(), got.copy(), hp)
    assert np.array_equal(hp, host(pt))
    ctx.close()


def test_download_over_several_chunks_waits_for_its_input(oracle_mod):
    """600 ciphertexts of 384 KiB (N = 8192, level 3) are four chunks of the pipeline (170 per 64 MiB): the download equals the device
    compaction, writes nothing around its host output, counts one compaction per chunk, and reads its input after the work queued
    before it on the legacy default stream; a batch of one is one chunk"""
    L, n, level, bits = 4, 600, 3, 33
    ctx, o = _setup(oracle_mod, 13, L)
    ct = dev(_ciphertexts(o, level, n, 9))
    want = empty(n, ctx.compact_words(bits))
    ctx.compact_ciphertexts(level, bits, T, ct, want, n)
    src = torch.zeros_like(ct)
    torch.cuda.synchronize()
    g = 4096
    arena = np.random.default_rng(1).integers(0, 1 << 63, size=n * ctx.compact_words(bits) + 2 * g, dtype=np.uint64)
    before = arena.copy()
    hout = arena[g:g + n * ctx.compact_words(bits)]
    for _ in range(16):            # pending writes of the input on the legacy default stream when the download starts
        src.add_(1)
    src.copy_(ct)
    n_launch = ctx.launch_count()
    ctx.download_compact_ciphertexts(level, bits, T, src, hout, n)
    assert ctx.launch_count() - n_launch == 4 * _launches(level, T)
    assert np.array_equal(hout, host(want).reshape(-1))
    assert np.array_equal(arena[:g], before[:g]) and np.array_equal(arena[-g:], before[-g:])
    one = np.zeros(ctx.compact_words(bits), dtype=np.uint64)
    ctx.download_compact_ciphertexts(level, bits, T, ct[n - 1:], one, 1)
    assert np.array_equal(one, host(want)[n - 1])
    ctx.close()


def test_scratch_is_counted_and_trimmed(oracle_mod):
    ctx, o = _setup(oracle_mod, 12, 3)
    base = ctx.device_bytes()
    ct = dev(_ciphertexts(o, 3, 4, 2))
    out = empty(4, ctx.compact_words(20))
    ctx.compact_ciphertexts(3, 20, T, ct, out, 4)
    torch.cuda.synchronize()
    assert ctx.device_bytes() >= base + 4 * 2 * 2 * o.N * 8     # the two buffers of the chain, at least
    ctx._chk(ctx._l.dpfhe_context_trim(ctx._h))
    assert ctx.device_bytes() == base
    ctx.close()


def test_argument_checks_leave_the_output_untouched(oracle_mod):
    import deeppowers_b200 as dp
    L = 4
    ctx, o = _setup(oracle_mod, 12, L)
    q0 = o.moduli[0]
    big = cr.max_bits(12, q0) + 1
    ct = dev(_ciphertexts(o, L, 2, 3))
    out = torch.full((2, ctx.compact_words(32)), 7, dtype=torch.int64, device="cuda")
    sk = empty(L, o.N)
    ctx.generate_secret(SEED, sk)
    pt = torch.full((2, 1, o.N), 7, dtype=torch.int64, device="cuda")
    hout = np.full(2 * ctx.compact_words(32), 7, dtype=np.uint64)
    hpt = np.full((2, 1, o.N), 7, dtype=np.uint64)
    torch.cuda.synchronize()
    n_launch = ctx.launch_count()
    bad = [
        lambda: ctx.compact_ciphertexts(0, 32, T, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L + 1, 32, T, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, 1, 0, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, -1, 0, ct, out, 2),           # 2^32 - 1 in the C ABI: bits + log_n would wrap
        lambda: ctx.compact_ciphertexts(L, (1 << 32) - 12, T, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, 64 - 12, 0, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, big, 0, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, 32, T + 1, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, 32, 1, ct, out, 2),
        lambda: ctx.compact_ciphertexts(L, 17, T, ct, out, 2),            # t must be below 2^(bits-1)
        lambda: ctx.compact_ciphertexts(L, 32, T, 0, out, 2),
        lambda: ctx.compact_ciphertexts(L, 32, T, ct, int(out.data_ptr()) + 8, 2),
        lambda: ctx.compact_ciphertexts(L, 32, T, ct, ct, 2),
        lambda: ctx.download_compact_ciphertexts(L, 32, T + 1, ct, hout, 2),
        lambda: ctx.download_compact_ciphertexts(0, 32, T, ct, hout, 2),
        lambda: ctx.decrypt_compact(big, 0, sk, out, pt, 2),
        lambda: ctx.decrypt_compact(-1, 0, sk, out, pt, 2),
        lambda: ctx.download_compact_ciphertexts(L, (1 << 32) - 1, T, ct, hout, 2),
        lambda: ctx.decrypt_compact_host((1 << 32) - 5, 0, host(sk).copy(), hout, hpt),
        lambda: ctx.decrypt_compact(32, 4, sk, out, pt, 2),
        lambda: ctx.decrypt_compact(32, T, sk, out, out, 2),
        lambda: ctx.decrypt_compact(32, T, sk, out, sk, 2),
        lambda: ctx.decrypt_compact(32, T, 0, out, pt, 2),
        lambda: ctx.decrypt_compact_host(1, T, host(sk).copy(), hout, hpt),
    ]
    for call in bad:
        with pytest.raises(dp.DpfheError):
            call()
    torch.cuda.synchronize()
    assert ctx.launch_count() == n_launch
    assert bool((out == 7).all()) and bool((pt == 7).all()) and np.all(hout == 7) and np.all(hpt == 7)
    ctx.close()


@pytest.mark.parametrize("shape", ["N4096-L3-b3", "N8192-L6-K2-l3", "N16384-L4-l2"])
def test_guard_words_of_every_call(oracle_mod, shape):
    """every call of dpfhe_compact.h through the memory-contract harness: outputs equal to the restatement, guard words and operands
    unchanged, outputs pre-filled with ones and with random words"""
    import deeppowers_b200 as dp
    import compact_contract as ccn
    from memory_contract import Shape
    from test_gpu_memory_contract import Refs, run_case
    s = {"N4096-L3-b3": Shape(12, 3, 0, 3), "N8192-L6-K2-l3": Shape(13, 6, 2, 2, level=3), "N16384-L4-l2": Shape(14, 4, 0, 1, level=2)}[shape]
    c = dp.Context(s.log_n, s.L)
    R = Refs(oracle_mod, s.log_n, s.L)
    try:
        for fn, row in sorted(ccn.build_rows().items()):
            run_case(row, c, R, s, 17)
    finally:
        torch.cuda.synchronize()
        c.close()


# ---- what it means: the library's keys and ciphertexts, decrypted through the scheme model ----------------------------------------

class Net:
    """a top-level context of Lq ciphertext moduli and K special primes, its secret and grouped relinearisation key"""

    def __init__(self, oracle_mod, log_n, moduli, K, t):
        import deeppowers_b200 as dp
        self.ctx = dp.Context(log_n, len(moduli), moduli)
        self.moduli, self.N, self.K, self.t = self.ctx.moduli, 1 << log_n, K, t
        self.o = oracle_mod.Oracle(log_n, len(moduli), self.moduli)
        self.model = sm.Model(oracle_mod, log_n, self.moduli)
        self.sk = empty(len(moduli), self.N)
        self.ctx.generate_secret(SEED, self.sk)
        self.evk = empty(self.ctx.key_digits(K), 2, len(moduli), self.N)
        self.ctx.generate_relin_key(K, t, self.sk, SEED, self.evk)
        self.index = 0

    def enc_bgv(self, ell, z):
        pt, ct = empty(1, ell, self.N), empty(1, 2, ell, self.N)
        self.ctx.bgv_encode_level(ell, dev(np.asarray(z, dtype=np.int64).reshape(1, 2, self.N // 2)), pt, 1, self.t)
        self.ctx.encrypt_level(ell, self.t, self.sk, SEED, self.index, pt, ct, 1)
        self.index += 1
        return ct

    def enc_ckks(self, ell, z, scale):
        pt, ct = empty(1, ell, self.N), empty(1, 2, ell, self.N)
        self.ctx.ckks_encode_level(ell, torch.from_numpy(np.ascontiguousarray(z).reshape(1, -1)).cuda(), pt, 1, scale)
        self.ctx.encrypt_level(ell, 0, self.sk, SEED, self.index, pt, ct, 1)
        self.index += 1
        return ct

    def phase1(self, ct):
        """the centred level-1 phase of ct [1][2][ell][N] after the modulus switches of the compaction (BGV) or limb 0 (CKKS)"""
        ell = ct.shape[2]
        x = ct.reshape(2, ell, self.N)
        while x.shape[1] > 1 and self.t:
            y = empty(2, x.shape[1] - 1, self.N)
            self.ctx.mod_switch_down_level(x.shape[1], x.contiguous(), y, 2, self.t)
            x = y
        X, _ = self.model.phase(host(self.sk), host(x[:, :1].contiguous()).reshape(2, 1, self.N))
        return X

    def compact_bgv(self, ct, bits, phase1_max):
        """(decoded level-1 slots [2][N/2], |phi| measured, its bound) of ct [1][2][ell][N] compacted at bits; phase1_max: the largest
        |phase_1| of ct"""
        ell = ct.shape[2]
        out, pt, slots = empty(1, self.ctx.compact_words(bits)), empty(1, 1, self.N), empty(1, 2, self.N // 2)
        self.ctx.compact_ciphertexts(ell, bits, self.t, ct, out, 1)
        self.ctx.decrypt_compact(bits, self.t, self.sk, out, pt, 1)
        self.ctx.bgv_decode_level(1, pt, slots, 1, self.t)
        phi = cr.phase(self.o, bits, host(self.sk).reshape(-1, self.N), host(out).reshape(1, 2, -1))
        bound = (1 << bits) * phase1_max / self.moduli[0] + (self.N + 1) * (self.t / 2 + 1)
        return host(slots)[0], int(np.abs(phi).max()), bound

    def close(self):
        self.ctx.close()


def _check_bgv(net, ct, what):
    """the compact slots are the model's slots of ct times (q_1 .. q_{ell-1})^-1 mod t (the switches down to q0), exactly, from the
    smallest bits whose phase bound is below 2^(bits-1); below it, the smallest bits that still decrypted is printed"""
    ell, t = ct.shape[2], net.t
    want, v, Q = net.model.bgv(host(net.sk), host(ct).reshape(2, ell, net.N), t)
    f = pow(sm.prod(net.moduli[1:ell]), -1, t) if ell > 1 else 1
    want = np.asarray(sm.bgv_scale(want, f, t)).astype(np.uint64)
    p1 = max(abs(x) for x in net.phase1(ct))
    smallest = None
    for bits in range(t.bit_length() + 1, cr.max_bits(int(math.log2(net.N)), net.moduli[0]) + 1):
        got, phi, bound = net.compact_bgv(ct, bits, p1)
        ok = np.array_equal(got, want)
        assert phi <= bound, (what, bits, phi, bound)
        if ok and smallest is None:
            smallest = bits
        if bound < 1 << (bits - 1):
            print("%s bits=%d: |phase_1| 2^%.1f, |phi| 2^%.1f, bound 2^%.1f < 2^%d; smallest bits that decrypted: %d (%d B per ciphertext "
                  "against %d at level %d)" % (what, bits, sm.bits(p1), sm.bits(phi), sm.bits(bound), bits - 1, smallest, net.N * smallest // 4,
                                                16 * ell * net.N, ell))
            assert ok, (what, bits)
            break
    else:
        raise AssertionError("%s: no bits has its bound below 2^(bits-1)" % what)


@pytest.mark.parametrize("log_n,Lq,K", [(12, 5, 2), (13, 6, 2), (14, 4, 1)])
def test_bgv_slots_after_a_product_and_a_polynomial(oracle_mod, log_n, Lq, K):
    """ct_mul_relin_rescale_grouped_level at level Lq - 1 and a PolyEval created at a level, then compaction at the level of the result"""
    moduli = oracle_mod.Oracle(log_n, Lq + K).moduli
    net = Net(oracle_mod, log_n, moduli, K, T)
    try:
        r = np.random.default_rng(log_n)
        zs = [r.integers(0, T, (2, net.N // 2), dtype=np.int64) for _ in range(3)]
        ell = Lq - 1
        x = [net.enc_bgv(ell, z) for z in zs[:2]]
        low = empty(1, 2, ell - 1, net.N)
        net.ctx.ct_mul_relin_rescale_grouped_level(K, ell, x[0], x[1], net.evk, low, 1, T)
        got, _, _ = net.model.bgv(host(net.sk), host(low).reshape(2, ell - 1, net.N), T)
        assert np.array_equal(got, sm.bgv_scale(sm.bgv_mul(zs[0], zs[1], T), pow(moduli[ell - 1], -1, T), T).astype(np.uint64))
        _check_bgv(net, low, "N=%d product at level %d" % (net.N, ell))
        import deeppowers_b200 as dp
        pe = dp.PolyEval(net.ctx, K, T, [3, 1, 2], host(net.evk).copy(), level=ell)
        xin = net.enc_bgv(ell, zs[2])
        out = empty(1, 2, pe.result_limbs, net.N)
        pe.apply(xin, out, 1)
        got, _, _ = net.model.bgv(host(net.sk), host(out).reshape(2, pe.result_limbs, net.N), T)
        zz = np.asarray(zs[2], dtype=object)
        assert np.array_equal(got, ((3 + zz + 2 * zz * zz) % T).astype(np.uint64))
        _check_bgv(net, out, "N=%d polynomial at level %d" % (net.N, ell))
        pe.close()
    finally:
        net.close()


@pytest.mark.parametrize("log_n,Lq,K", [(13, 5, 2), (14, 4, 1)])
def test_ckks_slots_after_a_product(oracle_mod, log_n, Lq, K):
    """CKKS on the rescaling chain: a multiply-and-rescale at level Lq - 1, compacted from level Lq - 2 (limb 0) and decoded at level 1;
    the slots are the model's within N ((q0 / 2^bits)(N + 1)/2 + 1/2) / scale and the decoder's slack"""
    delta = 2.0**40
    net = Net(oracle_mod, log_n, ckks_chain(oracle_mod, Lq, K), K, 0)
    try:
        r = np.random.default_rng(log_n)
        zs = [r.uniform(-1, 1, net.N // 2) + 1j * r.uniform(-1, 1, net.N // 2) for _ in range(2)]
        ell = Lq - 1
        x = [net.enc_ckks(ell, z, delta) for z in zs]
        low = empty(1, 2, ell - 1, net.N)
        net.ctx.ct_mul_relin_rescale_grouped_level(K, ell, x[0], x[1], net.evk, low, 1, 0)
        sc = delta * delta / net.moduli[ell - 1]
        model_slots, X, Q = net.model.ckks(host(net.sk), host(low).reshape(2, ell - 1, net.N), sc)
        q0 = net.moduli[0]
        assert max(abs(v) for v in X) < q0 // 2
        for bits in (40, cr.max_bits(log_n, q0)):
            out, pt = empty(1, net.ctx.compact_words(bits)), empty(1, 1, net.N)
            net.ctx.compact_ciphertexts(ell - 1, bits, 0, low, out, 1)
            net.ctx.decrypt_compact(bits, 0, net.sk, out, pt, 1)
            slots = torch.empty((1, net.N // 2), dtype=torch.complex128, device="cuda")
            net.ctx.ckks_decode_level(1, pt, slots, 1, sc)
            got = slots.cpu().numpy()[0]
            bound = net.N * (q0 / 2.0**bits * (net.N + 1) / 2 + 0.5) / sc + 2 * sm.ckks_decode_slack(net.N, 2)
            err = np.abs(got - model_slots).max()
            print("CKKS N=%d bits=%d: slot error against the model 2^%.1f, bound 2^%.1f; against the exact product 2^%.1f" %
                  (net.N, bits, sm.bits(err), sm.bits(bound), sm.bits(np.abs(got - zs[0] * zs[1]).max())))
            assert err <= bound
            phi = cr.phase(net.o, bits, host(net.sk).reshape(-1, net.N), host(out).reshape(1, 2, -1))
            pbound = (1 << bits) * max(abs(v) for v in net.phase1(low)) / q0 + (net.N + 1) / 2
            print("CKKS N=%d bits=%d: |phi| 2^%.1f, bound 2^%.1f" % (net.N, bits, sm.bits(int(np.abs(phi).max())), sm.bits(pbound)))
            assert np.abs(phi).max() <= pbound
    finally:
        net.close()


# ---- the networks of DESIGN.md section 2.22, their results compacted: the smallest bits that decrypts them -------------------------

def _phase1_max(c, model, sk, ct, t):
    """the largest |phase_1| of ct [B][2][l][N] after the switches of a compaction down to q0 (BGV) or of limb 0 (CKKS)"""
    B, ell, N = ct.shape[0], ct.shape[2], c.N
    x = ct.reshape(2 * B, ell, N).contiguous()
    while t and x.shape[1] > 1:
        y = empty(2 * B, x.shape[1] - 1, N)
        c.mod_switch_down_level(x.shape[1], x, y, 2 * B, t)
        x = y
    one = host(x[:, :1].contiguous()).reshape(B, 2, 1, N)
    return max(max(abs(v) for v in model.phase(host(sk), one[k])[0]) for k in range(B))


def _compact_sweep(c, o, model, sk, ct, t, accept, what):
    """compacts ct at every bits from the smallest t allows to the largest N 2^bits < q0 allows; accept(pt [B][1][N]) says whether the
    level-1 plaintexts decode correctly.  Prints, per bits, the measured |phi| and the bound against 2^(bits-1); returns the smallest bits
    that decoded and the smallest bits the bound guarantees (BGV)"""
    B, ell, N, q0 = ct.shape[0], ct.shape[2], c.N, int(c.moduli[0])
    p1 = _phase1_max(c, model, sk, ct, t)
    E = t / 2 + 1 if t else 0.5
    smallest = guaranteed = None
    for bits in range(max(2, t.bit_length() + 1), cr.max_bits(int(math.log2(N)), q0) + 1):
        out, pt = empty(B, c.compact_words(bits)), empty(B, 1, N)
        c.compact_ciphertexts(ell, bits, t, ct, out, B)
        c.decrypt_compact(bits, t, sk, out, pt, B)
        ok = accept(pt)
        phi = int(np.abs(cr.phase(o, bits, host(sk).reshape(-1, N), host(out).reshape(B, 2, -1))).max())
        bound = (1 << bits) * p1 / q0 + (N + 1) * E
        assert phi <= bound, (what, bits, phi, bound)
        if ok and smallest is None:
            smallest = bits
        if t and bound < 1 << (bits - 1):
            assert ok, (what, bits)
            guaranteed = guaranteed or bits
        print("%s bits=%d: %s, |phi| 2^%.1f (margin %.1f bits), bound 2^%.1f (margin %.1f bits)" %
              (what, bits, "decodes" if ok else "does not decode", sm.bits(phi), bits - 1 - sm.bits(phi), sm.bits(bound),
               bits - 1 - sm.bits(bound)))
    print("%s: |phase_1| 2^%.1f; the smallest bits that decoded: %s (%d B per ciphertext against %d at level %d); the smallest the bound "
          "guarantees: %s" % (what, sm.bits(p1), smallest, N * smallest // 4, 16 * ell * N, ell, guaranteed))
    return smallest, guaranteed


def test_smallest_bits_of_the_bgv_network(oracle_mod):
    """the BGV network of DESIGN.md section 2.22 (W1 -> + b1 -> p -> W2 + b2 -> p -> W3, N = 8192, Lq = 5, K = 2, t = 65537, one context
    and one key set) and its result compacted at every bits: from the bound's bits on, every slot decodes to the full-level result times
    (q_1 .. q_{l-1})^-1 mod t"""
    import deeppowers_b200 as dp
    from test_gpu_polyeval_level import _bsgs_periodic, _relin
    K, Lq, log_n, t, DIM, BABY, B = 2, 5, 13, 65537, 16, 4, 2
    coeffs = [3, -2, 1]
    L = Lq + K
    c = dp.Context(log_n, L)
    objs = [c]
    try:
        mods = [int(q) for q in c.moduli]
        o = oracle_mod.Oracle(log_n, L, mods)
        model = sm.Model(oracle_mod, log_n, mods)
        N, half = c.N, c.N // 2
        sk, evk = _relin(c, K, t)
        gk = empty(BABY, c.grouped_digits(K), 2, L, N)
        c.generate_galois_keys(K, t, sk, [c.galois_elt(s) for s in range(1, BABY + 1)], bytes(range(2, 34)), gk)
        hk = host(gk).reshape(gk.shape)
        kb, kg = np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1]
        rng = np.random.default_rng(51)
        W = [rng.integers(-8, 9, size=(DIM, DIM)) for _ in range(3)]
        x = rng.integers(-8, 9, size=(B, DIM))
        b1, b2 = rng.integers(-50, 51, size=DIM), rng.integers(-50, 51, size=DIM)
        i = np.arange(half)

        def periodic(v):
            s = np.zeros((v.shape[0], N), dtype=np.int64)
            s[:, :half] = v[:, i % DIM]
            return s

        def encode(slots, level):
            pt = empty(slots.shape[0], level, N)
            c.bgv_encode_level(level, torch.from_numpy(np.ascontiguousarray(slots)).cuda(), pt, slots.shape[0], t)
            return pt

        pe1 = dp.PolyEval(c, K, t, coeffs, evk)
        Lf1 = pe1.result_limbs
        pe2 = dp.PolyEval(c, K, t, coeffs, evk, level=Lf1)
        Lf2 = pe2.result_limbs
        layers = [dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[0], BABY, half), Lq)).reshape(DIM, Lq, N), BABY, kb, kg, t),
                  dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[1], BABY, half), Lf1)).reshape(DIM, Lf1, N), BABY, kb, kg, t,
                                         level=Lf1),
                  dp.LinearLayer.grouped(c, K, host(encode(_bsgs_periodic(W[2], BABY, half), Lf2)).reshape(DIM, Lf2, N), BABY, kb, kg, t,
                                         level=Lf2)]
        objs += [pe1, pe2] + layers
        ct = empty(B, 2, Lq, N)
        c.encrypt_level(Lq, t, sk, SEED, 0, encode(periodic(x), Lq), ct, B)
        y1 = torch.empty_like(ct)
        layers[0].apply(ct, y1, B)
        c.ct_add_plain_level(Lq, y1, encode(periodic(b1[None]), Lq)[0], y1, B)
        h1 = empty(B, 2, Lf1, N)
        pe1.apply(y1, h1, B)
        y2 = torch.empty_like(h1)
        layers[1].apply(h1, y2, B)
        c.ct_add_plain_level(Lf1, y2, encode(periodic(b2[None]), Lf1)[0], y2, B)
        h2 = empty(B, 2, Lf2, N)
        pe2.apply(y2, h2, B)
        y3 = torch.empty_like(h2)
        layers[2].apply(h2, y3, B)
        ph = empty(B, Lf2, N)
        c.decrypt_level(Lf2, sk, y3, 2, ph, B)
        full = empty(B, N)
        c.bgv_decode_level(Lf2, ph, full, B, t)

        def p(v):
            return sum(int(a) * v ** k for k, a in enumerate(coeffs)) % t

        act = np.vectorize(p, otypes=[object])
        ob = lambda a: a.astype(object)
        h = act((ob(x) @ ob(W[0]).T + ob(b1)) % t)
        h = act((h @ ob(W[1]).T + ob(b2)) % t)
        assert np.array_equal(host(full)[:, :DIM].astype(object), (h @ ob(W[2]).T) % t)
        f = pow(sm.prod(mods[1:Lf2]), -1, t)
        want = (host(full).astype(object) * f % t).astype(np.uint64)

        def accept(pt):
            slots = empty(B, N)
            c.bgv_decode_level(1, pt, slots, B, t)
            return np.array_equal(host(slots), want)

        smallest, guaranteed = _compact_sweep(c, o, model, sk, y3, t, accept, "BGV network of section 2.22, W3 h at %d limbs" % Lf2)
        assert smallest is not None and guaranteed is not None and smallest <= guaranteed
    finally:
        torch.cuda.synchronize()
        for obj in reversed(objs):
            obj.close()


def test_smallest_bits_of_the_ckks_chain(oracle_mod):
    """the CKKS chain of DESIGN.md section 2.22 (W1 -> rescale -> CkksPolyEval -> W2 -> rescale, N = 8192, Lq = 6, K = 2) and its result
    compacted at every bits: a bits decodes when the slots stay within the chain's own tolerance of the exact result"""
    import deeppowers_b200 as dp
    from ckks_polyeval_ref import ckks_chain as chain
    from test_gpu_polyeval_level import _relin
    K, Lq, log_n, DIM, BABY, B = 2, 6, 13, 16, 4, 2
    mods = chain(oracle_mod, Lq, K)
    c = dp.Context(log_n, Lq + K, mods)
    objs = [c]
    try:
        o = oracle_mod.Oracle(log_n, Lq + K, mods)
        model = sm.Model(oracle_mod, log_n, mods)
        N, half = c.N, c.N // 2
        sk, evk = _relin(c, K, 0)
        gk = empty(BABY, c.grouped_digits(K), 2, Lq + K, N)
        c.generate_galois_keys(K, 0, sk, [c.galois_elt(s) for s in range(1, BABY + 1)], bytes(range(2, 34)), gk)
        hk = host(gk).reshape(gk.shape)
        kb, kg = np.ascontiguousarray(hk[:BABY - 1]), hk[BABY - 1]
        rng = np.random.default_rng(43)
        W1, W2 = rng.uniform(-1, 1, (DIM, DIM)) / DIM, rng.uniform(-1, 1, (DIM, DIM)) / DIM
        xv = rng.uniform(-1, 1, (B, DIM))
        i = np.arange(half)
        scale = float(mods[1])

        def diags(W, level, wscale):
            d = np.zeros((DIM, half), dtype=np.complex128)
            for k in range(DIM):
                d[k, (i + (k // BABY) * BABY) % half] = W[i % DIM, (i % DIM + k) % DIM]
            pt = empty(DIM, level, N)
            c.ckks_encode_level(level, torch.from_numpy(d).cuda(), pt, DIM, wscale)
            return host(pt).reshape(DIM, level, N)

        z = np.zeros((B, half), dtype=np.complex128)
        z[:] = xv[:, i % DIM]
        pts = empty(B, Lq, N)
        c.ckks_encode_level(Lq, torch.from_numpy(z).cuda(), pts, B, scale)
        ct = empty(B, 2, Lq, N)
        c.encrypt_level(Lq, 0, sk, SEED, 0, pts, ct, B)
        w1scale = float(mods[Lq - 1])
        layer1 = dp.LinearLayer.grouped(c, K, diags(W1, Lq, w1scale), BABY, kb, kg, 0)
        objs.append(layer1)
        y = torch.empty_like(ct)
        layer1.apply(ct, y, B)
        l1 = Lq - 1
        r1 = empty(B, 2, l1, N)
        c.mod_switch_down_level(Lq, y, r1, 2 * B, 0)
        s1 = scale * w1scale / mods[Lq - 1]
        pe = dp.PolyEval.ckks(c, K, [0.5, 0.25, 0.125], s1, evk, level=l1)
        objs.append(pe)
        Lf = pe.result_limbs
        h = empty(B, 2, Lf, N)
        pe.apply(r1, h, B)
        w2scale = float(mods[Lf - 1])
        layer2 = dp.LinearLayer.grouped(c, K, diags(W2, Lf, w2scale), BABY, kb, kg, 0, level=Lf)
        objs.append(layer2)
        w = torch.empty_like(h)
        layer2.apply(h, w, B)
        r2 = empty(B, 2, Lf - 1, N)
        c.mod_switch_down_level(Lf, w, r2, 2 * B, 0)
        out_scale = pe.result_scale * w2scale / mods[Lf - 1]
        a = xv @ W1.T
        want = (0.5 + 0.25 * a + 0.125 * a ** 2) @ W2.T
        tol = DIM * DIM * 8.0 * (N / scale + N / w1scale + N / s1 + N / pe.result_scale + N / w2scale + N / out_scale)

        def accept(pt):
            out = torch.empty((B, half), dtype=torch.complex128, device="cuda")
            c.ckks_decode_level(1, pt, out, B, out_scale)
            return float(np.abs(out.cpu().numpy()[:, :DIM] - want).max()) < tol

        smallest, _ = _compact_sweep(c, o, model, sk, r2, 0, accept, "CKKS chain of section 2.22, result at %d limbs, scale 2^%.1f" %
                                     (Lf - 1, math.log2(out_scale)))
        assert smallest is not None
    finally:
        torch.cuda.synchronize()
        for obj in reversed(objs):
            obj.close()


def test_compact_example(tmp_path):
    """examples/encrypted_compact.cpp: the server runs a BGV product down the chain and writes compact results as wire kind 10, the
    client reads them, decrypts and decodes every slot"""
    import os
    import shutil
    import subprocess
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "deeppowers_b200")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "encrypted_compact")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), "-I", os.path.join(cuda, "include"),
                           os.path.join(root, "examples", "encrypted_compact.cpp"), "-L", libdir, "-ldpfhe", "-L", os.path.join(cuda, "lib64"),
                           "-lcudart", "-Wl,-rpath," + libdir + ":" + os.path.join(cuda, "lib64"), "-o", exe])
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ", 0 wrong" in r.stdout
