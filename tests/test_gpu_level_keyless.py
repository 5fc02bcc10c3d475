"""The keyless calls at level l on the top-level context (DESIGN.md section 2.22): encoding, decoding, encryption (secret and public key),
decryption, ct_add_plain, ct_mul_plain, ct_lincomb and mod_switch_down at every level 1 .. L, each bit for bit the call on a context over
the first l moduli.  Every call runs through its row of tests/memory_contract.py (guard words around every buffer, operands and keys
unchanged, outputs written without being read) against the oracle of the prefix basis, at N = 4096, 8192 and 16384 on the default basis
and on a generic one, and at level Lq = 5 of a context with two special primes; every output placed over any other buffer of its call
(by one 16-byte pair, at that buffer's start and end) is rejected with the arena untouched and no launch; the results are compared with
the call on a real prefix context, and level = L with the top-level call; the launch counts are the prefix context's; the argument
checks leave the output untouched and name the level; the host forms run several chunks."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import level_contract as lc  # noqa: E402
import memory_contract as mc  # noqa: E402
from memory_contract import Shape  # noqa: E402
from test_gpu_memory_contract import Arena, Refs, inputs, layout, run_case  # noqa: E402
from test_gpu_parity import dp  # noqa: E402,F401  (a fixture)

ROWS = lc.build_rows()

L = 4
KEYLESS = ["dpfhe_ckks_encode_level", "dpfhe_ckks_decode_level", "dpfhe_bgv_encode_level", "dpfhe_bgv_decode_level", "dpfhe_encrypt_level",
           "dpfhe_decrypt_level", "dpfhe_encrypt_public_level", "dpfhe_ct_add_plain_level", "dpfhe_ct_mul_plain_level", "dpfhe_ct_lincomb_level",
           "dpfhe_mod_switch_down_level"]
HOST = [fn + "_host" for fn in KEYLESS[:7]]


class BasisRefs(Refs):
    """Refs over the context's own moduli (a generic basis as well as the default one)"""

    def __init__(self, oracle_mod, log_n, moduli):
        self.oracle_mod, self.log_n = oracle_mod, log_n
        self.o = oracle_mod.Oracle(log_n, len(moduli), [int(q) for q in moduli])
        self._sub = {}


@pytest.fixture(scope="module")
def generic_moduli(oracle_mod):
    """the first L moduli of tests/bases.py's gen_mixed basis: none of the fast form k 2^32 + 1, so that every prefix runs the generic
    kernels, as a context over it would; 1 mod 2^15, so valid at every N"""
    from bases import catalogue
    return catalogue(oracle_mod)["gen_mixed"][:L]


@pytest.fixture
def make(dp, oracle_mod):
    made = []
    torch.cuda.empty_cache()

    def get(log_n, moduli=None, n_limbs=L):
        c = dp.Context(log_n, n_limbs, moduli)
        made.append(c)
        return c, BasisRefs(oracle_mod, log_n, c.moduli)

    yield get
    torch.cuda.synchronize()
    for c in made:
        c.close()
    torch.cuda.empty_cache()


def shape(fn, log_n, level, batch=2, **kw):
    return Shape(log_n, L, 0, batch, level=level, n_terms=3, n_comp=kw.pop("n_comp", 2), **kw)


def levels(fn):
    return range(2 if fn == "dpfhe_mod_switch_down_level" else 1, L + 1)


@pytest.mark.parametrize("basis", ["default", "generic"])
@pytest.mark.parametrize("log_n", [12, 13, 14])
@pytest.mark.parametrize("fn", KEYLESS)
def test_every_call_at_every_level(make, generic_moduli, fn, log_n, basis):
    c, R = make(log_n, generic_moduli if basis == "generic" else None)
    for lv in levels(fn):
        run_case(ROWS[fn], c, R, shape(fn, log_n, lv), 1000 + lv)


@pytest.mark.parametrize("n_comp", [2, 3])
def test_decrypt_three_components(make, n_comp):
    c, R = make(13)
    for lv in levels("dpfhe_decrypt_level"):
        run_case(ROWS["dpfhe_decrypt_level"], c, R, shape("dpfhe_decrypt_level", 13, lv, n_comp=n_comp), 1100 + lv)


@pytest.mark.parametrize("t", [0, mc.T])
def test_mod_switch_plain_modulus(make, t):
    """the BGV correction (t > 0) and plain rounding (t = 0, the CKKS rescale)"""
    c, R = make(13)
    for lv in levels("dpfhe_mod_switch_down_level"):
        run_case(ROWS["dpfhe_mod_switch_down_level"], c, R, shape("dpfhe_mod_switch_down_level", 13, lv, t=t), 1200 + lv)


@pytest.mark.parametrize("fn", HOST)
def test_host_forms_over_several_chunks(make, fn):
    """N = 4096 at level 4: a 64 MiB chunk holds 256 ciphertexts or 512 plaintexts of 4 limbs (abi.cu pick_chunk); 600 items run three
    chunks, the last one short, or two"""
    c, R = make(12)
    run_case(ROWS[fn], c, R, shape(fn, 12, L, batch=600), 1300)


def _rand(rng, mods, shape):
    out = np.empty(shape, dtype=np.uint64)
    for i, q in enumerate(mods):
        out[..., i, :] = rng.integers(0, int(q), size=out[..., i, :].shape, dtype=np.uint64)
    return torch.from_numpy(out.view(np.int64)).cuda()


@pytest.mark.parametrize("basis", ["default", "generic"])
@pytest.mark.parametrize("log_n", [12, 14])
def test_against_a_prefix_context(make, generic_moduli, log_n, basis):
    """each call at level l on the top context against the same call on a context over q_0 .. q_{l-1}: the same bits and the same
    launches; at l = L the level call is the top-level call"""
    c, _ = make(log_n, generic_moduli if basis == "generic" else None)
    N, mods, B, t = c.N, c.moduli, 3, mc.T
    rng = np.random.default_rng(7)
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    c.generate_secret(mc.SEED, sk)
    pk = torch.empty((2, L, N), dtype=torch.int64, device="cuda")
    c.public_keygen(t, sk, mc.SEED, pk)
    slots = torch.from_numpy(rng.integers(-1000, 1000, size=(B, N), dtype=np.int64)).cuda()
    zs = torch.from_numpy(rng.uniform(-1, 1, (B, N // 2)) + 1j * rng.uniform(-1, 1, (B, N // 2))).cuda()
    for lv in range(1, L + 1):
        low, _ = make(log_n, mods[:lv], lv)
        pt, ct, ct3 = _rand(rng, mods[:lv], (B, lv, N)), _rand(rng, mods[:lv], (B, 2, lv, N)), _rand(rng, mods[:lv], (B, 3, lv, N))
        pk_low = pk[:, :lv].contiguous()

        def both(name, level_call, low_call, out_shape, dtype=torch.int64):
            got, want = torch.full(out_shape, -1, dtype=dtype, device="cuda"), torch.full(out_shape, -1, dtype=dtype, device="cuda")
            n0, m0 = c.launch_count(), low.launch_count()
            level_call(got)
            low_call(want)
            torch.cuda.synchronize()
            assert torch.equal(got, want), (name, lv)
            assert c.launch_count() - n0 == low.launch_count() - m0, (name, lv)
            return got

        both("bgv_encode", lambda o: c.bgv_encode_level(lv, slots, o, B, t), lambda o: low.bgv_encode(slots, o, B, t), (B, lv, N))
        both("bgv_decode", lambda o: c.bgv_decode_level(lv, pt, o, B, t), lambda o: low.bgv_decode(pt, o, B, t), (B, N))
        both("ckks_encode", lambda o: c.ckks_encode_level(lv, zs, o, B, 2.0 ** 30), lambda o: low.ckks_encode(zs, o, B, 2.0 ** 30), (B, lv, N))
        both("ckks_decode", lambda o: c.ckks_decode_level(lv, pt, o, B, 2.0 ** 30), lambda o: low.ckks_decode(pt, o, B, 2.0 ** 30),
             (B, N // 2), torch.complex128)
        both("encrypt", lambda o: c.encrypt_level(lv, t, sk, mc.SEED, 5, pt, o, B),
             lambda o: low.encrypt(t, sk[:lv].contiguous(), mc.SEED, 5, pt, o, B), (B, 2, lv, N))
        both("encrypt_public", lambda o: c.encrypt_public_level(lv, t, pk, mc.SEED, 5, pt, o, B),
             lambda o: low.encrypt_public(t, pk_low, mc.SEED, 5, pt, o, B), (B, 2, lv, N))
        for n_comp, x in ((2, ct), (3, ct3)):
            both("decrypt", lambda o: c.decrypt_level(lv, sk, x, n_comp, o, B), lambda o: low.decrypt(sk[:lv].contiguous(), x, n_comp, o, B),
                 (B, lv, N))
        both("ct_add_plain", lambda o: c.ct_add_plain_level(lv, ct, pt[0], o, B), lambda o: low.ct_add_plain(ct, pt[0], o, B), (B, 2, lv, N))
        both("ct_mul_plain", lambda o: c.ct_mul_plain_level(lv, ct, pt[0], o, B), lambda o: low.ct_mul_plain(ct, pt[0], o, B), (B, 2, lv, N))
        both("ct_lincomb", lambda o: c.ct_lincomb_level(lv, [ct, ct3[:, :2].contiguous()], [3, -(1 << 61)], 9, o, B),
             lambda o: low.ct_lincomb([ct, ct3[:, :2].contiguous()], [3, -(1 << 61)], 9, o, B), (B, 2, lv, N))
        if lv >= 2:
            for tt in (0, mc.T):
                both("mod_switch_down", lambda o: c.mod_switch_down_level(lv, ct, o, 2 * B, tt), lambda o: low.mod_switch_down(ct, o, 2 * B, tt),
                     (B, 2, lv - 1, N))
        low.close()
    # level L is the call itself
    pt, ct = _rand(rng, mods, (B, L, N)), _rand(rng, mods, (B, 2, L, N))
    a, b = torch.empty((B, 2, L, N), dtype=torch.int64, device="cuda"), torch.empty((B, 2, L, N), dtype=torch.int64, device="cuda")
    c.encrypt_level(L, t, sk, mc.SEED, 9, pt, a, B)
    c.encrypt(t, sk, mc.SEED, 9, pt, b, B)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    a2, b2 = torch.empty((B, 2, L - 1, N), dtype=torch.int64, device="cuda"), torch.empty((B, 2, L - 1, N), dtype=torch.int64, device="cuda")
    c.mod_switch_down_level(L, ct, a2, 2 * B, mc.T)
    c.mod_switch_down(ct, b2, 2 * B, mc.T)
    torch.cuda.synchronize()
    assert torch.equal(a2, b2)


def test_argument_checks(make):
    """level 0, level L + 1 and mod_switch_down at level 1 are rejected, naming the level; overlaps are measured at the level's sizes;
    a rejected call leaves its output untouched and launches nothing"""
    c, _ = make(12)
    N, B = c.N, 2
    sk = torch.zeros((L, N), dtype=torch.int64, device="cuda")
    buf = torch.full((4, 2, L, N), 7, dtype=torch.int64, device="cuda")
    out = torch.full((B, 2, L, N), 7, dtype=torch.int64, device="cuda")
    pt = torch.zeros((B, L, N), dtype=torch.int64, device="cuda")
    calls = {
        "encrypt": lambda lv, o: c.encrypt_level(lv, mc.T, sk, mc.SEED, 0, pt, o, B),
        "decrypt": lambda lv, o: c.decrypt_level(lv, sk, buf, 2, o, B),
        "add_plain": lambda lv, o: c.ct_add_plain_level(lv, buf, pt[0], o, B),
        "mul_plain": lambda lv, o: c.ct_mul_plain_level(lv, buf, pt[0], o, B),
        "lincomb": lambda lv, o: c.ct_lincomb_level(lv, [buf], [1], 0, o, B),
        "mod_switch": lambda lv, o: c.mod_switch_down_level(lv, buf, o, 2 * B, 0),
        "bgv_encode": lambda lv, o: c.bgv_encode_level(lv, pt, o, B, mc.T),
    }
    for name, call in calls.items():
        for lv in (0, L + 1) + ((1,) if name == "mod_switch" else ()):
            before, n0 = out.clone(), c.launch_count()
            with pytest.raises(RuntimeError, match="level %d" % lv):
                call(lv, out)
            torch.cuda.synchronize()
            assert torch.equal(out, before) and c.launch_count() == n0, (name, lv)
    # the input [B][2][l][N] at the start of buf, the output B * 2 N words further on: over the input at level 2, clear of it at level 1
    flat = buf.view(-1)
    src, dst = flat[:B * 2 * 2 * N], flat[B * 2 * N:][:B * 2 * 2 * N]
    snap = flat.clone()
    with pytest.raises(RuntimeError, match="level 2: output must"):
        c.ct_mul_plain_level(2, src, pt[0, :2].contiguous(), dst, B)
    torch.cuda.synchronize()
    assert torch.equal(flat, snap)
    c.ct_mul_plain_level(1, src[:B * 2 * N], pt[0, :1].contiguous(), dst[:B * 2 * N], B)
    torch.cuda.synchronize()


# ---- at a level of a context with special primes: Lq = 5 of L = 7 --------------------------------------------------------------------

SPECIAL = Shape(12, 7, 2, 3, n_terms=3)   # the calls at lv = Lq = 5


@pytest.mark.parametrize("fn", sorted(ROWS))
def test_at_the_ciphertext_level_of_a_special_prime_context(make, oracle_mod, fn):
    """every row, keyless calls and host forms at lv = 5 of 7 limbs, the polynomial evaluators at level 3 of K = 2, Lq = 5"""
    s, moduli = SPECIAL, None
    if fn.startswith("dpfhe_polyeval"):
        s = Shape(12, 7, 2, 3, level=3, t=0 if "ckks" in fn else mc.T)
        if "ckks" in fn:   # the CKKS row wants the chain of DESIGN.md section 2.16
            import ckks_polyeval_ref as cr
            moduli = cr.ckks_chain(oracle_mod, 5, 2)
    c, R = make(12, moduli, s.L)
    run_case(ROWS[fn], c, R, s, 1400)


def overlap_cases():
    out = []
    for fn, row in sorted(ROWS.items()):
        if row.host:
            continue
        names = [n for b in row.bufs for n in b.names(SPECIAL)]
        for b in row.outputs():
            for o in b.names(SPECIAL):
                out += [(fn, o, x, w) for x in names if x != o for w in ("start", "end")]
    return out


@pytest.mark.parametrize("fn,out,other,where", overlap_cases())
def test_overlapping_output_is_rejected(make, fn, out, other, where):
    """the output over one 16-byte pair of another buffer of the call, measured at the level's sizes: DPFHE_ERR_INVALID naming the
    level, nothing written, nothing launched"""
    row, s = ROWS[fn], SPECIAL
    c, R = make(12, None, s.L)
    at, total = layout(row, s, over=(out, other, where))
    arena = Arena(row, s, at, total, 8000, "cuda")
    for n, v in inputs(row, R, s, np.random.default_rng(8001)).items():
        if n != out:
            arena.write(n, v)
    torch.cuda.synchronize()
    before, launches = arena.snapshot(), c.launch_count()
    with pytest.raises(RuntimeError, match="level %d: .*(overlap|must be)" % s.lv):
        row.run(c, s, arena.ptrs())
    torch.cuda.synchronize()
    assert c.launch_count() == launches
    assert np.array_equal(before[0], arena.snapshot()[0]), "%s: a rejected call wrote into the arena" % fn
