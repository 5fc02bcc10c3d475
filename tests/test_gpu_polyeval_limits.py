"""Polynomial evaluation on the GPU at its limits (DESIGN.md sections 2.15, 4.11), bit for bit against the restatement composed on the
oracle (tests/polyeval_ref.py): degree 64 over six levels; every level view of the persistent grouped key-switch kernel over several
rounds of its grid; the round numbering restarting inside view launches and on the context between applications; two evaluators on one
context and three streams; the host form with chunks that cut through rounds; and ct_lincomb / ct_add_plain where the grid-stride loop
wraps, against the oracle's pointwise products and sums.

The grid is made deterministic with DPFHE_KS_OCC=1 (read at context creation): ks_grouped_kernel then has one CTA per SM, so a view
at level l (group size l + K) runs floor(SMs / (l + K)) groups, and an application to B ciphertexts takes ceil(B / groups) rounds of
that view.  Ciphertexts are independent, so at large batches the restatement runs on a subset of batch indices: the first and last
ciphertext, and the last of every round and the first of the next at every view the application runs."""
import numpy as np
import pytest

import bases
import polyeval_ref as pr
from test_gpu_polyeval import SEED, T, _decrypt_slots, _encrypt_slots, _noise_bits, _setup_chain, dev, empty, host
from test_polyeval_limits_cpu import CHAINS, POLYS

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def product_levels(Lq, coeffs, t=T):
    """the level of every product of the schedule (DESIGN.md 2.15), in launch order: the powers k >= 2 the schedule makes, in increasing
    k, x^k at level Lq - ceil(log2 k) + 1"""
    d = len(coeffs) - 1
    need = [False] + [int(c) % t != 0 for c in coeffs[1:]]
    if not any(need):
        need[1] = True
    for k in range(d, 1, -1):
        if need[k]:
            u, v = pr.split(k)
            need[u] = need[v] = True
    return [Lq - pr.ceil_log2(k) + 1 for k in range(2, d + 1) if need[k]]


def view_groups(Lq, K, coeffs, sms):
    """{level: groups of ks_grouped_kernel} for every view the application runs, with one CTA per SM"""
    return {l: sms // (l + K) for l in set(product_levels(Lq, coeffs))}


def rounds(batch, groups):
    return -(-batch // groups)


def multi_round_batch(groups, exact):
    """the smallest batch r * g_min (+ 1 unless `exact`: one ciphertext into a further round) with r >= 3 that gives at least three
    rounds at every view, g_min the smallest group count of the schedule"""
    g_min, g_max = min(groups), max(groups)
    r = 3
    while r * g_min + (not exact) <= 2 * g_max:
        r += 1
    return r * g_min + (not exact)


def boundary_subset(batch, groups):
    """the first and last ciphertext, and at every view the last ciphertext of each round and the first of the next"""
    idx = {0, batch - 1}
    for g in groups:
        for r in range(g, batch, g):
            idx.update((r - 1, r))
    return sorted(idx)


def _context_with(monkeypatch, logn, moduli, **env):
    """a context created with the environment variables `env` set (DPFHE_KS_OCC, DPFHE_EPOCH_LIMIT: read at creation), unset again
    afterwards"""
    import deeppowers_b200 as dp
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    try:
        return dp.Context(logn, len(moduli), moduli)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def _relin_key(ctx, K, seed=SEED):
    """the device-generated grouped relinearisation key of the top level for K special primes (host)"""
    sk = empty(ctx.L, ctx.N)
    ctx.generate_secret(seed, sk)
    key = empty(ctx.key_digits(K), 2, ctx.L, ctx.N)
    ctx.generate_relin_key(K, T, sk, seed, key)
    return host(key)


def gen_mixed_wide(oracle_mod, Lq, K):
    """gen_mixed (tests/bases.py) widened to Lq ciphertext moduli and K special primes by generic primes of 52, 57 and 47 bits: its first
    four moduli, then the extra ciphertext moduli, then its two special primes and the extra special primes"""
    mixed = bases.catalogue(oracle_mod)["gen_mixed"]
    lib = oracle_mod.lib()
    extra = [bases._generic_prime(lib, b) for b in (52, 57, 47)]
    n_q = Lq - 4
    moduli = mixed[:4] + extra[:n_q] + mixed[4:] + extra[n_q:n_q + K - 2]
    assert len(moduli) == Lq + K and len(set(moduli)) == Lq + K
    assert bases.selects(moduli)[:2] == (False, True)   # the generic kernels, with the lift reduction
    return moduli


def restated(oracle_mod, logn, moduli, K, coeffs, ct, key, subset):
    """the restatement of the application to the ciphertexts `subset` of ct ([batch][2][Lq][N], host)"""
    return pr.polyeval(pr.Chain(oracle_mod, logn, moduli, K), T, coeffs, np.ascontiguousarray(ct[subset]), key)


def uniform_cts(oracle_mod, logn, moduli, B, seed):
    """[B][2][Lq][N] uniform residues under `moduli` (host): bit-exactness does not need encryptions"""
    o = oracle_mod.Oracle(logn, len(moduli), moduli)
    return o.fill_uniform(seed, 2 * B).reshape(B, 2, len(moduli), o.N)


# ---- 1. degree 64 and deep chains ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("Lq,K", CHAINS)
@pytest.mark.parametrize("name", list(POLYS))
def test_degree_64_over_six_levels(oracle_mod, capsys, Lq, K, name):
    """N = 4096, Lq = 7, K = 1 and 2 (ragged last digits at the views of levels 7, 5 and 3 with K = 2): degree 64 with every coefficient
    non-zero (INT64_MIN, INT64_MAX), degrees 33 and 63, a sparse degree 64.  Bit-exact at batch 2, the launch count of the restatement,
    and the slots decrypt to p(z) mod t (tests/test_polyeval_limits_cpu.py shows that the restatement decrypts at these shapes)"""
    import deeppowers_b200 as dp
    coeffs = POLYS[name]
    logn, B = 12, 2
    ctx, moduli, sk, key = _setup_chain(oracle_mod, logn, Lq, K, None)
    N = ctx.N
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    z = np.random.default_rng(Lq * 10 + K + len(coeffs)).integers(0, T, (B, 2, N // 2), dtype=np.int64)
    ct = _encrypt_slots(ctx_q, sk, z, T)
    pe = dp.PolyEval(ctx, K, T, coeffs, key)
    assert pe.result_limbs == 1
    out = empty(B, 2, 1, N)
    n0 = ctx.launch_count()
    pe.apply(ct, out, B)
    launches = ctx.launch_count() - n0
    stats = {}
    want = pr.polyeval(pr.Chain(oracle_mod, logn, moduli, K), T, coeffs, host(ct), key, stats=stats)
    assert np.array_equal(host(out), want)
    assert stats["mul"] == len(product_levels(Lq, coeffs))
    assert launches == stats["mul"] + 2 * stats["switch"] + stats["lincomb"]
    ctx_f = dp.Context(logn, 1, moduli[:1])
    assert np.array_equal(_decrypt_slots(ctx_f, sk, out, T), pr.poly_mod_t(coeffs, z, T))
    with capsys.disabled():
        print("\n[polyeval limits] N = %d, Lq = %d, K = %d, %s: %d products, noise %d bits on q_0"
              % (N, Lq, K, name, stats["mul"], _noise_bits(ctx_f, sk, out)))
    pe.close()
    for c in (ctx_f, ctx_q, ctx):
        c.close()


# ---- 2. every view over several rounds ---------------------------------------------------------------------------------------------

DEG8 = [3, -1, 2, 5, I64_MIN, 7, 1, -4, I64_MAX]
DEG4 = [1, -2, 3, -4, 5]
DEG3 = [-5, 2, 0, 11]
DEG2 = [7, 0, -9]
# (log N, Lq, K, basis, coefficients): the default basis at N = 4096 and 8192 (views at levels 4, 3, 2), gen_mixed widened to Lq = 5 with
# K = 3 and 4 (ragged last digits, the generic kernels), N = 16384 (views at levels 4 and 3)
MULTI = [
    (12, 4, 2, None, DEG8),
    (13, 4, 2, None, DEG8),
    (12, 5, 3, "gen_mixed", DEG4),
    (12, 5, 3, "gen_mixed", DEG2),
    (12, 5, 4, "gen_mixed", DEG4),
    (12, 5, 4, "gen_mixed", DEG2),
    (14, 4, 2, None, DEG3),
]


@pytest.mark.parametrize("exact", [False, True], ids=["one_past_a_round", "on_a_round_boundary"])
@pytest.mark.parametrize("logn,Lq,K,basis,coeffs", MULTI)
def test_every_view_over_several_rounds(oracle_mod, monkeypatch, logn, Lq, K, basis, coeffs, exact):
    """one CTA per SM: at least three rounds at every view, the batch one ciphertext past whole rounds of the smallest group count or
    ending exactly on them.  The boundary subset against the restatement, and the full batch against a context without the cap, whose
    grid has other group counts and so other round boundaries"""
    import deeppowers_b200 as dp
    moduli = gen_mixed_wide(oracle_mod, Lq, K) if basis else oracle_mod.Oracle(logn, Lq + K).moduli
    groups = view_groups(Lq, K, coeffs, _sms())
    B = multi_round_batch(groups.values(), exact)
    assert all(rounds(B, g) >= 3 for g in groups.values()), (B, groups)
    assert (B % min(groups.values()) == 0) == exact
    ctx = _context_with(monkeypatch, logn, moduli, DPFHE_KS_OCC=1)
    key = _relin_key(ctx, K)
    x = uniform_cts(oracle_mod, logn, moduli[:Lq], B, 300 + logn + K)
    pe = dp.PolyEval(ctx, K, T, coeffs, key)
    Lf = pe.result_limbs
    out = empty(B, 2, Lf, ctx.N)
    pe.apply(dev(x), out, B)
    got = host(out)
    subset = boundary_subset(B, groups.values())
    assert np.array_equal(got[subset], restated(oracle_mod, logn, moduli, K, coeffs, x, key, subset))
    free = dp.Context(logn, Lq + K, moduli)
    pe_free = dp.PolyEval(free, K, T, coeffs, key)
    out_free = empty(B, 2, Lf, ctx.N)
    pe_free.apply(dev(x), out_free, B)
    assert np.array_equal(host(out_free), got)
    for e in (pe_free, pe):
        e.close()
    free.close()
    ctx.close()


# ---- 3. the round numbering restarts inside applications ---------------------------------------------------------------------------

def simulate_epochs(batches, limit, epoch=0):
    """epoch_guard (csrc/kernels.cu) over a sequence of persistent launches of `batches` ciphertexts each: a launch restarts the numbering
    (epoch = 0) when epoch + b + 1 >= limit, then consumes b + 1 rounds.  Returns which launches restart."""
    out = []
    for b in batches:
        restart = epoch + b + 1 >= limit
        if restart:
            epoch = 0
        out.append(restart)
        epoch += b + 1
    return out


def test_round_numbering_restarts_inside_applications(oracle_mod, monkeypatch):
    """DPFHE_EPOCH_LIMIT = 40, N = 4096, Lq = 4, K = 2, degree 8: seven products per application on the views of levels 4, 3, 3, 2, 2, 2,
    2, each on B = 9 ciphertexts (10 rounds).  After each application the context itself runs ct_mul_relin_grouped on 9 ciphertexts
    (10 rounds) and rotate_hoisted_grouped on 20 (one ks_hoistg_kernel launch, 21 rounds).  The counter after each launch (R: the
    launch restarted the numbering):
        application 1:  10 20 30 R10 20 30 R10     restarts at products 4 and 7 (level 2)
        context:        20 (ct x ct), R21 (rotation: 20 + 21 >= 40)
        application 2:  31 R10 20 30 R10 20 30     starts from the context's restarted count; restarts at products 2 (level 3), 5
        context:        R10 (ct x ct: 30 + 10 >= 40), 31 (rotation)
        application 3:  R10 20 30 R10 20 30 R10    restarts at products 1 (level 4), 4 and 7
        context:        20, R21
    So the numbering restarts inside view launches at all three levels and at different products, a restarted count goes from a view
    back to the context (the ct x ct after application 1 continues from 10) and from the context to a view (application 2 starts at
    21).  Every result equals the restatement or the oracle."""
    import deeppowers_b200 as dp
    logn, Lq, K, B, Bm, Br, limit = 12, 4, 2, 9, 9, 20, 40
    coeffs = DEG8
    levels = product_levels(Lq, coeffs)
    assert levels == [4, 3, 3, 2, 2, 2, 2]
    launches = (levels + ["ct_mul", "rotate"]) * 3
    restart = simulate_epochs([B] * 7 + [Bm, Br] + [B] * 7 + [Bm, Br] + [B] * 7 + [Bm, Br], limit)
    per_app = [[j + 1 for j in range(7) if restart[9 * a + j]] for a in range(3)]
    assert per_app == [[4, 7], [2, 5], [1, 4, 7]]
    assert {levels[j - 1] for p in per_app for j in p} == {4, 3, 2}
    assert [launches[i] for i in range(len(launches)) if restart[i] and isinstance(launches[i], str)] == ["rotate", "ct_mul", "rotate"]
    moduli = oracle_mod.Oracle(logn, Lq + K).moduli
    ctx = _context_with(monkeypatch, logn, moduli, DPFHE_EPOCH_LIMIT=limit)
    key = _relin_key(ctx, K)
    o = oracle_mod.Oracle(logn, Lq + K, moduli)
    x = uniform_cts(oracle_mod, logn, moduli[:Lq], B, 401)
    a = uniform_cts(oracle_mod, logn, moduli[:Lq], Bm, 402)
    b = uniform_cts(oracle_mod, logn, moduli[:Lq], Bm, 403)
    r = uniform_cts(oracle_mod, logn, moduli[:Lq], Br, 404)
    gk = o.fill_uniform(405, 2 * o.grouped_digits(K)).reshape(-1, 2, Lq + K, o.N)
    g = o.galois_elt(3)
    want = restated(oracle_mod, logn, moduli, K, coeffs, x, key, list(range(B)))
    want_mul = o.ct_mul_relin_grouped(K, a, b, key, T)
    want_rot = o.rotate_hoisted_grouped(K, r, [g], gk[None], T)
    pe = dp.PolyEval(ctx, K, T, coeffs, key)
    dx, da, db, dr, dkey, dgk = (dev(v) for v in (x, a, b, r, key, gk))
    out = empty(B, 2, pe.result_limbs, o.N)
    out_mul = empty(Bm, 2, Lq, o.N)
    out_rot = empty(1, Br, 2, Lq, o.N)
    for app in range(3):
        pe.apply(dx, out, B)
        assert np.array_equal(host(out), want), app
        ctx.ct_mul_relin_grouped(K, da, db, dkey, out_mul, Bm, T)
        assert np.array_equal(host(out_mul), want_mul), app
        ctx.rotate_hoisted_grouped(K, dr, [g], [dgk], out_rot, Br, T)
        assert np.array_equal(host(out_rot), want_rot), app
    pe.close()
    ctx.close()


# ---- 4. two evaluators on one context ----------------------------------------------------------------------------------------------

def _apply_on(pe, ct, out, batch, stream):
    """stream: a torch stream, or "own" for the context's own stream (a null stream handle through the C ABI)"""
    if stream == "own":
        pe.ctx._chk(pe._l.dpfhe_polyeval_apply(pe._h, ct.data_ptr(), out.data_ptr(), batch, None))
    else:
        pe.apply(ct, out, batch, stream=stream)


def test_two_evaluators_on_one_context(oracle_mod, monkeypatch):
    """K = 1 (Lq = 5, degree 5: views at levels 5, 4, 3) and K = 2 (Lq = 4, degree 4: views at levels 4, 3) on one L = 6 context at
    N = 4096 with one CTA per SM: their views share the context's digit slots, flags, mailboxes, ticket and round counter.  The
    applications alternate between the evaluators and between two streams and the context's own stream, with batches that go up and
    then down, so that each evaluator's scratch grows while the other's work may still be in flight.  Each result equals the
    restatement for its own K on the boundary subset, and the same rows of one application to the largest batch run alone."""
    import deeppowers_b200 as dp
    logn, L = 12, 6
    moduli = oracle_mod.Oracle(logn, L).moduli
    sms = _sms()
    ctx = _context_with(monkeypatch, logn, moduli, DPFHE_KS_OCC=1)
    spec = {1: [2, -3, 0, 5, 1, I64_MIN], 2: [I64_MAX, 4, -1, 0, 6]}
    groups = {K: view_groups(L - K, K, c, sms) for K, c in spec.items()}
    assert sorted(groups[1]) == [3, 4, 5] and sorted(groups[2]) == [3, 4]
    b_max = max(multi_round_batch(g.values(), False) for g in groups.values())
    assert all(rounds(b_max, n) >= 3 for g in groups.values() for n in g.values())
    batches = [2, b_max // 3, b_max // 2, b_max, b_max // 2 + 1, 5]   # up, then down
    ev, key, x, dx = {}, {}, {}, {}
    for K, coeffs in spec.items():
        key[K] = _relin_key(ctx, K, bytes(range(K, K + 32)))
        ev[K] = dp.PolyEval(ctx, K, T, coeffs, key[K])
        x[K] = uniform_cts(oracle_mod, logn, moduli[:L - K], b_max, 500 + K)
        dx[K] = dev(x[K])
    legs = [torch.cuda.Stream(), torch.cuda.Stream(), "own"]
    outs = []
    torch.cuda.synchronize()
    for i, b in enumerate(batches):
        for j, K in enumerate(spec):
            o = empty(b, 2, ev[K].result_limbs, ctx.N)
            _apply_on(ev[K], dx[K], o, b, legs[(i + j) % 3])
            outs.append((K, b, o))
    torch.cuda.synchronize()
    ctx.synchronize()
    for K, coeffs in spec.items():
        alone = empty(b_max, 2, ev[K].result_limbs, ctx.N)
        ev[K].apply(dx[K], alone, b_max)
        alone = host(alone)
        subset = sorted(set(boundary_subset(b_max, groups[K].values())) | {b - 1 for b in batches})
        want = dict(zip(subset, restated(oracle_mod, logn, moduli, K, coeffs, x[K], key[K], subset)))
        assert np.array_equal(alone[subset], np.stack([want[i] for i in subset]))
        for k, b, o in outs:
            if k == K:
                got = host(o)
                assert np.array_equal(got, alone[:b]), (K, b)
                assert all(np.array_equal(got[i], want[i]) for i in subset if i < b), (K, b)
    for e in ev.values():
        e.close()
    ctx.close()


# ---- 5. the host form across rounds ------------------------------------------------------------------------------------------------

def test_host_form_chunks_cut_through_rounds(oracle_mod, monkeypatch):
    """N = 4096, Lq = 4, K = 2, degree 8, one CTA per SM.  DPFHE_POLYEVAL_CHUNK is one and a half rounds of the smallest group count,
    moved off every view's round boundary, and the batch is four chunks and one ciphertext: five chunks, more than the three staging
    slots, cutting through the middle of rounds, the last a single ciphertext.  The host form equals the device form on the whole batch,
    which equals the restatement on the round and chunk boundaries"""
    import deeppowers_b200 as dp
    logn, Lq, K, coeffs = 12, 4, 2, DEG8
    moduli = oracle_mod.Oracle(logn, Lq + K).moduli
    groups = sorted(set(view_groups(Lq, K, coeffs, _sms()).values()))
    chunk = 3 * groups[0] // 2
    while any(chunk % g == 0 for g in groups):
        chunk += 1
    B = 4 * chunk + 1
    assert all(rounds(B, g) >= 3 for g in groups) and chunk % groups[0]
    ctx = _context_with(monkeypatch, logn, moduli, DPFHE_KS_OCC=1)
    key = _relin_key(ctx, K)
    x = uniform_cts(oracle_mod, logn, moduli[:Lq], B, 601)
    pe = dp.PolyEval(ctx, K, T, coeffs, key)
    Lf = pe.result_limbs
    out = empty(B, 2, Lf, ctx.N)
    pe.apply(dev(x), out, B)
    got = host(out)
    subset = sorted(set(boundary_subset(B, groups)) | {i for c in range(chunk, B, chunk) for i in (c - 1, c)})
    assert np.array_equal(got[subset], restated(oracle_mod, logn, moduli, K, coeffs, x, key, subset))
    monkeypatch.setenv("DPFHE_POLYEVAL_CHUNK", str(chunk))
    h = np.empty((B, 2, Lf, ctx.N), dtype=np.uint64)
    pe.apply_host(x, h)
    assert np.array_equal(h, got)
    pe.close()
    ctx.close()


# ---- 6. ct_lincomb / ct_add_plain where the grid-stride loop wraps -----------------------------------------------------------------

# (log N, L): the largest coefficient table (L = 16) at both row lengths, and L = 7, which does not divide a grid pass's rows
WRAP_SHAPES = [(14, 16), (12, 16), (12, 7)]
N_TERMS = (8, 9, 64)   # LincombArgs<8>, and LincombArgs<64> at 9 and 64 terms


def grid_pass(sms):
    """128-bit chunks one pass of ct_lincomb_kernel's grid covers: launch_lincomb_t caps the grid at 32 CTAs of 256 threads per SM"""
    return 32 * sms * 256


def wrap_batch(logn, L, sms):
    """the smallest batch whose B * 2 * L * N / 2 chunks take the grid-stride loop past its second pass"""
    return 2 * grid_pass(sms) // (L << logn) + 1


def test_wrap_shapes_move_limbs_between_passes():
    """a pass covers grid_pass / (N / 2) rows; a shape whose L does not divide that puts the chunk at first-pass position p and the
    chunk one pass later on different limbs, so that limb parameters read for the first-pass position give wrong results"""
    sms = _sms()
    assert any((grid_pass(sms) >> (logn - 1)) % L for logn, L in WRAP_SHAPES)


@pytest.mark.parametrize("logn,L", WRAP_SHAPES)
def test_lincomb_and_add_plain_where_the_grid_wraps(oracle_mod, logn, L):
    """8, 9 and 64 terms with INT64_MIN, INT64_MAX, 0, 1 and -1 among the coefficients and the constant INT64_MIN, inputs at q - 1 in
    places, the output apart and aliasing the last input; ct_add_plain apart and in place.  Every word of the output against the
    oracle's pointwise products (by c mod q_l on limb l) and sums: exact 128-bit arithmetic outside csrc/"""
    import deeppowers_b200 as dp
    sms = _sms()
    B, N = wrap_batch(logn, L, sms), 1 << logn
    assert B * L * N > 2 * grid_pass(sms)
    ctx = dp.Context(logn, L)
    o = oracle_mod.Oracle(logn, L, ctx.moduli)
    shape = (B, 2, L, N)
    d = []
    for i in range(max(N_TERMS)):
        x = empty(*shape)
        ctx.fill_uniform(700 + i, x, 2 * B)
        d.append(x)
    top = torch.tensor([q - 1 for q in ctx.moduli], dtype=torch.int64, device="cuda")[:, None]
    d[0][:, :, :, :64] = top   # the first 64 coefficients of every row
    d[1][-1] = top             # the whole last ciphertext
    d[2][B // 2:] = top        # the second half of the batch: rows of the second and third passes
    rng = np.random.default_rng(L)
    coeffs = [I64_MIN, I64_MAX, 0, 1, -1] + [int(c) for c in rng.integers(I64_MIN, I64_MAX, 59, dtype=np.int64, endpoint=True)]
    coeffs[10::7] = [-1] * len(coeffs[10::7])
    constant = I64_MIN
    hx = [host(v) for v in d]

    def limbwise(c):
        return np.array([pr.floor_mod(c, q) for q in o.moduli], dtype=np.uint64)[None, None, :, None]

    acc = np.zeros(shape, dtype=np.uint64)
    acc[:, 0] = limbwise(constant)[0]
    want = {}
    for i in range(max(N_TERMS)):
        acc = o.poly_add(acc, o.poly_mul_pointwise(hx[i], np.broadcast_to(limbwise(coeffs[i]), shape)))
        if i + 1 in N_TERMS:
            want[i + 1] = acc
    out = empty(*shape)
    for n in N_TERMS:
        ctx.ct_lincomb(d[:n], coeffs[:n], constant, out, B)
        assert np.array_equal(host(out), want[n]), n
        alias = d[n - 1].clone()
        ctx.ct_lincomb(d[:n - 1] + [alias], coeffs[:n], constant, alias, B)
        assert np.array_equal(host(alias), want[n]), n
    pt = empty(1, L, N)
    ctx.fill_uniform(800, pt, 1)
    ptc0 = np.zeros(shape, dtype=np.uint64)
    ptc0[:, 0] = host(pt)[0]
    want_pt = o.poly_add(hx[1], ptc0)
    ctx.ct_add_plain(d[1], pt[0], out, B)
    assert np.array_equal(host(out), want_pt)
    ctx.ct_add_plain(d[1], pt[0], d[1], B)
    assert np.array_equal(host(d[1]), want_pt)
    ctx.close()
