"""CKKS polynomial evaluation on the GPU (DESIGN.md sections 2.16, 4.12): PolyEval.ckks bit for bit against the restatement composed
on the oracle (tests/ckks_polyeval_ref.py) with its launch count, the decoded slots against p(z) in float64 within the recorded
bound, the host form, a CKKS and a BGV evaluator on one context over two streams, device bytes, argument checks, and the C++ example."""
import math
import os
import subprocess

import numpy as np
import pytest

import bases
import ckks_polyeval_ref as cr
import polyeval_ref as pr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(100, 132))
DELTA = 2.0**45
ERR_REL = 2.0**-24   # as tests/test_ckks_polyeval_cpu.py (DESIGN.md section 2.16)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def _moduli(oracle_mod, logn, Lq, K, basis):
    if basis == "ckks":
        return cr.ckks_chain(oracle_mod, Lq, K)
    if basis:
        return bases.catalogue(oracle_mod)[basis][:Lq + K]
    return oracle_mod.Oracle(logn, Lq + K).moduli


def _setup(oracle_mod, logn, Lq, K, basis):
    import deeppowers_b200 as dp
    moduli = _moduli(oracle_mod, logn, Lq, K, basis)
    ctx = dp.Context(logn, Lq + K, moduli)
    sk = empty(Lq + K, ctx.N)
    ctx.generate_secret(SEED, sk)
    key = empty(ctx.key_digits(K), 2, Lq + K, ctx.N)
    ctx.generate_relin_key(K, 0, sk, SEED, key)
    return ctx, moduli, sk, host(key)


def _encrypt(ctx_q, sk, z, scale=DELTA):
    B = z.shape[0]
    pt, ct = empty(B, ctx_q.L, ctx_q.N), empty(B, 2, ctx_q.L, ctx_q.N)
    ctx_q.ckks_encode(torch.from_numpy(np.ascontiguousarray(z, dtype=np.complex128)).cuda(), pt, B, scale)
    ctx_q.encrypt(0, sk[:ctx_q.L].contiguous(), SEED, 0, pt, ct, B)
    return ct


def _decode(ctx_f, sk, ct, scale):
    B = ct.shape[0]
    ph = empty(B, ctx_f.L, ctx_f.N)
    ctx_f.decrypt(sk[:ctx_f.L].contiguous(), ct.contiguous(), 2, ph, B)
    z = torch.empty((B, ctx_f.N // 2), dtype=torch.complex128, device="cuda")
    ctx_f.ckks_decode(ph, z, B, scale)
    return z.cpu().numpy()


def _slots(seed, B, n):
    return np.random.default_rng(seed).uniform(-1, 1, (B, n)) + 0j


GELU7 = [0.0, 0.5, 0.39894228, 0.0, -0.06649038, 0.0, 0.00997356, 0.0]   # degree-7 Taylor fit of GELU at 0
# (log N, Lq, K, basis, coefficients): K = 1 .. 4 (K = 3 with Lq = 5 and K = 4 with Lq = 6: ragged last digits), every N, the CKKS
# chain, the default basis and a generic basis (bit-exactness only: their scales drift)
CASES = [
    (12, 5, 1, "ckks", GELU7),
    (12, 5, 2, "ckks", [1.0, -2.0, 3.0, -4.0, 5.0, -6.0, 7.0, -8.0, 9.0]),
    (13, 5, 2, "ckks", [0.1, 0.0, 0.0, 0.7]),
    (14, 5, 2, "ckks", GELU7),
    (12, 5, 3, "ckks", [0.5, 0.0, 0.25, 0.0, -0.125]),
    (12, 6, 4, "ckks", [0.3, 0.2, 0.1]),
    (12, 4, 1, "ckks", [0.25, 0.5]),
    (12, 4, 2, None, [0.5, 0.25, 0.125, -1.0]),
    (13, 4, 2, "gen_mixed", [0.5, -1.5, 0.0, 2.0]),
    (14, 4, 2, "gen_mixed", [-0.0, 1.0, 1e3]),
]


@pytest.mark.parametrize("logn,Lq,K,basis,coeffs", CASES)
def test_ckks_polyeval_bit_exact_and_decodes(oracle_mod, logn, Lq, K, basis, coeffs):
    import deeppowers_b200 as dp
    ctx, moduli, sk, key = _setup(oracle_mod, logn, Lq, K, basis)
    N, B = ctx.N, 2
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    z = _slots(logn * 100 + Lq * 10 + K, B, N // 2)
    ct = _encrypt(ctx_q, sk, z)
    pe = dp.PolyEval.ckks(ctx, K, coeffs, DELTA, key)
    Lf = pe.result_limbs
    assert Lf == Lq - pr.ceil_log2(len(coeffs) - 1) - 1 and pe.result_scale == DELTA
    out = empty(B, 2, Lf, N)
    n0 = ctx.launch_count()
    pe.apply(ct, out, B)
    launches = ctx.launch_count() - n0
    stats = {}
    want = cr.polyeval(pr.Chain(oracle_mod, logn, moduli, K), coeffs, DELTA, host(ct), key, stats=stats)
    assert np.array_equal(host(out), want)
    assert launches == stats["launches"]
    if basis == "ckks":
        ctx_f = dp.Context(logn, Lf, moduli[:Lf])
        got = _decode(ctx_f, sk, out, pe.result_scale)
        err = float(np.max(np.abs(got - cr.poly_eval(coeffs, z)) / (1 + cr.power_sum(coeffs, z))))
        print("\n[ckks polyeval] N = %d, Lq = %d, K = %d, d = %d: relative error %.3g" % (N, Lq, K, len(coeffs) - 1, err))
        assert err <= ERR_REL
        ctx_f.close()
    pe.close()
    ctx_q.close()
    ctx.close()


def test_degree_64(oracle_mod):
    """every coefficient non-zero (64 terms: the 64-term parameter block) on Lq = 8, K = 2 at N = 4096"""
    import deeppowers_b200 as dp
    logn, Lq, K, B = 12, 8, 2, 2
    ctx, moduli, sk, key = _setup(oracle_mod, logn, Lq, K, "ckks")
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    rng = np.random.default_rng(64)
    coeffs = [float(rng.normal()) / 2**(k // 4) for k in range(65)]
    z = _slots(64, B, ctx.N // 2)
    ct = _encrypt(ctx_q, sk, z)
    pe = dp.PolyEval.ckks(ctx, K, coeffs, DELTA, key)
    out = empty(B, 2, pe.result_limbs, ctx.N)
    n0 = ctx.launch_count()
    pe.apply(ct, out, B)
    launches = ctx.launch_count() - n0
    stats = {}
    assert np.array_equal(host(out), cr.polyeval(pr.Chain(oracle_mod, logn, moduli, K), coeffs, DELTA, host(ct), key, stats=stats))
    assert launches == stats["launches"] and pe.result_limbs == 1
    ctx_f = dp.Context(logn, 1, moduli[:1])
    got = _decode(ctx_f, sk, out, DELTA)
    err = float(np.max(np.abs(got - cr.poly_eval(coeffs, z)) / (1 + cr.power_sum(coeffs, z))))
    print("\n[ckks polyeval] N = 4096, d = 64 dense: relative error %.3g" % err)
    assert err <= ERR_REL
    for c in (pe, ctx_f, ctx_q, ctx):
        c.close()


def test_host_form_and_device_bytes(oracle_mod, monkeypatch):
    """chunks of 3 over a batch of 7 (the last chunk one ciphertext) equal the device form; scratch grows with the batch by
    16 N batch (R + 1) bytes (DESIGN.md section 4.12), counts in the context's device bytes and is released on destroy"""
    import deeppowers_b200 as dp
    logn, Lq, K, B = 12, 5, 2, 7
    ctx, moduli, sk, key = _setup(oracle_mod, logn, Lq, K, "ckks")
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    ct = _encrypt(ctx_q, sk, _slots(3, B, ctx.N // 2))
    before = ctx.device_bytes()
    pe = dp.PolyEval.ckks(ctx, K, GELU7, DELTA, key, scale_out=2.0**40)
    assert pe.result_scale == 2.0**40
    Lf = pe.result_limbs
    out = empty(B, 2, Lf, ctx.N)
    pe.apply(ct[:2], out[:2], 2)
    at2 = ctx.device_bytes()
    pe.apply(ct, out, B)
    at7 = ctx.device_bytes()
    # GELU7 makes x^2 (level 4), x^4 (3), x^6 (2) and cuts x^2 to level 3, with one top-level product buffer: R = 5 + 4 + 3 + 2 + 3
    R = 17
    assert before < at2 and at7 - at2 == 16 * ctx.N * (B - 2) * (R + 1)
    monkeypatch.setenv("DPFHE_POLYEVAL_CHUNK", "3")
    h = np.empty((B, 2, Lf, ctx.N), dtype=np.uint64)
    pe.apply_host(host(ct), h)   # chunks of 3: the scratch does not grow
    assert np.array_equal(h, host(out))
    alive = ctx.device_bytes()
    pe.close()
    assert alive - ctx.device_bytes() >= 16 * ctx.N * B * (R + 1)   # the scratch, the level tables and the keys
    ctx_q.close()
    ctx.close()


def test_ckks_and_bgv_evaluators_on_one_context_over_two_streams(oracle_mod):
    import deeppowers_b200 as dp
    logn, Lq, K, B, T = 13, 5, 2, 32, 65537
    ctx, moduli, sk, key = _setup(oracle_mod, logn, Lq, K, "ckks")
    bkey = empty(ctx.key_digits(K), 2, Lq + K, ctx.N)
    ctx.generate_relin_key(K, T, sk, SEED, bkey)
    ctx_q = dp.Context(logn, Lq, moduli[:Lq])
    ct = _encrypt(ctx_q, sk, _slots(8, B, ctx.N // 2))
    o = oracle_mod.Oracle(logn, Lq, moduli[:Lq])
    bct = dev(o.fill_uniform(9, 2 * B).reshape(B, 2, Lq, o.N))
    pc = dp.PolyEval.ckks(ctx, K, GELU7, DELTA, key)
    pb = dp.PolyEval(ctx, K, T, [1, 2, 3, 4], host(bkey))
    assert pb.result_scale == 0.0
    rc, rb = empty(B, 2, pc.result_limbs, ctx.N), empty(B, 2, pb.result_limbs, ctx.N)
    pc.apply(ct, rc, B)
    pb.apply(bct, rb, B)
    ctx.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    oc, ob = torch.zeros_like(rc), torch.zeros_like(rb)
    for _ in range(3):
        pc.apply(ct, oc, B, stream=s1)
        pb.apply(bct, ob, B, stream=s2)
    torch.cuda.synchronize()
    assert np.array_equal(host(oc), host(rc)) and np.array_equal(host(ob), host(rb))
    chain = pr.Chain(oracle_mod, logn, moduli, K)
    assert np.array_equal(host(rc), cr.polyeval(chain, GELU7, DELTA, host(ct), key))
    assert np.array_equal(host(rb), pr.polyeval(chain, T, [1, 2, 3, 4], host(bct), host(bkey)))
    for c in (pc, pb, ctx_q, ctx):
        c.close()


def test_argument_errors(oracle_mod):
    import deeppowers_b200 as dp
    logn, Lq, K = 12, 5, 2
    ctx, moduli, sk, key = _setup(oracle_mod, logn, Lq, K, "ckks")
    bad = [
        dict(coeffs=[1.0] * 17),                         # d = 16: D = 4 > Lq - 2 (d = 8, D = 3, is the deepest valid)
        dict(coeffs=[1.0]),                              # d = 0
        dict(coeffs=[1.0] * 66),                         # d = 65
        dict(coeffs=[1.0, math.inf]),
        dict(coeffs=[math.nan, 1.0]),
        dict(coeffs=[1.0, 1.0], scale_in=0.0),
        dict(coeffs=[1.0, 1.0], scale_in=math.inf),
        dict(coeffs=[1.0, 1.0], scale_out=-1.0),
        dict(coeffs=[1.0, 1.0], scale_out=math.nan),
    ]
    for b in bad:
        with pytest.raises(dp.DpfheError):
            dp.PolyEval.ckks(ctx, K, b["coeffs"], b.get("scale_in", DELTA), key, scale_out=b.get("scale_out"))
    ctx4 = dp.Context(logn, 7, moduli)                    # K = 4: Lq = 3, D <= Lq - K + 1 = 0 and D <= 1
    with pytest.raises(dp.DpfheError):
        dp.PolyEval.ckks(ctx4, 4, [1.0, 1.0, 1.0], DELTA, np.zeros((1, 2, 7, ctx.N), dtype=np.uint64))
    lib = ctx._l
    C = dp.evaluator.C
    cs = (C.c_double * 2)(1.0, 1.0)
    pe = C.c_void_p()
    assert lib.dpfhe_polyeval_create_ckks(ctx._h, K, None, 1, DELTA, DELTA, key.ctypes.data, C.byref(pe)) == -1
    assert lib.dpfhe_polyeval_create_ckks(ctx._h, K, cs, 1, DELTA, DELTA, None, C.byref(pe)) == -1
    assert lib.dpfhe_polyeval_result_scale(None) == 0.0
    pev = dp.PolyEval.ckks(ctx, K, [0.0, 1.0, 1.0], DELTA, key)
    x = empty(1, 2, Lq, ctx.N)
    with pytest.raises(dp.DpfheError, match="overlap"):
        pev.apply(x, x, 1)
    pev.close()
    ctx4.close()
    ctx.close()


def test_cpp_ckks_activation_example(tmp_path):
    """examples/encrypted_ckks_activation.cpp links libdpfhe.so alone and reports an error within the recorded bound"""
    import deeppowers_b200
    deeppowers_b200.load_library()
    torch.cuda.empty_cache()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir, exe = os.path.join(root, "deeppowers_b200"), str(tmp_path / "encrypted_ckks_activation")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           os.path.join(root, "examples", "encrypted_ckks_activation.cpp"), "-L", lib_dir, "-ldpfhe", "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout)
    line = [ln for ln in r.stdout.splitlines() if "largest error" in ln][0]
    err = float(line.split("largest error")[1].split()[0])
    assert err <= ERR_REL * 4, line   # |z| <= 1: 1 + sum |a_k| < 4 for the fit
