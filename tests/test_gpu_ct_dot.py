"""Encrypted inner products on the GPU (DESIGN.md section 2.18 / 4.15): dpfhe_ct_dot_grouped through the C ABI, bit-exact against
the oracle restatement (tests/ct_dot_ref.py), against the device composition it replaces (ct_tensor + poly_add + keyswitch_grouped +
poly_add) and, for one pair, against dpfhe_ct_mul_relin_grouped; aliasing, the host form, argument checks, launch count and scratch;
attention scores of 64 components end to end.  Every case runs once."""
import os
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import ct_dot_ref as cdr  # noqa: E402
from bases import catalogue  # noqa: E402
from test_gpu_parity import ctxs, dev, dp, host  # noqa: E402,F401  (ctxs and dp are fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_TERMS = [1, 2, 7, 8, 9, 15, 16, 17, 33, 64]


@pytest.fixture(scope="module", autouse=True)
def _release_cached_blocks():
    """the library allocates with cudaMalloc, which cannot use blocks torch keeps cached: hand this module's back when it is done"""
    yield
    torch.cuda.empty_cache()


def _setup(ctxs, oracle_mod, log_n, L, K, moduli=None):
    c, o = ctxs(log_n, L, moduli)
    cq, oq = ctxs(log_n, L - K, list(o.moduli[:L - K]))
    return c, o, cq, oq


def _pool(oq, n_pool, batch, seed):
    pool = oq.fill_uniform(seed, n_pool * batch * 2).reshape(n_pool, batch, 2, oq.L, oq.N)
    q = np.array(oq.moduli, dtype=np.uint64)
    pool[0, -1, 0] = (q - 1)[:, None]
    pool[-1, 0, 1] = 0
    return pool


def _pairs(n, n_pool):
    ia = [(2 * t) % n_pool for t in range(n)]
    ib = [(2 * t + 1) % n_pool for t in range(n)]
    ib[-1] = ia[-1]   # a square
    return ia, ib


def _device_composition(c, cq, K, a_list, b_list, dkey, batch, t):
    """the calls the inner product replaces, with the same bits"""
    Lq, N = cq.L, cq.N
    d = torch.empty((batch, 3, Lq, N), dtype=torch.int64, device="cuda")
    acc = torch.empty_like(d)
    cq.ct_tensor(a_list[0], b_list[0], acc, batch)
    for x, y in zip(a_list[1:], b_list[1:]):
        cq.ct_tensor(x, y, d, batch)
        cq.poly_add(acc, d, acc, 3 * batch)
    d2 = acc[:, 2].contiguous()
    ks = torch.empty((batch, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.keyswitch_grouped(K, d2, dkey, ks, batch, t)
    d01 = acc[:, :2].contiguous()
    out = torch.empty_like(ks)
    cq.poly_add(d01, ks, out, 2 * batch)
    return out


@pytest.mark.parametrize("n_terms", N_TERMS)
def test_every_term_count(ctxs, oracle_mod, n_terms):
    K, L, log_n, batch = 2, 6, 12, 3
    c, o, cq, oq = _setup(ctxs, oracle_mod, log_n, L, K)
    n_pool = min(2 * n_terms, 12)
    pool = _pool(oq, n_pool, batch, 300 + n_terms)
    ia, ib = _pairs(n_terms, n_pool)
    key = o.fill_uniform(400 + n_terms, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    a_list, b_list = [dpool[i] for i in ia], [dpool[i] for i in ib]
    for t in (0, 65537):
        out = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
        c.ct_dot_grouped(K, a_list, b_list, dkey, out, batch, t)
        want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], key, t)
        assert np.array_equal(host(out).reshape(want.shape), want), t
        assert torch.equal(out, _device_composition(c, cq, K, a_list, b_list, dkey, batch, t)), t
        if n_terms == 1:
            ref = torch.empty_like(out)
            c.ct_mul_relin_grouped(K, a_list[0], b_list[0], dkey, ref, batch, t)
            assert torch.equal(out, ref)


@pytest.mark.parametrize("log_n,L,K,batch,n_terms,t", [(12, 4, 1, 3, 9, 65537), (13, 6, 2, 1, 17, 65537), (13, 7, 2, 4, 8, 0), (14, 6, 2, 3, 16, 65537),
                                                       (12, 7, 3, 2, 33, 65537), (12, 8, 4, 2, 15, 0), (13, 6, 2, 300, 2, 65537),
                                                       (14, 6, 2, 70, 3, 0)])
def test_shapes_degrees_and_batches(ctxs, oracle_mod, log_n, L, K, batch, n_terms, t):
    """K = 1 .. 4, ragged digits (Lq = 5, K = 2), every ring degree, a batch of one and batches over more than three grid rounds"""
    c, o, cq, oq = _setup(ctxs, oracle_mod, log_n, L, K)
    n_pool = min(2 * n_terms, 4)
    pool = _pool(oq, n_pool, batch, 500 + log_n + L)
    ia, ib = _pairs(n_terms, n_pool)
    key = o.fill_uniform(600 + L, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    a_list, b_list = [dpool[i] for i in ia], [dpool[i] for i in ib]
    out = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
    c.ct_dot_grouped(K, a_list, b_list, dkey, out, batch, t)
    assert torch.equal(out, _device_composition(c, cq, K, a_list, b_list, dkey, batch, t))
    m = min(batch, 4)   # the restatement on the first and the last ciphertexts
    for sl in (slice(0, m), slice(batch - m, batch)):
        want = cdr.ct_dot(o, oq, K, [pool[i][sl] for i in ia], [pool[i][sl] for i in ib], key, t)
        assert np.array_equal(host(out[sl]).reshape(want.shape), want)


@pytest.mark.parametrize("basis", ["gen_mixed", "fast_mixed"])
def test_other_bases(ctxs, oracle_mod, basis):
    mods = catalogue(oracle_mod)[basis]
    K, L, log_n, batch, n_terms = 2, len(mods), 12, 2, 17
    c, o, cq, oq = _setup(ctxs, oracle_mod, log_n, L, K, mods)
    pool = _pool(oq, 6, batch, 700)
    ia, ib = _pairs(n_terms, 6)
    key = o.fill_uniform(701, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    dpool = [dev(p) for p in pool]
    out = torch.empty((batch, 2, L - K, o.N), dtype=torch.int64, device="cuda")
    c.ct_dot_grouped(K, [dpool[i] for i in ia], [dpool[i] for i in ib], dev(key), out, batch, 65537)
    want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], key, 65537)
    assert np.array_equal(host(out).reshape(want.shape), want)


def test_host_form_launches_scratch_and_checks(ctxs, oracle_mod, dp):
    K, L, log_n, n_terms = 2, 6, 12, 5
    c, o, cq, oq = _setup(ctxs, oracle_mod, log_n, L, K)
    batch = 700   # the host form splits it into several chunks
    a = oq.fill_uniform(800, n_terms * batch * 2).reshape(n_terms, batch, 2, L - K, o.N)
    b = oq.fill_uniform(801, n_terms * batch * 2).reshape(n_terms, batch, 2, L - K, o.N)
    key = o.fill_uniform(802, 2 * o.grouped_digits(K)).reshape(-1, 2, L, o.N)
    da, db, dkey = [dev(x) for x in a], [dev(x) for x in b], dev(key)
    out = torch.full((batch, 2, L - K, o.N), -1, dtype=torch.int64, device="cuda")
    ref = torch.empty_like(out)
    c.ct_mul_relin_grouped(K, da[0], db[0], dkey, ref, batch, 65537)   # reserves what the grouped family reserves
    torch.cuda.synchronize()
    bytes0, n0 = c.device_bytes(), c.launch_count()
    c.ct_dot_grouped(K, da, db, dkey, out, batch, 65537)
    torch.cuda.synchronize()
    assert c.launch_count() - n0 == 2 and c.device_bytes() == bytes0
    h_out = np.zeros((batch, 2, L - K, o.N), dtype=np.uint64)
    c.ct_dot_grouped_host(K, a, b, key, h_out, 65537)
    assert np.array_equal(h_out, host(out).reshape(h_out.shape))
    want = cdr.ct_dot(o, oq, K, [x[:2] for x in a], [x[:2] for x in b], key, 65537)
    assert np.array_equal(h_out[:2], want)
    # rejected calls leave the output untouched
    small = 2
    mark = torch.full((small, 2, L - K, o.N), -7, dtype=torch.int64, device="cuda")
    bad_calls = [
        lambda: c.ct_dot_grouped(K, [], [], dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(K, da[:1] * 65, db[:1] * 65, dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(0, da, db, dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(4, da, db, dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(K, da[:2] + [mark], db[:3], dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(K, da[:3], db[:2] + [mark[1:]], dkey, mark, small, 65537),
        lambda: c.ct_dot_grouped(K, da, db, dkey, mark, small, o.moduli[-1]),
    ]
    for k, call in enumerate(bad_calls):
        with pytest.raises(dp.DpfheError):
            call()
        assert bool((mark == -7).all()), k
    lib = dp.load_library()
    import ctypes as C
    ptrs = (C.c_void_p * 2)(da[0].data_ptr(), None)
    assert lib.dpfhe_ct_dot_grouped(c._h, K, 2, ptrs, ptrs, dkey.data_ptr(), mark.data_ptr(), small, 65537, None) != 0
    assert bool((mark == -7).all())
    c.ct_dot_grouped(K, da, db, dkey, mark, 0, 65537)   # an empty batch is fine and launches nothing
    assert bool((mark == -7).all())


def test_round_numbering_restarts(oracle_mod, monkeypatch):
    """a context whose flag / mailbox round numbers restart every few launches keeps producing the same bits"""
    import deeppowers_b200
    monkeypatch.setenv("DPFHE_EPOCH_LIMIT", "40")
    c = deeppowers_b200.Context(12, 6)
    monkeypatch.delenv("DPFHE_EPOCH_LIMIT")
    o = oracle_mod.Oracle(12, 6)
    oq = oracle_mod.Oracle(12, 4, o.moduli[:4])
    K, batch, n_terms = 2, 9, 3
    pool = _pool(oq, 4, batch, 900)
    ia, ib = _pairs(n_terms, 4)
    key = o.fill_uniform(901, 2 * o.grouped_digits(K)).reshape(-1, 2, 6, o.N)
    want = cdr.ct_dot(o, oq, K, [pool[i] for i in ia], [pool[i] for i in ib], key, 65537)
    dpool, dkey = [dev(p) for p in pool], dev(key)
    out = torch.empty((batch, 2, 4, o.N), dtype=torch.int64, device="cuda")
    for _ in range(6):   # ~10 rounds per launch against a limit of 40
        c.ct_dot_grouped(K, [dpool[i] for i in ia], [dpool[i] for i in ib], dkey, out, batch, 65537)
        assert np.array_equal(host(out).reshape(want.shape), want)
    c.close()


def test_attention_scores_end_to_end(ctxs, oracle_mod):
    """64 ciphertexts Q_d and 64 K_d (int8 components of 8192 query / key pairs in the slots), keys, encryption, decryption and
    decoding on the device: every slot is sum_d q_d k_d exactly"""
    K, L, log_n, t, D = 2, 6, 13, 167772161, 64
    c, o, cq, oq = _setup(ctxs, oracle_mod, log_n, L, K)
    N, Lq = o.N, L - K
    rng = np.random.default_rng(5)
    qv = rng.integers(-128, 128, size=(D, 2, N // 2), dtype=np.int64)
    kv = rng.integers(-128, 128, size=(D, 2, N // 2), dtype=np.int64)
    seed = c.random_seed()
    sk = torch.empty((L, N), dtype=torch.int64, device="cuda")
    c.generate_secret(seed, sk)
    evk = torch.empty((c.grouped_digits(K), 2, L, N), dtype=torch.int64, device="cuda")
    c.generate_relin_key(K, t, sk, c.random_seed(), evk)
    skq = sk[:Lq].contiguous()
    pts = torch.empty((2 * D, Lq, N), dtype=torch.int64, device="cuda")
    cq.bgv_encode(torch.from_numpy(np.concatenate([qv, kv])).cuda(), pts, 2 * D, t)
    cts = torch.empty((2 * D, 2, Lq, N), dtype=torch.int64, device="cuda")
    cq.encrypt(t, skq, c.random_seed(), 0, pts, cts, 2 * D)
    out = torch.empty((1, 2, Lq, N), dtype=torch.int64, device="cuda")
    c.ct_dot_grouped(K, [cts[d:d + 1] for d in range(D)], [cts[D + d:D + d + 1] for d in range(D)], evk, out, 1, t)
    ph = torch.empty((1, Lq, N), dtype=torch.int64, device="cuda")
    cq.decrypt(skq, out, 2, ph, 1)
    slots = torch.empty((1, N), dtype=torch.int64, device="cuda")
    cq.bgv_decode(ph, slots, 1, t)
    want = (qv * kv).sum(axis=0) % t
    assert np.array_equal(host(slots).reshape(want.shape), want.astype(np.uint64))


def test_cpp_example(tmp_path):
    """examples/encrypted_dot_product.cpp against libdpfhe.so alone: compiled with the host compiler, 0 wrong scores"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no host C++ compiler")
    import deeppowers_b200
    deeppowers_b200.load_library()
    libdir = os.path.join(ROOT, "deeppowers_b200")
    exe = str(tmp_path / "encrypted_dot_product")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "encrypted_dot_product.cpp"),
                           "-L", libdir, "-ldpfhe", "-Wl,-rpath," + libdir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 wrong" in r.stdout
