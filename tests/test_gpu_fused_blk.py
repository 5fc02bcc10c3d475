"""The fused key switch at N <= 8192 (ks_fused_kernel: one 4096-point block per CTA, CTA pairs at N = 8192, accumulators in shared
memory; DESIGN.md §4.4) on the GPU against the oracle, bit for bit: batches on the boundaries of the persistent grid's groups and
rounds, with the default grid and under DPFHE_KS_OCC=1; L = 1, 2, 4 and 16; N = 4096 and 8192; every mode, the hoisted-rotation
fallback with zero digits, and outputs written through the gather's peer stores."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_gpu_parity import ctxs, dev, dp, edge_polys, host  # noqa: E402,F401  (ctxs and dp are fixtures)


def groups(L, log_n, ctas_per_sm):
    """groups of the persistent grid: 2 CTAs per SM, 2L CTAs per group at N = 8192 (a pair per limb), L at N = 4096"""
    per_group = L * (2 if log_n == 13 else 1)
    return ctas_per_sm * torch.cuda.get_device_properties(0).multi_processor_count // per_group


def mul_inputs(o, batch, seed):
    L = o.L
    a = edge_polys(o, 2 * batch, seed).reshape(batch, 2, L, o.N)
    b = edge_polys(o, 2 * batch, seed + 1)[::-1].copy().reshape(batch, 2, L, o.N)
    key = o.fill_uniform(seed + 2, 2 * L).reshape(L, 2, L, o.N)
    return a, b, key


@pytest.mark.parametrize("log_n", [12, 13])
@pytest.mark.parametrize("rounds,extra", [(1, -1), (1, 0), (1, 1), (2, 0), (2, 1), (3, 1)])
def test_batches_on_group_and_round_boundaries(ctxs, log_n, rounds, extra):
    """G groups in the grid: batch = rounds * G + extra, i.e. 32, 33, 34, 66, 67 and 100 for 33 groups (L = 4 on 132 SMs)"""
    L = 4
    c, o = ctxs(log_n, L)
    batch = rounds * groups(L, log_n, 2) + extra
    a, b, key = mul_inputs(o, batch, 100 + batch)
    out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin(dev(a), dev(b), dev(key), out, batch)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin(a, b, key)), batch


@pytest.mark.parametrize("log_n", [12, 13])
def test_one_cta_per_sm(dp, oracle_mod, monkeypatch, log_n):
    """DPFHE_KS_OCC=1: half the grid, every group over more than three rounds"""
    L = 4
    monkeypatch.setenv("DPFHE_KS_OCC", "1")
    c = dp.Context(log_n, L)
    monkeypatch.delenv("DPFHE_KS_OCC")
    o = oracle_mod.Oracle(log_n, L)
    batch = 3 * groups(L, log_n, 1) + 1
    a, b, key = mul_inputs(o, batch, 7)
    out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin(dev(a), dev(b), dev(key), out, batch)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin(a, b, key))
    c.close()


@pytest.mark.parametrize("log_n", [12, 13])
@pytest.mark.parametrize("L", [1, 2, 4, 16])
def test_every_mode(ctxs, log_n, L):
    """ct x ct, the bare key switch and rotations (one of them the conjugation)"""
    c, o = ctxs(log_n, L)
    batch = 5
    a, b, key = mul_inputs(o, batch, 20 + L)
    out = torch.full(a.shape, -1, dtype=torch.int64, device="cuda")
    c.ct_mul_relin(dev(a), dev(b), dev(key), out, batch)
    assert np.array_equal(host(out).reshape(a.shape), o.ct_mul_relin(a, b, key))
    d = edge_polys(o, batch, 30 + L)
    c.keyswitch(dev(d), dev(key), out, batch)
    ref = np.stack([np.stack(o.keyswitch(d[k], key)) for k in range(batch)])
    assert np.array_equal(host(out).reshape(ref.shape), ref)
    for g in (o.galois_elt(3), 2 * o.N - 1):
        c.rotate(dev(a), g, dev(key), out, batch)
        assert np.array_equal(host(out).reshape(a.shape), o.rotate(a, g, key)), g


@pytest.mark.parametrize("log_n,L", [(12, 4), (13, 4), (13, 2)])
def test_hoisted_rotation_fallback(ctxs, log_n, L):
    """ciphertexts with zero digits take the fused kernel's FILTER instance; the others the hoisted path"""
    c, o = ctxs(log_n, L)
    batch = 2 * groups(L, log_n, 2) + 3
    ct = edge_polys(o, 2 * batch, 91).reshape(batch, 2, L, o.N)
    ct[batch - 1, 1] = 0
    ct[1, 1, L - 1] = 0
    ct[batch // 2, 1, 0] = 0
    galois = [o.galois_elt(1), 2 * o.N - 1]
    keys = [o.fill_uniform(100 + r, 2 * L).reshape(L, 2, L, o.N) for r in range(len(galois))]
    out = torch.full((len(galois), batch, 2, L, o.N), -1, dtype=torch.int64, device="cuda")
    c.rotate_hoisted(dev(ct), galois, [dev(k) for k in keys], out, batch)
    for r, g in enumerate(galois):
        assert np.array_equal(host(out[r]).reshape(ct.shape), o.rotate(ct, g, keys[r])), r


@pytest.mark.parametrize("log_n,L,batch", [(12, 2, 9), (13, 4, 41)])
def test_peer_store_output(dp, oracle_mod, log_n, L, batch):
    """every shard's kernel writes its rows of the result straight into the root device's buffer (logical shards on one GPU,
    real peers where there are several)"""
    o = oracle_mod.Oracle(log_n, L)
    a, b, key = mul_inputs(o, batch, 60)
    want = o.ct_mul_relin(a, b, key)
    n = torch.cuda.device_count()
    devices = [0, 0] if n < 2 else [0, 1]
    m = dp.MultiContext(log_n, L, devices=devices)
    a_sh, b_sh, k_sh = [], [], []
    for r, d in enumerate(devices):
        first, count = m.shard(batch, r)
        a_sh.append(torch.from_numpy(np.ascontiguousarray(a[first:first + count]).view(np.int64)).to("cuda:%d" % d))
        b_sh.append(torch.from_numpy(np.ascontiguousarray(b[first:first + count]).view(np.int64)).to("cuda:%d" % d))
        k_sh.append(torch.from_numpy(np.ascontiguousarray(key).view(np.int64)).to("cuda:%d" % d))
    out_root = torch.zeros((batch, 2, L, o.N), dtype=torch.int64, device="cuda:0")
    for d in set(devices):
        torch.cuda.synchronize(d)
    m.ct_mul_relin_gather(a_sh, b_sh, k_sh, out_root, 0, batch)
    assert np.array_equal(host(out_root), want)
    m.close()
