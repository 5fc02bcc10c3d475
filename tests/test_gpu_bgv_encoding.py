"""BGV slot encoding on the GPU (DESIGN.md section 2.13): bit for bit against the reference (tests/bgv_ref.py), host forms against
device forms, the table cache under alternating plaintext moduli and streams, config 4's linear layer end to end with diagonals
encoded and results decoded by the library, and the C++ wrapper."""
import os
import subprocess

import numpy as np
import pytest

import bases
import bgv_ref
from bgv_ref import T_VALUES

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_PLAIN = 167772161


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def _slots(rng, n_vec, n):
    return rng.integers(-(2**63), 2**63 - 1, (n_vec, 2, n // 2), dtype=np.int64, endpoint=True)


# every ring degree with one limb up to eight (sixteen at N = 4096) on the default basis, and the generic and fast six-limb
# bases of tests/bases.py
CASES = [(12, 1, None), (12, 4, None), (12, 16, None), (13, 4, None), (13, 8, None), (14, 1, None), (14, 8, None),
         (12, 6, "gen_mixed"), (13, 6, "gen_mixed"), (14, 6, "gen_mixed"), (12, 6, "fast_mixed"), (14, 6, "fast_mixed")]


@pytest.mark.parametrize("logn,L,basis", CASES)
def test_encode_decode_bit_exact(oracle_mod, logn, L, basis):
    import deeppowers_b200 as dp
    n = 1 << logn
    moduli = bases.catalogue(oracle_mod)[basis][:L] if basis else None
    o = oracle_mod.Oracle(logn, L, moduli)
    ctx = dp.Context(logn, L, o.moduli)
    rng = np.random.default_rng(logn * 100 + L)
    for t in T_VALUES:
        z = _slots(rng, 133, n)
        z[1:67] %= 2 * t                              # small values too: both signs of the centred lift in every vector
        z[67:] = rng.integers(-t, t, (66, 2, n // 2))
        pt = torch.empty((133, L, n), dtype=torch.int64, device="cuda")
        ctx.bgv_encode(dev(z), pt, 133, t)
        want = bgv_ref.encode(o, z, t)
        assert np.array_equal(host(pt), want)
        before = pt.clone()
        out = torch.empty((133, 2, n // 2), dtype=torch.int64, device="cuda")
        ctx.bgv_decode(pt, out, 133, t)
        assert torch.equal(pt, before)                # the input plaintexts are const
        assert np.array_equal(host(out), z % t)       # decode(encode(x)) = x mod t
        # one plaintext that is no encoding: uniform residues, centred values anywhere in (-Q/2, Q/2]
        u = o.fill_uniform(5 + t % 7, 1)
        out1 = torch.empty((1, 2, n // 2), dtype=torch.int64, device="cuda")
        ctx.bgv_decode(dev(u), out1, 1, t)
        assert np.array_equal(host(out1), bgv_ref.decode(o, u, t))
    ctx.close()


def test_host_forms_equal_device_forms():
    import deeppowers_b200 as dp
    logn, L, n = 14, 8, 1 << 14
    ctx = dp.Context(logn, L)
    n_vec = 300   # more than one pipeline chunk (132-item chunks of 1 MiB plaintexts)
    z = _slots(np.random.default_rng(1), n_vec, n)
    pt_h = np.empty((n_vec, L, n), dtype=np.uint64)
    ctx.bgv_encode_host(z, pt_h, T_PLAIN)
    pt_d = torch.empty((n_vec, L, n), dtype=torch.int64, device="cuda")
    ctx.bgv_encode(dev(z), pt_d, n_vec, T_PLAIN)
    assert np.array_equal(pt_h, host(pt_d))
    z_h = np.empty((n_vec, 2, n // 2), dtype=np.int64)
    ctx.bgv_decode_host(pt_h, z_h, T_PLAIN)
    z_d = torch.empty((n_vec, 2, n // 2), dtype=torch.int64, device="cuda")
    ctx.bgv_decode(pt_d, z_d, n_vec, T_PLAIN)
    assert np.array_equal(z_h, z_d.cpu().numpy())
    assert np.array_equal(z_h, z % T_PLAIN)
    ctx.close()


def test_argument_errors_and_launch_counts():
    import deeppowers_b200 as dp
    logn, L, n = 12, 2, 1 << 12
    ctx = dp.Context(logn, L)
    z = torch.zeros((2, 2, n // 2), dtype=torch.int64, device="cuda")
    pt = torch.empty((2, L, n), dtype=torch.int64, device="cuda")
    out = torch.empty_like(z)
    n0 = ctx.launch_count()
    ctx.bgv_encode(z, pt, 2, 65537)
    assert ctx.launch_count() - n0 == 2
    ctx.bgv_decode(pt, out, 2, 65537)
    assert ctx.launch_count() - n0 == 4
    ctx.bgv_encode(0, 0, 0, 65537)                    # n_vec = 0: nothing to do, no pointer needed
    ctx.bgv_decode(0, 0, 0, 65537)
    assert ctx.launch_count() - n0 == 4
    for t in (0, 2, 65539, (2 * n + 1) ** 2, 3 * 2**30 + 1, 2**64 - 1):   # not prime, not 1 mod 2N, or not below 2^31
        for call in (lambda: ctx.bgv_encode(z, pt, 2, t), lambda: ctx.bgv_decode(pt, out, 2, t), lambda: ctx.bgv_encode(z, pt, 0, t),
                     lambda: ctx.bgv_encode_host(z.cpu().numpy(), np.empty((2, L, n), dtype=np.uint64), t),
                     lambda: ctx.bgv_decode_host(np.zeros((2, L, n), dtype=np.uint64), np.empty((2, 2, n // 2), dtype=np.int64), t)):
            with pytest.raises(dp.DpfheError):
                call()
    with pytest.raises(dp.DpfheError):
        ctx.bgv_encode(0, pt, 2, 65537)
    with pytest.raises(dp.DpfheError):
        ctx.bgv_decode(pt, 0, 2, 65537)
    assert ctx.launch_count() - n0 == 4
    ctx.close()


def test_plaintext_moduli_alternate_on_two_streams(oracle_mod):
    """the context caches the tables of the last t: alternating two values on two streams replaces them on every call"""
    import deeppowers_b200 as dp
    logn, L, n = 13, 3, 1 << 13
    o = oracle_mod.Oracle(logn, L)
    ctx = dp.Context(logn, L)
    rng = np.random.default_rng(9)
    ts = (T_VALUES[1], T_VALUES[2])
    zs = [_slots(rng, 40, n) for _ in range(4)]
    pts = [torch.empty((40, L, n), dtype=torch.int64, device="cuda") for _ in range(4)]
    outs = [torch.empty((40, 2, n // 2), dtype=torch.int64, device="cuda") for _ in range(4)]
    zd = [dev(z) for z in zs]
    torch.cuda.synchronize()
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    b0 = ctx.device_bytes()
    for k in range(4):
        ctx.bgv_encode(zd[k], pts[k], 40, ts[k % 2], stream=streams[k % 2])
        ctx.bgv_decode(pts[k], outs[k], 40, ts[(k + 1) % 2], stream=streams[(k + 1) % 2])
    ctx.synchronize()
    for k in range(4):
        assert np.array_equal(host(pts[k]), bgv_ref.encode(o, zs[k], ts[k % 2]))
        assert np.array_equal(host(outs[k]), bgv_ref.decode(o, host(pts[k]), ts[(k + 1) % 2]))
    tables = 5 * n * 4                                # the cached tables of one t: twiddle rows and slot positions
    b1 = ctx.device_bytes()
    assert b1 >= b0 + tables
    ctx._chk(ctx._l.dpfhe_context_trim(ctx._h))       # releases the tables and the scratch; they come back on demand
    assert ctx.device_bytes() <= b1 - tables
    ctx.bgv_encode(zd[0], pts[0], 40, ts[0])
    assert np.array_equal(host(pts[0]), bgv_ref.encode(o, zs[0], ts[0]))
    ctx.close()


DIM = 768


def _input_slots(X, n):
    s = np.zeros((X.shape[0], 2, n // 2), dtype=np.int64)
    s[:, 0, :DIM] = X[:, :DIM]
    s[:, 0, DIM:2 * DIM] = X[:, :DIM]
    return s


def _diag_slots(W, baby, n, dim):
    out = np.zeros((dim, 2, n // 2), dtype=np.int64)
    ar = np.arange(dim)
    for d in range(dim):
        out[d, 0, :dim] = W[ar, (ar + d) % dim]
        out[d] = np.roll(out[d], (d // baby) * baby, axis=1)   # D_{g,b} = rot_{-g*baby}(diag_d)
    return out


def _decrypt_decode(ctx, ct, s_dev, B, L, n, t):
    """phase c0 + c1 * s formed on the device, then bgv_decode"""
    ph = torch.empty((B, L, n), dtype=torch.int64, device="cuda")
    for b in range(B):
        ctx.poly_mul_pointwise(ct[b, 1], s_dev, ph[b], 1)
        ctx.poly_add(ct[b, 0], ph[b], ph[b], 1)
    out = torch.empty((B, 2, n // 2), dtype=torch.int64, device="cuda")
    ctx.bgv_decode(ph, out, B, t)
    return out.cpu().numpy()


def test_config4_linear_layer_end_to_end(oracle_mod):
    """768 x 768 int8 layer, N = 8192, L = 4: diagonals encoded on the device, LinearLayer.apply, phase and decode on the device"""
    import deeppowers_b200 as dp
    log_n, L, B, BABY = 13, 4, 2, 32
    o = oracle_mod.Oracle(log_n, L)
    ctx = dp.Context(log_n, L)
    N = o.N
    enc = bgv_ref.encoder(N, T_PLAIN)
    rng = np.random.default_rng(0xD3390004)
    W = rng.integers(-127, 128, (DIM, DIM))
    X = rng.integers(-127, 128, (B, DIM))
    s = o.keygen_secret(1)
    ct = np.stack([o.encrypt(10 + b, T_PLAIN, s, enc.encode(sl)) for b, sl in enumerate(_input_slots(X, N))])
    dslots = _diag_slots(W, BABY, N, DIM)
    diags = torch.empty((DIM, L, N), dtype=torch.int64, device="cuda")
    ctx.bgv_encode(dev(dslots), diags, DIM, T_PLAIN)
    diags_h = host(diags)
    for d in list(range(0, DIM, 37)) + [DIM - 1]:
        assert np.array_equal(diags_h[d], bgv_ref.to_rns_eval(o, enc.encode(dslots[d]), T_PLAIN))
    assert np.array_equal(diags_h, bgv_ref.encode(o, dslots, T_PLAIN))   # all 768, byte for byte
    gk_baby = np.stack([o.keygen_galois(100 + b, T_PLAIN, s, o.galois_elt(b)) for b in range(1, BABY)])
    gk_giant = o.keygen_galois(3, T_PLAIN, s, o.galois_elt(BABY))
    layer = dp.LinearLayer(ctx, np.ascontiguousarray(diags_h), BABY, gk_baby, gk_giant)
    out = torch.empty((B, 2, L, N), dtype=torch.int64, device="cuda")
    layer.apply(dev(ct), out, B)
    y = _decrypt_decode(ctx, out, dev(s), B, L, N, T_PLAIN)[:, 0, :DIM]
    for b in range(B):
        assert np.array_equal(y[b], (W @ X[b]) % T_PLAIN)
    layer.close()
    ctx.close()


def test_grouped_linear_layer_end_to_end(oracle_mod):
    """a 128 x 128 layer through LinearLayer.grouped (N = 4096, 3 ciphertext limbs + 2 special primes), the diagonals encoded by the
    context over the ciphertext moduli"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY, dim = 12, 3, 2, 2, 8, 128
    L = Lq + K
    o = oracle_mod.Oracle(log_n, L)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    ctx, ctx_q = dp.Context(log_n, L), dp.Context(log_n, Lq, o.moduli[:Lq])
    N = o.N
    enc = bgv_ref.encoder(N, T_PLAIN)
    rng = np.random.default_rng(0xD3390045)
    W = rng.integers(-127, 128, (dim, dim))
    X = rng.integers(-127, 128, (B, dim))
    s = o.keygen_secret(1)
    sq = np.ascontiguousarray(s[:Lq])
    xs = np.zeros((B, 2, N // 2), dtype=np.int64)
    xs[:, 0, :dim] = X
    xs[:, 0, dim:2 * dim] = X
    ct = np.stack([oq.encrypt(10 + b, T_PLAIN, sq, enc.encode(xs[b])) for b in range(B)])
    dslots = _diag_slots(W, BABY, N, dim)
    diags = torch.empty((dim, Lq, N), dtype=torch.int64, device="cuda")
    ctx_q.bgv_encode(dev(dslots), diags, dim, T_PLAIN)
    diags_h = np.ascontiguousarray(host(diags))
    assert np.array_equal(diags_h, bgv_ref.encode(oq, dslots, T_PLAIN))
    kb = np.stack([o.keygen_galois_grouped(K, 100 + b, T_PLAIN, s, o.galois_elt(b)) for b in range(1, BABY)])
    kg = o.keygen_galois_grouped(K, 3, T_PLAIN, s, o.galois_elt(BABY))
    lay = dp.LinearLayer.grouped(ctx, K, diags_h, BABY, kb, kg, T_PLAIN)
    out = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    lay.apply(dev(ct), out, B)
    y = _decrypt_decode(ctx_q, out, dev(sq), B, Lq, N, T_PLAIN)[:, 0, :dim]
    for b in range(B):
        assert np.array_equal(y[b], (W @ X[b]) % T_PLAIN)
    lay.close()
    ctx.close()
    ctx_q.close()


_CPP = r'''
#include <cstdio>
#include <vector>
#include "deeppowers_fhe.hpp"
int main() {
    deeppowers::api::fhe::EncryptionParameters parms;
    parms.log_n = 13;
    parms.n_limbs = 4;
    deeppowers::api::fhe::Evaluator ev(parms);
    const std::size_t count = 3, n = ev.poly_degree();
    const std::uint64_t t = 167772161ull;
    std::vector<std::int64_t> z(count * n);
    std::vector<std::uint64_t> back(count * n), pt(count * ev.poly_words());
    for (std::size_t i = 0; i < z.size(); ++i) z[i] = (std::int64_t)(i * 2654435761u % 1000003) - 500000;
    z[0] = INT64_MIN;
    ev.encode_bgv(z.data(), count, t, pt.data());
    ev.decode_bgv(pt.data(), count, t, back.data());
    std::size_t bad = 0;
    for (std::size_t i = 0; i < z.size(); ++i) {
        const std::int64_t r = z[i] % (std::int64_t)t;
        bad += back[i] != (std::uint64_t)(r < 0 ? r + (std::int64_t)t : r);
    }
    std::printf("slots %zu mismatches %zu\n", n, bad);
    return bad == 0 ? 0 : 1;
}
'''


def test_cpp_wrapper_round_trip(tmp_path):
    import deeppowers_b200
    deeppowers_b200.load_library()
    src, exe = tmp_path / "bgv_round_trip.cpp", str(tmp_path / "bgv_round_trip")
    src.write_text(_CPP)
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib_dir = os.path.join(ROOT, "deeppowers_b200")
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-L", lib_dir, "-ldpfhe",
                           "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "slots 8192 mismatches 0" in r.stdout
