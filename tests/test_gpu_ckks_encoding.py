"""CKKS slot encoding on the GPU (DESIGN.md section 2.12): bit for bit against its restatement (tests/ckks_ref.c), host forms
against device forms, a full-slot encrypted pipeline, and the C++ wrapper."""
import os
import subprocess

import numpy as np
import pytest

import bases
import ckks_ref

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def _slots(rng, n_vec, n):
    return rng.uniform(-1, 1, (n_vec, n // 2)) + 1j * rng.uniform(-1, 1, (n_vec, n // 2))


# (log_n, L, basis): every ring degree with one limb up to eight (sixteen at N = 4096) on the default basis, and the generic and
# fast six-limb bases of tests/bases.py
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
    for n_vec, scale in ((133, 2.0**40), (1, 2.0**50), (1, 2.0**80)):
        z = _slots(rng, n_vec, n) * 8
        pt = torch.empty((n_vec, L, n), dtype=torch.int64, device="cuda")
        ctx.ckks_encode(torch.from_numpy(z).cuda(), pt, n_vec, scale)
        want = ckks_ref.encode(o, z, scale)
        assert np.array_equal(host(pt), want)
        # decode the restatement's plaintexts and uniform residues (coefficients anywhere in (-Q/2, Q/2])
        for src in (want, o.fill_uniform(5, n_vec)):
            src_d = dev(src)
            before = src_d.clone()
            out = torch.empty((n_vec, n // 2), dtype=torch.complex128, device="cuda")
            ctx.ckks_decode(src_d, out, n_vec, scale)
            assert torch.equal(src_d, before)   # the input plaintexts are const
            ref = ckks_ref.decode(o, src, scale)
            assert np.array_equal(out.cpu().numpy().view(np.uint64), ref.view(np.uint64))
    ctx.close()


def test_host_forms_equal_device_forms(oracle_mod):
    import deeppowers_b200 as dp
    logn, L, n = 14, 8, 1 << 14
    ctx = dp.Context(logn, L)
    n_vec = 300   # more than one pipeline chunk (132-item chunks of 1 MiB plaintexts)
    z = _slots(np.random.default_rng(1), n_vec, n)
    scale = 2.0**45
    pt_h = np.empty((n_vec, L, n), dtype=np.uint64)
    ctx.ckks_encode_host(z, pt_h, scale)
    pt_d = torch.empty((n_vec, L, n), dtype=torch.int64, device="cuda")
    ctx.ckks_encode(torch.from_numpy(z).cuda(), pt_d, n_vec, scale)
    assert np.array_equal(pt_h, host(pt_d))
    z_h = np.empty((n_vec, n // 2), dtype=np.complex128)
    ctx.ckks_decode_host(pt_h, z_h, scale)
    z_d = torch.empty((n_vec, n // 2), dtype=torch.complex128, device="cuda")
    ctx.ckks_decode(pt_d, z_d, n_vec, scale)
    assert np.array_equal(z_h.view(np.uint64), z_d.cpu().numpy().view(np.uint64))
    assert np.abs(z_h - z).max() < 1e-6
    with pytest.raises(dp.DpfheError):
        ctx.ckks_encode_host(z, pt_h, float("inf"))
    with pytest.raises(dp.DpfheError):
        ctx.ckks_decode_host(pt_h, z_h, 0.0)
    ctx.close()


def test_full_slot_pipeline(oracle_mod):
    """all 4096 slots: GPU encode -> encrypt -> hybrid ct x ct (plain rounding) -> rescale -> decrypt with library calls -> GPU decode"""
    import deeppowers_b200 as dp
    logn, n = 13, 8192
    o4 = oracle_mod.Oracle(logn, 4)
    o3 = oracle_mod.Oracle(logn, 3, o4.moduli[:3])
    c4, c3 = dp.Context(logn, 4), dp.Context(logn, 3, o4.moduli[:3])
    c2 = dp.Context(logn, 2, o4.moduli[:2])
    s4 = o4.keygen_secret(5)
    s3, s2 = np.ascontiguousarray(s4[:3]), np.ascontiguousarray(s4[:2])
    rng = np.random.default_rng(12)
    z1, z2 = _slots(rng, 1, n)[0], _slots(rng, 1, n)[0]
    scale = 2.0**50
    pts = torch.empty((2, 3, n), dtype=torch.int64, device="cuda")
    c3.ckks_encode(torch.from_numpy(np.stack([z1, z2])).cuda(), pts, 2, scale)

    def encrypt(pt, seed):
        ct = o3.encrypt(seed, 1, s3, np.zeros(n, dtype=np.uint64))
        ct[0] = o3.poly_add(ct[0][None], pt[None])[0]
        return ct

    def decrypt(ctx, ct, s, L):
        """c0 + c1 s with ct_mul_plain and poly_add"""
        ct_d, prod = dev(ct), torch.empty((1, 2, L, n), dtype=torch.int64, device="cuda")
        ctx.ct_mul_plain(ct_d, dev(s), prod, 1)
        m = torch.empty((L, n), dtype=torch.int64, device="cuda")
        ctx.poly_add(ct_d[0], prod[0, 1], m, 1)
        return m

    pt_h = host(pts)
    ct1, ct2 = encrypt(pt_h[0], 21), encrypt(pt_h[1], 22)
    prod = torch.zeros((1, 2, 3, n), dtype=torch.int64, device="cuda")
    c4.ct_mul_relin_hybrid(dev(ct1[None]), dev(ct2[None]), dev(o4.keygen_relin_hybrid(23, 1, s4)), prod, 1, 0)
    low = torch.zeros((2, 2, n), dtype=torch.int64, device="cuda")
    c3.mod_switch_down(prod, low, 2, 0)
    out = torch.empty((1, n // 2), dtype=torch.complex128, device="cuda")
    c2.ckks_decode(decrypt(c2, host(low).reshape(2, 2, n), s2, 2), out, 1, scale * scale / o3.moduli[2])
    assert np.abs(out.cpu().numpy()[0] - z1 * z2).max() < 1e-5
    for k in (1, 7):
        g = o4.galois_elt(k)
        rot = torch.zeros_like(prod)
        c4.rotate_hybrid(dev(ct1[None]), g, dev(o4.keygen_galois_hybrid(24 + k, 1, s4, g)), rot, 1, 0)
        c3.ckks_decode(decrypt(c3, host(rot).reshape(2, 3, n), s3, 3), out, 1, scale)
        assert np.abs(out.cpu().numpy()[0] - np.roll(z1, -k)).max() < 1e-5
    c4.close()
    c3.close()
    c2.close()


_CPP = r'''
#include <algorithm>
#include <complex>
#include <cstdio>
#include <vector>
#include "deeppowers_fhe.hpp"
int main() {
    deeppowers::api::fhe::EncryptionParameters parms;
    parms.log_n = 13;
    parms.n_limbs = 4;
    deeppowers::api::fhe::Evaluator ev(parms);
    const std::size_t count = 3, slots = ev.slot_count();
    std::vector<std::complex<double>> z(count * slots), back(count * slots);
    for (std::size_t i = 0; i < z.size(); ++i) z[i] = {double(i % 97) / 97.0 - 0.5, double(i % 31) / 31.0};
    std::vector<std::uint64_t> pt(count * ev.poly_words());
    ev.encode_ckks(z.data(), count, 1099511627776.0, pt.data());
    ev.decode_ckks(pt.data(), count, 1099511627776.0, back.data());
    double err = 0;
    for (std::size_t i = 0; i < z.size(); ++i) err = std::max(err, std::abs(back[i] - z[i]));
    std::printf("slots %zu max error %.3e\n", slots, err);
    return err < 1e-7 ? 0 : 1;
}
'''


def test_cpp_wrapper_round_trip(tmp_path):
    import deeppowers_b200
    deeppowers_b200.load_library()
    src, exe = tmp_path / "ckks_round_trip.cpp", str(tmp_path / "ckks_round_trip")
    src.write_text(_CPP)
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib_dir = os.path.join(ROOT, "deeppowers_b200")
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-L", lib_dir, "-ldpfhe",
                           "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "slots 4096" in r.stdout
