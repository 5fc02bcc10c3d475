"""The encrypted linear layer with grouped special-prime keys as a library object (dpfhe_linear_create_grouped, LinearLayer.grouped, the
C++ LinearLayer): bit for bit against the Python composition linear_bsgs_grouped and against the oracle's composition, on the device and
host-buffer forms, with the launch count it promises, and decrypting the 768x768 config-4 layer to W x."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from bases import catalogue  # noqa: E402
from slots import SlotEncoder  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_PLAIN = 167772161      # 5 * 2^25 + 1, as tests/test_gpu_linear_layer.py
DIM = 768


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


class Setup:
    """a grouped layer's inputs: contexts / oracles over all L limbs and over the Lq ciphertext moduli, uniform ciphertexts,
    diagonals and keys (bit-exactness needs no meaning)"""

    def __init__(self, oracle_mod, log_n, Lq, K, baby, giant, batch, moduli=None, seed=1):
        import deeppowers_b200 as dp
        L = Lq + K
        self.o = oracle_mod.Oracle(log_n, L, moduli)
        mods = self.o.moduli
        self.oq = oracle_mod.Oracle(log_n, Lq, mods[:Lq])
        self.ctx, self.ctx_q = dp.Context(log_n, L, mods), dp.Context(log_n, Lq, mods[:Lq])
        self.K, self.Lq, self.L, self.N, self.baby, self.giant, self.batch = K, Lq, L, 1 << log_n, baby, giant, batch
        dnum = self.o.grouped_digits(K)
        self.ct = self.oq.fill_uniform(seed, 2 * batch).reshape(batch, 2, Lq, self.N)
        q = np.array(mods[:Lq], dtype=np.uint64)
        self.ct[0, 1] = (q - 1)[:, None]
        self.diags = self.oq.fill_uniform(seed + 1, baby * giant)
        self.diags[-1] = (q - 1)[:, None]
        self.gk_baby = self.o.fill_uniform(seed + 2, 2 * dnum * max(baby - 1, 1)).reshape(-1, dnum, 2, L, self.N)[:baby - 1]
        self.gk_giant = self.o.fill_uniform(seed + 3, 2 * dnum).reshape(dnum, 2, L, self.N)

    def layer(self, t_plain):
        import deeppowers_b200 as dp
        return dp.LinearLayer.grouped(self.ctx, self.K, self.diags, self.baby, np.ascontiguousarray(self.gk_baby) if self.baby > 1 else None,
                                      self.gk_giant if self.giant > 1 else None, t_plain)

    def python(self, t_plain):
        """linear_bsgs_grouped on the device; returns (result, launches on both contexts)"""
        import deeppowers_b200 as dp
        out = torch.empty((self.batch, 2, self.Lq, self.N), dtype=torch.int64, device="cuda")
        n0, m0 = self.ctx.launch_count(), self.ctx_q.launch_count()
        dp.linear_bsgs_grouped(self.ctx, self.ctx_q, self.K, dev(self.ct), dev(self.diags), [dev(k) for k in self.gk_baby], dev(self.gk_giant),
                               self.baby, out, self.batch, t_plain)
        torch.cuda.synchronize()
        return host(out).reshape(self.ct.shape), self.ctx.launch_count() - n0, self.ctx_q.launch_count() - m0

    def oracle(self, t_plain):
        """the same schedule from oracle calls: hoisted baby steps, inner products over Lq moduli, Horner with rotate_grouped + poly_add"""
        o, oq, K = self.o, self.oq, self.K
        steps = [self.ct]
        if self.baby > 1:
            steps += list(o.rotate_hoisted_grouped(K, self.ct, [o.galois_elt(b) for b in range(1, self.baby)], self.gk_baby, t_plain))
        inner = oq.ct_mul_plain_inner(np.stack(steps), self.diags.reshape(self.giant, self.baby, self.Lq, self.N))
        acc = inner[self.giant - 1]
        for g in range(self.giant - 2, -1, -1):
            acc = oq.poly_add(o.rotate_grouped(K, acc, o.galois_elt(self.baby), self.gk_giant, t_plain), inner[g])
        return acc

    def close(self):
        self.ctx.close()
        self.ctx_q.close()


# (log_n, Lq, K, baby, giant, batch, t_plain, basis)
CASES = [
    (12, 3, 1, 4, 3, 3, 65537, None),
    (12, 4, 2, 3, 4, 3, 0, None),
    (12, 5, 2, 4, 2, 3, 65537, None),        # ragged last digit
    (12, 4, 3, 2, 3, 2, 65537, None),
    (12, 4, 4, 3, 2, 2, 0, None),
    (14, 4, 2, 3, 3, 2, 65537, None),
    (12, 4, 2, 4, 3, 3, 65537, "gen_mixed"),
    (12, 4, 2, 1, 4, 3, 65537, None),        # baby = 1: no baby steps
    (12, 4, 2, 5, 1, 3, 0, None),            # giant = 1: no giant steps
]


@pytest.mark.parametrize("log_n,Lq,K,baby,giant,batch,t,basis", CASES)
def test_layer_is_the_reference_composition(oracle_mod, log_n, Lq, K, baby, giant, batch, t, basis):
    mods = catalogue(oracle_mod)[basis] if basis else None
    s = Setup(oracle_mod, log_n, Lq, K, baby, giant, batch, mods)
    ref, py_ctx, py_ctx_q = s.python(t)
    assert np.array_equal(ref, s.oracle(t))
    bytes_before = s.ctx.device_bytes()
    lay = s.layer(t)
    out = torch.full((batch, 2, Lq, s.N), -1, dtype=torch.int64, device="cuda")
    d_ct = dev(s.ct)
    lay.apply(d_ct, out, batch)                  # first application: sizes the layer's scratch
    n0 = s.ctx.launch_count()
    lay.apply(d_ct, out, batch)
    torch.cuda.synchronize()
    n_layer = s.ctx.launch_count() - n0
    assert np.array_equal(host(out).reshape(ref.shape), ref)
    # launches: [baby > 1] * (1 + 3 (baby - 1)) + (inner-product launches) + (giant - 1); the composition's inner products and adds
    # ran on ctx_q: its count less the giant - 1 adds is the inner-product launches
    pti = py_ctx_q - (giant - 1)
    assert n_layer == (1 + 3 * (baby - 1) if baby > 1 else 0) + pti + (giant - 1)
    assert (py_ctx + py_ctx_q) - n_layer == (baby - 1) + 2 * (giant - 1)   # no companion builds, no separate additions
    # the inner products run on a view of the context: the layer adds nothing to its device memory
    assert s.ctx.device_bytes() == bytes_before
    h_out = np.zeros_like(ref)
    lay.apply_host(s.ct, h_out)
    assert np.array_equal(h_out, ref)
    lay.close()
    s.close()


def test_host_form_over_several_chunks(oracle_mod, monkeypatch):
    """apply_host in chunks of one grid round (DPFHE_LINEAR_CHUNK_ROUNDS=1: num_sms * 3 / L ciphertexts), the last chunk ragged"""
    s = Setup(oracle_mod, 12, 4, 2, 3, 3, 1, seed=11)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    groups = n_sm * 3 // s.L
    batch = 2 * groups + groups // 2 + 1          # two whole chunks and a ragged third
    ct = s.oq.fill_uniform(21, 2 * batch).reshape(batch, 2, s.Lq, s.N)
    lay = s.layer(65537)
    want = torch.empty((batch, 2, s.Lq, s.N), dtype=torch.int64, device="cuda")
    lay.apply(dev(ct), want, batch)
    import deeppowers_b200 as dp
    ref = torch.empty_like(want)
    dp.linear_bsgs_grouped(s.ctx, s.ctx_q, s.K, dev(ct), dev(s.diags), [dev(k) for k in s.gk_baby], dev(s.gk_giant), s.baby, ref, batch, 65537)
    torch.cuda.synchronize()
    assert torch.equal(want, ref)
    want = host(want).reshape(ct.shape)
    for rounds in ("1", "2"):
        monkeypatch.setenv("DPFHE_LINEAR_CHUNK_ROUNDS", rounds)
        out = np.zeros_like(ct)
        lay.apply_host(ct, out)
        assert np.array_equal(out, want), rounds
    # a batch smaller than one chunk, and the first ciphertexts alone: the same rows
    monkeypatch.delenv("DPFHE_LINEAR_CHUNK_ROUNDS")
    few = np.zeros_like(ct[:5])
    lay.apply_host(np.ascontiguousarray(ct[:5]), few)
    assert np.array_equal(few, want[:5])
    lay.close()
    s.close()


def test_invalid_arguments_leave_no_layer(oracle_mod):
    import deeppowers_b200 as dp
    s = Setup(oracle_mod, 12, 4, 2, 2, 2, 2, seed=31)
    lib = s.ctx._l
    hp = lambda a: C.c_void_p(np.ascontiguousarray(a).ctypes.data) if a is not None else None
    kb, kg = np.ascontiguousarray(s.gk_baby), s.gk_giant

    def create(K, n_diags, baby, gk_baby, gk_giant, t):
        h = C.c_void_p(0x1234)
        rc = lib.dpfhe_linear_create_grouped(s.ctx._h, K, hp(s.diags), n_diags, baby, hp(gk_baby), hp(gk_giant), t, C.byref(h))
        return rc, h.value

    special = min(s.o.moduli[s.Lq:])
    for args in [(0, 4, 2, kb, kg, 65537),            # n_special 0
                 (4, 4, 2, kb, kg, 65537),            # more special primes than half the limbs
                 (2, 4, 2, kb, kg, special),          # t_plain at a special prime
                 (2, 4, 2, kb, kg, special + 2),      # and above it
                 (2, 4, 2, None, kg, 65537),          # baby-step keys missing
                 (2, 4, 2, kb, None, 65537),          # giant-step key missing
                 (2, 3, 2, kb, kg, 65537),            # n_diags not a multiple of baby
                 (2, 0, 2, kb, kg, 65537)]:           # no diagonals
        rc, h = create(*args)
        assert rc == -1 and h is None, args        # DPFHE_ERR_INVALID, *out cleared
    lay = s.layer(65537)
    ct = dev(s.ct)
    with pytest.raises(dp.DpfheError, match="overlap"):
        lay.apply(ct, ct, s.batch)
    # an output that starts inside the input's last ciphertext (Lq-limb sizes: L-limb sizes would reach further)
    big = torch.zeros((2 * s.batch, 2, s.Lq, s.N), dtype=torch.int64, device="cuda")
    big[:s.batch].copy_(ct)
    with pytest.raises(dp.DpfheError, match="overlap"):
        lay.apply(big[:s.batch], big[s.batch - 1:2 * s.batch - 1], s.batch)
    out = big[s.batch:]
    lay.apply(big[:s.batch], out, s.batch)      # adjacent, not overlapping: accepted
    ref, _, _ = s.python(65537)
    assert np.array_equal(host(out).reshape(ref.shape), ref)
    lay.close()
    s.close()


def to_rns_eval(o, coeffs_mod_t):
    c = coeffs_mod_t.astype(np.int64)
    c = np.where(c > T_PLAIN // 2, c - T_PLAIN, c)
    limbs = np.stack([(c % q).astype(np.uint64) for q in o.moduli])
    return o.ntt_fwd(limbs[None])[0]


_CPP = r'''
#include <cstdio>
#include <vector>
#include "deeppowers_fhe.hpp"
static std::vector<std::uint64_t> load(const char *path, std::size_t words) {
    std::vector<std::uint64_t> v(words);
    FILE *f = std::fopen(path, "rb");
    if (!f || std::fread(v.data(), 8, words, f) != words) throw std::runtime_error(path);
    std::fclose(f);
    return v;
}
int main(int argc, char **argv) {
    // argv: dir; the layer of the Python test: N = 8192, 4 ciphertext limbs + 2 special primes, 768 diagonals, baby 32
    const std::size_t N = 8192, Lq = 4, K = 2, L = Lq + K, dnum = 2, n = 768, baby = 32, batch = 2;
    const std::string dir = argv[1];
    deeppowers::api::fhe::EncryptionParameters parms;
    parms.log_n = 13;
    parms.n_limbs = L;
    deeppowers::api::fhe::Evaluator ev(parms);
    const std::size_t key = dnum * 2 * L * N, ct = 2 * Lq * N;
    auto diags = load((dir + "/diags.bin").c_str(), n * Lq * N), kb = load((dir + "/baby.bin").c_str(), (baby - 1) * key);
    auto kg = load((dir + "/giant.bin").c_str(), key), in = load((dir + "/ct.bin").c_str(), batch * ct);
    deeppowers::api::fhe::LinearLayer layer(ev, K, diags.data(), n, baby, kb.data(), kg.data(), 167772161ull);
    std::vector<std::uint64_t> out(batch * ct);
    layer.apply(deeppowers::api::fhe::ConstCiphertextBatch(in.data(), batch), deeppowers::api::fhe::CiphertextBatch{out.data(), batch});
    FILE *f = std::fopen((dir + "/out.bin").c_str(), "wb");
    std::fwrite(out.data(), 8, out.size(), f);
    std::fclose(f);
    std::printf("applied %zu ciphertexts\n", batch);
    return 0;
}
'''


def test_768_layer_decrypts_to_w_x(oracle_mod, tmp_path):
    """the layer of test_encrypted_linear_layer_special_prime_keys through the library object and the C++ class: W x exactly"""
    import deeppowers_b200 as dp
    log_n, Lq, K, B, BABY = 13, 4, 2, 2, 32
    L = Lq + K
    o = oracle_mod.Oracle(log_n, L)
    oq = oracle_mod.Oracle(log_n, Lq, o.moduli[:Lq])
    N = o.N
    enc = SlotEncoder(N, T_PLAIN)
    rng = np.random.default_rng(0xD3390046)
    W = rng.integers(-127, 128, (DIM, DIM))
    X = rng.integers(-127, 128, (B, DIM))
    s = o.keygen_secret(1)
    sq = np.ascontiguousarray(s[:Lq])
    cts = []
    for b in range(B):
        slots = np.zeros((2, N // 2), dtype=np.int64)
        slots[0, :DIM] = X[b]
        slots[0, DIM:2 * DIM] = X[b]
        cts.append(oq.encrypt(10 + b, T_PLAIN, sq, enc.encode(slots)))
    ct = np.stack(cts)
    diags = np.empty((DIM, Lq, N), dtype=np.uint64)
    ar = np.arange(DIM)
    for d in range(DIM):
        slots = np.zeros((2, N // 2), dtype=np.int64)
        slots[0, :DIM] = W[ar, (ar + d) % DIM]
        diags[d] = to_rns_eval(oq, enc.encode(np.roll(slots, (d // BABY) * BABY, axis=1)))
    kb = np.stack([o.keygen_galois_grouped(K, 100 + b, T_PLAIN, s, o.galois_elt(b)) for b in range(1, BABY)])
    kg = o.keygen_galois_grouped(K, 3, T_PLAIN, s, o.galois_elt(BABY))

    def check(res):
        for b in range(B):
            y = enc.decode(oq.decrypt(sq, res[b], T_PLAIN))[0, :DIM].astype(np.int64)
            assert np.array_equal(np.where(y > T_PLAIN // 2, y - T_PLAIN, y), W @ X[b])

    ctx, ctx_q = dp.Context(log_n, L), dp.Context(log_n, Lq, o.moduli[:Lq])
    lay = dp.LinearLayer.grouped(ctx, K, diags, BABY, kb, kg, T_PLAIN)
    out = torch.empty((B, 2, Lq, N), dtype=torch.int64, device="cuda")
    lay.apply(dev(ct), out, B)
    res = host(out).reshape(ct.shape)
    check(res)
    ref = torch.empty_like(out)
    dp.linear_bsgs_grouped(ctx, ctx_q, K, dev(ct), dev(diags), [dev(k) for k in kb], dev(kg), BABY, ref, B, T_PLAIN)
    assert torch.equal(out, ref)
    lay.close()
    ctx.close()
    ctx_q.close()
    # the C++ class, host buffers
    for name, arr in (("diags", diags), ("baby", kb), ("giant", kg), ("ct", ct)):
        np.ascontiguousarray(arr).tofile(str(tmp_path / (name + ".bin")))
    src, exe = tmp_path / "linear_grouped.cpp", str(tmp_path / "linear_grouped")
    src.write_text(_CPP)
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib_dir = os.path.join(ROOT, "deeppowers_b200")
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-L", lib_dir, "-ldpfhe",
                           "-Wl,-rpath," + lib_dir, "-o", exe])
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    cpp = np.fromfile(str(tmp_path / "out.bin"), dtype=np.uint64).reshape(ct.shape)
    assert np.array_equal(cpp, res)
    check(cpp)
