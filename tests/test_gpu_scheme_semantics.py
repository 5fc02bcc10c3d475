"""What every key-switching call means on the device, with the library's own keys: decrypted slots against tests/scheme_model.py.

Every secret, key and ciphertext comes from the library (dpfhe_secret_keygen, dpfhe_relin_keygen, dpfhe_galois_keygen for per-limb,
hybrid and grouped keys, dpfhe_encrypt and dpfhe_encrypt_public of dpfhe_bgv_encode / dpfhe_ckks_encode plaintexts).  Each case runs
a call, decrypts a few of its ciphertexts through the model, and asserts the BGV slots exactly (or the CKKS slots within the model's
error), the noise at or below the model's analytic bound (printed beside it), and that the library's own dpfhe_decrypt and slot
decoders agree with the model.  The shapes are those where the per-shape code paths differ: N = 4096, 8192 and 16384 (the CTA-pair
geometry), per-limb digits up to 16 limbs, K = 1 ... 4 special primes with and without a ragged last digit, Lq + K = 16 at N = 16384,
the default basis and a generic one, the level views' key shift at their lowest, a middle and their highest level, and batches of
one and of one ciphertext past a full grid round."""
import math

import numpy as np
import pytest

import bases
import scheme_model as sm
from ckks_polyeval_ref import ckks_chain

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SEED = bytes(range(40, 72))
ENC_SEED = bytes(range(90, 122))
T1, T2 = 65537, 167772161
DELTA = 2.0**40


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def past_round(group):
    """one ciphertext past the first full round of a persistent launch of `group` CTAs per ciphertext at the default occupancy (three
    CTAs per SM, DESIGN.md section 4): the last group of the grid carries a ciphertext of the second round"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (3 * sms) // group + 1


def steps_of(n):
    """rotation steps 1, -1, N/4 - 1 and the conjugation (None)"""
    return [1, -1, n // 4 - 1, None]


class Setup:
    """One basis on the device: the top-level context (ciphertext moduli then K special primes), contexts over every ciphertext prefix
    (levels) for encoding, encryption and decryption, the secret, and the model."""

    def __init__(self, dp, oracle_mod, log_n, moduli, K):
        self.dp, self.log_n, self.N, self.K = dp, log_n, 1 << log_n, K
        self.L = len(moduli)
        self.Lq = self.L - K
        self.ctx = dp.Context(log_n, self.L, moduli)
        self.moduli = self.ctx.moduli
        self.qs, self.ps = self.moduli[:self.Lq], self.moduli[self.Lq:]
        self.sk = empty(self.L, self.N)
        self.ctx.generate_secret(SEED, self.sk)
        self.model = sm.Model(oracle_mod, log_n, self.moduli)
        self._lv = {}
        self._keys = {}
        self._pk = {}
        self.index = 0

    def lv(self, ell):
        if ell == self.L:
            return self.ctx
        if ell not in self._lv:
            self._lv[ell] = self.dp.Context(self.log_n, ell, self.moduli[:ell])
        return self._lv[ell]

    def close(self):
        for c in self._lv.values():
            c.close()
        self.ctx.close()

    def galois(self, step):
        return 2 * self.N - 1 if step is None else self.ctx.galois_elt(step)

    def relin_key(self, K, t):
        key = ("relin", K, t)
        if key not in self._keys:
            k = empty(self.ctx.key_digits(K), 2, self.L, self.N)
            self.ctx.generate_relin_key(K, t, self.sk, SEED, k)
            self._keys[key] = k
        return self._keys[key]

    def galois_keys(self, K, t, elts):
        """one dpfhe_galois_keygen call for all elements: a list of [digits][2][L][N] views"""
        key = ("galois", K, t, tuple(elts))
        if key not in self._keys:
            k = empty(len(elts), self.ctx.key_digits(K), 2, self.L, self.N)
            self.ctx.generate_galois_keys(K, t, self.sk, list(elts), SEED, k)
            self._keys[key] = k
        k = self._keys[key]
        return [k[i] for i in range(len(elts))]

    def encrypt(self, ell, pt, t, public=False):
        """ciphertexts [n][2][ell][N] of the plaintexts pt [n][ell][N], each with its own item number"""
        c, n = self.lv(ell), pt.shape[0]
        ct = empty(n, 2, ell, self.N)
        if public:
            if (ell, t) not in self._pk:
                pk = empty(2, ell, self.N)
                c.public_keygen(t, self.sk[:ell].contiguous(), SEED, pk)
                self._pk[(ell, t)] = pk
            c.encrypt_public(t, self._pk[(ell, t)], ENC_SEED, self.index, pt, ct, n)
        else:
            c.encrypt(t, self.sk[:ell].contiguous(), SEED, self.index, pt, ct, n)
        self.index += n
        return ct

    def enc_bgv(self, ell, z, t, n=1, public=False):
        """n encryptions of the BGV slots z [2][N/2] at level ell"""
        c = self.lv(ell)
        zs = dev(np.broadcast_to(np.asarray(z, dtype=np.int64), (n, 2, self.N // 2)))
        pt = empty(n, ell, self.N)
        c.bgv_encode(zs, pt, n, t)
        return self.encrypt(ell, pt, t, public)

    def enc_ckks(self, ell, z, scale, n=1):
        c = self.lv(ell)
        zs = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(z, (n, self.N // 2)))).cuda()
        pt = empty(n, ell, self.N)
        c.ckks_encode(zs, pt, n, scale)
        return self.encrypt(ell, pt, 0)

    def check_bgv(self, ct, want, t, bound, what):
        """ct [2][ell][N] on the device decrypts to the slots `want` with noise at or below `bound` (units of t); the library's own
        decryption and decoding agree"""
        ell = ct.shape[-2]
        got, v, Q = self.model.bgv(host(self.sk), host(ct).reshape(2, ell, self.N), t)
        want = np.asarray(want, dtype=object) % t
        assert np.array_equal(got, want.astype(np.uint64)), "%s: %d of %d slots differ" % (what, int((got != want.astype(np.uint64)).sum()), got.size)
        print("%s: noise 2^%.1f t, bound 2^%.1f t, Q/2t 2^%.1f" % (what, sm.bits(v), sm.bits(bound), sm.bits(Q // (2 * t))))
        assert v <= bound, (what, v, bound)
        assert bound < Q / (2 * t) - 1, (what, "bound beyond the modulus")
        c = self.lv(ell)
        ph, out = empty(1, ell, self.N), empty(1, 2, self.N // 2)
        c.decrypt(self.sk[:ell].contiguous(), ct.reshape(1, 2, ell, self.N).contiguous(), 2, ph, 1)
        c.bgv_decode(ph, out, 1, t)
        assert np.array_equal(host(out)[0], got), what
        return v

    def check_ckks(self, ct, want, scale, slot_bound, what, z_max):
        """ct [2][ell][N] decodes at `scale` within the model's slot error `slot_bound` of the exact slots `want` (largest modulus
        z_max); the library agrees"""
        ell = ct.shape[-2]
        got, X, Q = self.model.ckks(host(self.sk), host(ct).reshape(2, ell, self.N), scale)
        bound = slot_bound + sm.ckks_decode_slack(self.N, z_max)
        err = np.abs(got - want).max()
        print("%s: slot error 2^%.1f, bound 2^%.1f" % (what, sm.bits(err), sm.bits(bound)))
        assert err <= bound, (what, err, bound)
        assert bound < 2.0**-4, (what, "bound too loose to tell a wrong slot from a right one")
        c = self.lv(ell)
        ph = empty(1, ell, self.N)
        c.decrypt(self.sk[:ell].contiguous(), ct.reshape(1, 2, ell, self.N).contiguous(), 2, ph, 1)
        out = torch.empty((1, self.N // 2), dtype=torch.complex128, device="cuda")
        c.ckks_decode(ph, out, 1, scale)
        assert np.abs(out.cpu().numpy()[0] - got).max() <= 2 * sm.ckks_decode_slack(self.N, z_max), what
        return err


@pytest.fixture(scope="module")
def setups(oracle_mod):
    import deeppowers_b200 as dp
    made = {}

    def get(log_n, L, K, basis=None):
        key = (log_n, L, K, basis)
        if key not in made:
            while made:                       # one basis at a time: N = 16384 with 17 keys of 16 limbs is hundreds of MiB
                made.popitem()[1].close()
            torch.cuda.empty_cache()
            if basis == "ckks_chain":
                moduli = ckks_chain(oracle_mod, L - K, K)
            elif basis:
                moduli = bases.catalogue(oracle_mod)[basis][:L]
            else:
                moduli = oracle_mod.Oracle(log_n, L).moduli
            made[key] = Setup(dp, oracle_mod, log_n, moduli, K)
        return made[key]

    yield get
    for s in made.values():
        s.close()


def rng_slots(n, t, seed, count=1):
    r = np.random.default_rng(seed)
    z = r.integers(0, t, (count, 2, n // 2), dtype=np.int64)
    return z[0] if count == 1 else z


# ---- per-limb digits (no special prime): ct_mul_relin, rotate, rotate_hoisted ---------------------------------------------------------

@pytest.mark.parametrize("log_n,L,basis,t", [(12, 2, None, T2), (13, 8, None, T1), (14, 16, None, T1), (12, 6, "gen_mixed", T1)])
def test_per_limb_digits(setups, log_n, L, basis, t):
    s = setups(log_n, L, 0, basis)
    n, c = s.N, s.ctx
    z1, z2 = rng_slots(n, t, 1), rng_slots(n, t, 2)
    ks = sm.ks_bound(n, s.qs, 0)
    v0 = sm.fresh_bound(n)
    B = past_round(L)
    a, b = s.enc_bgv(L, z1, t, B), s.enc_bgv(L, z2, t, B)
    evk = s.relin_key(0, t)
    out = empty(B, 2, L, n)
    c.ct_mul_relin(a, b, evk, out, B)
    for k in (0, B - 1):
        s.check_bgv(out[k], sm.bgv_mul(z1, z2, t), t, sm.mul_bound(n, t, v0, v0, ks), "ct_mul_relin L=%d [%d/%d]" % (L, k, B))
    steps = steps_of(n)
    elts = [s.galois(k) for k in steps]
    gks = s.galois_keys(0, t, elts)
    one = empty(1, 2, L, n)
    for k, g, gk in zip(steps, elts, gks):
        c.rotate(a[:1], g, gk, one, 1)
        s.check_bgv(one[0], sm.bgv_galois(z1, g, n), t, sm.rotate_bound(v0, ks), "rotate L=%d step %s" % (L, k))
    # hoisted: a fresh ciphertext and a trivial one (c1 = 0: every digit zero, the fallback to the ordinary rotation)
    pt = empty(1, L, n)
    s.lv(L).bgv_encode(dev(z2[None]), pt, 1, t)
    pair = torch.cat([a[:1], torch.stack([pt, torch.zeros_like(pt)], dim=1)])
    hout = empty(len(elts), 2, 2, L, n)
    c.rotate_hoisted(pair, elts, gks, hout, 2)
    for r, (k, g) in enumerate(zip(steps, elts)):
        s.check_bgv(hout[r, 0], sm.bgv_galois(z1, g, n), t, sm.rotate_bound(v0, ks), "rotate_hoisted L=%d step %s" % (L, k))
        s.check_bgv(hout[r, 1], sm.bgv_galois(z2, g, n), t, sm.rotate_bound(0, ks), "rotate_hoisted zero digits L=%d step %s" % (L, k))


# ---- one special prime: ct_mul_relin_hybrid, rotate_hybrid -------------------------------------------------------------------------

@pytest.mark.parametrize("log_n,Lq,t", [(12, 4, T1), (14, 15, T2)])
def test_hybrid(setups, log_n, Lq, t):
    s = setups(log_n, Lq + 1, 1)
    n, c = s.N, s.ctx
    z1, z2 = rng_slots(n, t, 3), rng_slots(n, t, 4)
    ks = sm.ks_bound(n, s.qs, 1, s.ps)
    v0 = sm.fresh_bound(n)
    B = past_round(s.L)
    a, b = s.enc_bgv(Lq, z1, t, B), s.enc_bgv(Lq, z2, t, B)
    out = empty(B, 2, Lq, n)
    c.ct_mul_relin_hybrid(a, b, s.relin_key(1, t), out, B, t)
    for k in (0, B - 1):
        s.check_bgv(out[k], sm.bgv_mul(z1, z2, t), t, sm.mul_bound(n, t, v0, v0, ks), "ct_mul_relin_hybrid [%d/%d]" % (k, B))
    steps = steps_of(n)
    elts = [s.galois(k) for k in steps]
    for k, g, gk in zip(steps, elts, s.galois_keys(1, t, elts)):
        c.rotate_hybrid(a[:1], g, gk, out[:1], 1, t)
        s.check_bgv(out[0], sm.bgv_galois(z1, g, n), t, sm.rotate_bound(v0, ks), "rotate_hybrid step %s" % k)


# ---- K special primes: every grouped call at the top level, its level forms, the divisions --------------------------------------------

GROUPED = [(12, 4, 1, None, T1), (13, 15, 1, None, T2), (12, 6, 2, None, T1), (14, 5, 3, None, T1), (13, 12, 4, None, T2),
           (14, 12, 4, None, T1), (12, 6, 4, None, T2), (12, 4, 2, "gen_mixed", T1), (14, 3, 2, "gen_mixed", T2)]


@pytest.mark.parametrize("log_n,Lq,K,basis,t", GROUPED)
def test_grouped_top_level(setups, log_n, Lq, K, basis, t):
    s = setups(log_n, Lq + K, K, basis)
    n, c, qs, ps = s.N, s.ctx, s.qs, s.ps
    public = (log_n, Lq, K) == (12, 6, 2)
    v0 = sm.fresh_bound(n, public)
    ks = sm.ks_bound(n, qs, K, ps)
    zs = rng_slots(n, t, 10 + Lq + K, 4)
    xs = [s.enc_bgv(Lq, z, t, 1, public) for z in zs]
    evk = s.relin_key(K, t)
    tag = "N=%d Lq=%d K=%d%s" % (n, Lq, K, " " + basis if basis else "")
    # ct x ct over one full round and one ciphertext more
    B = past_round(s.L)
    a, b = s.enc_bgv(Lq, zs[0], t, B, public), s.enc_bgv(Lq, zs[1], t, B, public)
    out = empty(B, 2, Lq, n)
    c.ct_mul_relin_grouped(K, a, b, evk, out, B, t)
    want = sm.bgv_mul(zs[0], zs[1], t)
    for k in (0, B - 1):
        s.check_bgv(out[k], want, t, sm.mul_bound(n, t, v0, v0, ks), "ct_mul_relin_grouped %s [%d/%d]" % (tag, k, B))
    # rotations: one, hoisted, summed (1 and 15 rotations, the conjugation among them)
    steps = steps_of(n)
    sum_steps = list(range(1, 15)) + [None]
    all_steps = steps + [k for k in sum_steps if k not in steps]
    elts = [s.galois(k) for k in all_steps]
    gks = dict(zip(all_steps, s.galois_keys(K, t, elts)))
    one = empty(1, 2, Lq, n)
    c.rotate_grouped(K, xs[0], s.galois(-1), gks[-1], one, 1, t)
    s.check_bgv(one[0], sm.bgv_rotate(zs[0], -1), t, sm.rotate_bound(v0, ks), "rotate_grouped %s step -1" % tag)
    hout = empty(len(steps), 1, 2, Lq, n)
    c.rotate_hoisted_grouped(K, xs[0], [s.galois(k) for k in steps], [gks[k] for k in steps], hout, 1, t)
    for r, k in enumerate(steps):
        s.check_bgv(hout[r, 0], sm.bgv_galois(zs[0], s.galois(k), n), t, sm.rotate_bound(v0, ks),
                    "rotate_hoisted_grouped %s step %s" % (tag, k))
    for chosen in ([None], sum_steps):
        c.rotate_sum_grouped(K, xs[1], [s.galois(k) for k in chosen], [gks[k] for k in chosen], one, 1, t)
        want = sum((sm.bgv_galois(zs[1], s.galois(k), n) for k in chosen), np.asarray(zs[1], dtype=object))
        s.check_bgv(one[0], want, t, sm.rotate_sum_bound(n, qs, K, ps, v0, len(chosen)),
                    "rotate_sum_grouped %s %d rotations" % (tag, len(chosen)))
    # inner products of 1, 17 and 64 pairs over four ciphertexts repeated across the pairs
    for n_pairs in (1, 17, 64):
        ia = [i % 4 for i in range(n_pairs)]
        ib = [(3 * i + 1) % 4 for i in range(n_pairs)]
        c.ct_dot_grouped(K, [xs[i] for i in ia], [xs[i] for i in ib], evk, one, 1, t)
        want = sm.bgv_dot([zs[i] for i in ia], [zs[i] for i in ib], t)
        s.check_bgv(one[0], want, t, sm.dot_bound(n, t, [(v0, v0)] * n_pairs, ks), "ct_dot_grouped %s %d pairs" % (tag, n_pairs))
    # multiply-and-rescale: the message times q_last^-1 mod t
    low = empty(1, 2, Lq - 1, n)
    qbar = qs[-1]
    acc = sm.ks_acc_bound(n, qs, K, ps)
    c.ct_mul_relin_rescale_grouped(K, xs[0], xs[1], evk, low, 1, t)
    s.check_bgv(low[0], sm.bgv_scale(sm.bgv_mul(zs[0], zs[1], t), pow(qbar, -1, t), t), t,
                sm.divide_bound(n, sm.tensor_bound(n, t, v0, v0), qbar, K + 1, acc), "ct_mul_relin_rescale_grouped %s" % tag)
    ia, ib = [i % 4 for i in range(17)], [(i + 2) % 4 for i in range(17)]
    c.ct_dot_rescale_grouped(K, [xs[i] for i in ia], [xs[i] for i in ib], evk, low, 1, t)
    want = sm.bgv_scale(sm.bgv_dot([zs[i] for i in ia], [zs[i] for i in ib], t), pow(qbar, -1, t), t)
    s.check_bgv(low[0], want, t, sm.divide_bound(n, 17 * sm.tensor_bound(n, t, v0, v0), qbar, K + 1, acc),
                "ct_dot_rescale_grouped %s 17 pairs" % tag)


def levels_of(Lq, K):
    return sorted({K, (K + Lq) // 2, Lq})


@pytest.mark.parametrize("log_n,Lq,K,basis,t", [(12, 6, 2, None, T1), (14, 5, 3, None, T2), (14, 12, 4, None, T1), (12, 4, 2, "gen_mixed", T2)])
def test_grouped_level_calls(setups, log_n, Lq, K, basis, t):
    """every *_grouped_level call at the lowest (K), a middle and the highest (Lq) level, on the top-level keys read in place"""
    s = setups(log_n, Lq + K, K, basis)
    n, c, ps = s.N, s.ctx, s.ps
    v0 = sm.fresh_bound(n)
    evk = s.relin_key(K, t)
    steps = [1, -1, None]
    gks = dict(zip(steps, s.galois_keys(K, t, [s.galois(k) for k in steps])))
    for ell in levels_of(Lq, K):
        qs = s.moduli[:ell]
        ks = sm.ks_bound(n, qs, K, ps)
        tag = "N=%d Lq=%d K=%d level %d" % (n, Lq, K, ell)
        zs = rng_slots(n, t, 100 + ell, 3)
        xs = [s.enc_bgv(ell, z, t) for z in zs]
        one = empty(1, 2, ell, n)
        c.ct_mul_relin_grouped_level(K, ell, xs[0], xs[1], evk, one, 1, t)
        s.check_bgv(one[0], sm.bgv_mul(zs[0], zs[1], t), t, sm.mul_bound(n, t, v0, v0, ks), "ct_mul_relin_grouped_level " + tag)
        c.rotate_grouped_level(K, ell, xs[0], s.galois(-1), gks[-1], one, 1, t)
        s.check_bgv(one[0], sm.bgv_rotate(zs[0], -1), t, sm.rotate_bound(v0, ks), "rotate_grouped_level " + tag)
        hout = empty(2, 1, 2, ell, n)
        c.rotate_hoisted_grouped_level(K, ell, xs[1], [s.galois(1), s.galois(None)], [gks[1], gks[None]], hout, 1, t)
        s.check_bgv(hout[0, 0], sm.bgv_rotate(zs[1], 1), t, sm.rotate_bound(v0, ks), "rotate_hoisted_grouped_level step 1 " + tag)
        s.check_bgv(hout[1, 0], sm.bgv_conjugate(zs[1]), t, sm.rotate_bound(v0, ks), "rotate_hoisted_grouped_level conj " + tag)
        c.rotate_sum_grouped_level(K, ell, xs[2], [s.galois(k) for k in steps], [gks[k] for k in steps], one, 1, t)
        want = sum((sm.bgv_galois(zs[2], s.galois(k), n) for k in steps), np.asarray(zs[2], dtype=object))
        s.check_bgv(one[0], want, t, sm.rotate_sum_bound(n, qs, K, ps, v0, 3), "rotate_sum_grouped_level " + tag)
        ia, ib = [0, 1, 2, 0, 1], [1, 2, 0, 0, 2]
        c.ct_dot_grouped_level(K, ell, [xs[i] for i in ia], [xs[i] for i in ib], evk, one, 1, t)
        want = sm.bgv_dot([zs[i] for i in ia], [zs[i] for i in ib], t)
        s.check_bgv(one[0], want, t, sm.dot_bound(n, t, [(v0, v0)] * 5, ks), "ct_dot_grouped_level " + tag)
        if ell < 2:
            continue
        low = empty(1, 2, ell - 1, n)
        qbar, acc = qs[-1], sm.ks_acc_bound(n, qs, K, ps)
        f = pow(qbar, -1, t)
        c.ct_mul_relin_rescale_grouped_level(K, ell, xs[0], xs[2], evk, low, 1, t)
        s.check_bgv(low[0], sm.bgv_scale(sm.bgv_mul(zs[0], zs[2], t), f, t), t,
                    sm.divide_bound(n, sm.tensor_bound(n, t, v0, v0), qbar, K + 1, acc), "ct_mul_relin_rescale_grouped_level " + tag)
        c.ct_dot_rescale_grouped_level(K, ell, [xs[i] for i in ia], [xs[i] for i in ib], evk, low, 1, t)
        want = sm.bgv_scale(sm.bgv_dot([zs[i] for i in ia], [zs[i] for i in ib], t), f, t)
        s.check_bgv(low[0], want, t, sm.divide_bound(n, 5 * sm.tensor_bound(n, t, v0, v0), qbar, K + 1, acc),
                    "ct_dot_rescale_grouped_level " + tag)


@pytest.mark.parametrize("log_n,Lq,K,basis", [(12, 6, 2, None), (14, 12, 4, None), (13, 4, 1, "gen_mixed")])
def test_divisions(setups, log_n, Lq, K, basis):
    """mod_switch_down (the last ciphertext modulus) and mod_down_special (the special primes), with t and with t = 0: BGV slots times
    the divisor's inverse mod t, CKKS slots at the scale divided by the divisor"""
    s = setups(log_n, Lq + K, K, basis)
    n, L, qs, ps = s.N, s.L, s.qs, s.ps
    P, qbar = sm.prod(ps), qs[-1]
    tag = "N=%d Lq=%d K=%d" % (n, Lq, K)
    t = T1
    z = rng_slots(n, t, 7)
    v0 = sm.fresh_bound(n)
    x = s.enc_bgv(Lq, z, t)
    low = empty(1, 2, Lq - 1, n)
    s.lv(Lq).mod_switch_down(x, low, 2, t)
    s.check_bgv(low[0], sm.bgv_scale(z, pow(qbar, -1, t), t), t, sm.divide_bound(n, v0, qbar, 1), "mod_switch_down t %s" % tag)
    xt = s.enc_bgv(L, z, t)          # over all L limbs, special primes included
    q_out = empty(1, 2, Lq, n)
    s.ctx.mod_down_special(K, xt, q_out, 2, t)
    s.check_bgv(q_out[0], sm.bgv_scale(z, pow(P, -1, t), t), t, sm.divide_bound(n, v0, P, K), "mod_down_special t %s" % tag)
    r = np.random.default_rng(8)
    zc = r.uniform(-1, 1, n // 2) + 1j * r.uniform(-1, 1, n // 2)
    zmax = math.sqrt(2)
    xc = s.enc_ckks(Lq, zc, DELTA * qbar)
    s.lv(Lq).mod_switch_down(xc, low, 2, 0)
    s.check_ckks(low[0], zc, DELTA, sm.ckks_fresh_slot(n, DELTA * qbar, zmax) + sm.ckks_div_slot(n, 1, DELTA), "mod_switch_down t=0 %s" % tag, 2)
    xc = s.enc_ckks(L, zc, DELTA * P)
    s.ctx.mod_down_special(K, xc, q_out, 2, 0)
    s.check_ckks(q_out[0], zc, DELTA, sm.ckks_fresh_slot(n, DELTA * P, zmax) + sm.ckks_div_slot(n, K, DELTA), "mod_down_special t=0 %s" % tag, 2)


@pytest.mark.parametrize("log_n,Lq,K", [(13, 5, 2), (14, 6, 4), (12, 5, 3)])
def test_ckks_on_the_rescaling_chain(setups, log_n, Lq, K):
    """CKKS at Delta = 2^40 on the chain whose middle primes are about 2^45: multiply-and-rescale (top and level forms), the inner
    product, rotations by 1, -1, N/4 - 1 and the conjugation, and a 15-rotation sum"""
    s = setups(log_n, Lq + K, K, "ckks_chain")
    n, c, qs, ps = s.N, s.ctx, s.qs, s.ps
    tag = "N=%d Lq=%d K=%d" % (n, Lq, K)
    r = np.random.default_rng(log_n + Lq)
    zs = [r.uniform(-1, 1, n // 2) + 1j * r.uniform(-1, 1, n // 2) for _ in range(3)]
    zmax = math.sqrt(2)
    e0 = sm.ckks_fresh_slot(n, DELTA, zmax)
    xs = [s.enc_ckks(Lq, z, DELTA) for z in zs]
    evk = s.relin_key(K, 0)
    acc = sm.ks_acc_bound(n, qs, K, ps)
    e_t = sm.ckks_mul_slot(zmax, e0, zmax, e0)
    qbar = qs[-1]
    sc = DELTA * DELTA / qbar
    low = empty(1, 2, Lq - 1, n)
    c.ct_mul_relin_rescale_grouped(K, xs[0], xs[1], evk, low, 1, 0)
    s.check_ckks(low[0], zs[0] * zs[1], sc, e_t + sm.ckks_ks_slot(n, acc, DELTA * DELTA) + sm.ckks_div_slot(n, K + 1, sc), "ckks ct_mul_relin_rescale_grouped " + tag, 2)
    ia, ib = [0, 1, 2, 0, 1, 2, 0], [1, 2, 0, 0, 1, 2, 2]
    c.ct_dot_rescale_grouped(K, [xs[i] for i in ia], [xs[i] for i in ib], evk, low, 1, 0)
    want = sum(zs[i] * zs[j] for i, j in zip(ia, ib))
    s.check_ckks(low[0], want, sc, 7 * e_t + sm.ckks_ks_slot(n, acc, DELTA * DELTA) + sm.ckks_div_slot(n, K + 1, sc), "ckks ct_dot_rescale_grouped 7 pairs " + tag, 14)
    ell = Lq - 1
    if ell >= K:
        x2 = [s.enc_ckks(ell, z, DELTA) for z in zs[:2]]
        low2 = empty(1, 2, ell - 1, n)
        q2 = qs[ell - 1]
        c.ct_mul_relin_rescale_grouped_level(K, ell, x2[0], x2[1], evk, low2, 1, 0)
        s.check_ckks(low2[0], zs[0] * zs[1], DELTA * DELTA / q2,
                     e_t + sm.ckks_ks_slot(n, sm.ks_acc_bound(n, qs[:ell], K, ps), DELTA * DELTA) + sm.ckks_div_slot(n, K + 1, DELTA * DELTA / q2),
                     "ckks ct_mul_relin_rescale_grouped_level %d %s" % (ell, tag), 2)
    steps = steps_of(n)
    sum_steps = list(range(1, 15)) + [None]
    all_steps = steps + [k for k in sum_steps if k not in steps]
    gks = dict(zip(all_steps, s.galois_keys(K, 0, [s.galois(k) for k in all_steps])))
    ks = sm.ks_bound(n, qs, K, ps)
    hout = empty(len(steps), 1, 2, Lq, n)
    c.rotate_hoisted_grouped(K, xs[2], [s.galois(k) for k in steps], [gks[k] for k in steps], hout, 1, 0)
    for i, k in enumerate(steps):
        s.check_ckks(hout[i, 0], sm.ckks_galois(zs[2], s.galois(k), n), DELTA, e0 + sm.ckks_ks_slot(n, ks, DELTA), "ckks rotate_hoisted_grouped step %s %s" % (k, tag), 2)
    one = empty(1, 2, Lq, n)
    c.rotate_sum_grouped(K, xs[2], [s.galois(k) for k in sum_steps], [gks[k] for k in sum_steps], one, 1, 0)
    want = zs[2] + sum(sm.ckks_galois(zs[2], s.galois(k), n) for k in sum_steps)
    s.check_ckks(one[0], want, DELTA, 16 * e0 + sm.ckks_ks_slot(n, sm.rotate_sum_bound(n, qs, K, ps, 0, 15), DELTA), "ckks rotate_sum_grouped 15 rotations " + tag, 32)


# ---- the library objects at a level below the top -----------------------------------------------------------------------------------

def test_linear_layer_and_slot_sum_below_the_top(setups):
    """LinearLayer.grouped and SlotSum.grouped at level Lq - 1 on the top-level keys: W x mod t and the window sums"""
    import deeppowers_b200 as dp
    log_n, Lq, K, t = 13, 4, 2, T1
    s = setups(log_n, Lq + K, K)
    n, ps = s.N, s.ps
    ell = Lq - 1
    qs = s.moduli[:ell]
    ks = sm.ks_bound(n, qs, K, ps)
    v0 = sm.fresh_bound(n)
    DIM, BABY = 16, 4
    r = np.random.default_rng(12)
    W = r.integers(-8, 9, (DIM, DIM))
    x = r.integers(-8, 9, DIM)
    xs = np.zeros((2, n // 2), dtype=np.int64)
    xs[0, :DIM] = x
    xs[0, DIM:2 * DIM] = x
    ds = np.zeros((DIM, 2, n // 2), dtype=np.int64)
    ar = np.arange(DIM)
    for d in range(DIM):
        ds[d, 0, :DIM] = W[ar, (ar + d) % DIM]
        ds[d] = np.roll(ds[d], (d // BABY) * BABY, axis=1)        # diagonal g baby + b pre-rotated by -g baby
    diags = empty(DIM, ell, n)
    s.lv(ell).bgv_encode(dev(ds), diags, DIM, t)
    keys = s.galois_keys(K, t, [s.galois(b) for b in range(1, BABY + 1)])
    kh = np.stack([host(k) for k in keys])
    layer = dp.LinearLayer.grouped(s.ctx, K, host(diags), BABY, np.ascontiguousarray(kh[:BABY - 1]), np.ascontiguousarray(kh[BABY - 1]), t,
                                   level=ell)
    ct = s.enc_bgv(ell, xs, t)
    out = empty(1, 2, ell, n)
    layer.apply(ct, out, 1)
    layer.close()
    want = np.zeros((2, n // 2), dtype=object)
    want[0, :DIM] = W @ x
    got_noise = s.check_bgv(out[0], want, t, sm.linear_bound(n, t, v0, ks, DIM, DIM // BABY), "LinearLayer.grouped level %d" % ell)
    # a slot sum of 2 x 3 windows of stride 1 on the layer's output
    radices = [2, 3]
    st = dp.slotsum_steps(1, radices)
    skeys = np.stack([host(k) for k in s.galois_keys(K, t, [s.galois(k) for k in st])])
    ss = dp.SlotSum.grouped(s.ctx, K, 1, radices, np.ascontiguousarray(skeys), t, level=ell)
    summed = empty(1, 2, ell, n)
    ss.apply(out, summed, 1)
    ss.close()
    bound = sm.linear_bound(n, t, v0, ks, DIM, DIM // BABY)
    for rdx in radices:
        bound = sm.rotate_sum_bound(n, qs, K, ps, bound, rdx - 1)
    assert got_noise <= bound
    s.check_bgv(summed[0], sm.window_sums(want, 1, 6), t, bound, "SlotSum.grouped level %d radices %s" % (ell, radices))
