"""The memory contract of the C ABI (include/dpfhe.h), one row per entry point that takes device or host buffers (test
infrastructure).

A row names every buffer of its call, its size as items of `limbs` rows of N words for a case's shape, and its role:
  OPERAND  read only: bit-identical after the call;
  KEY      a switch key, Galois key, secret or public key every work item reads: bit-identical after the call;
  OUTPUT   written, and never read before it is written: pre-filled with all-ones words or with random words, the result is the same;
  INPLACE  read and written (the transforms' data, ct_mul_plain_acc's accumulator).
A buffer with `count` is a host table of device pointers (d_gks, d_cts, d_as / d_bs), one placed buffer per entry, named
"<name>.<i>".  `aliases` lists the exact aliases the header permits, as tuples of buffer names that share one placement.

`run(c, s, p)` makes the call through deeppowers_b200.evaluator on context c (a MultiContext for the dpfhe_multi_* rows) with
the buffers at p[name] (device addresses, or numpy views for host rows); `ref(R, s, x)` computes the expected outputs (and in-place
results) from the inputs x[name], with the reference the call's own test file uses: the oracle R.o of the context, an oracle over
other moduli R.sub(moduli) (the ciphertext moduli, a level's basis), ct_dot_ref, mul_rescale_ref, slot_sum_ref, keys_ref,
public_key_ref, ckks_ref, bgv_ref, polyeval_ref.  `gen` overrides the inputs of a buffer whose words are not residues (slots)."""
import ctypes as C

import numpy as np

import bgv_ref
import ckks_ref
import ct_dot_ref
import keys_ref
import mul_rescale_ref as mrr
import polyeval_ref as pr
import public_key_ref
import slot_sum_ref

OPERAND, KEY, OUTPUT, INPLACE = "operand", "key", "output", "in-place"
T = 65537            # BGV plaintext modulus of the key-switching rows
T_SLOTS = 40961      # a prime below 2^31 that is 1 mod 2N up to N = 16384 (BGV slot encoding)
SEED = bytes(range(32))
SCALE = float(1 << 40)


class Shape:
    """the parameters of one case: context (log_n, L, K special primes), batch, level (None: the top, Lq = L - K) and the counts of
    the calls that take them"""

    def __init__(self, log_n=12, L=2, K=0, batch=1, level=None, n_rot=1, n_terms=1, n_steps=1, n_groups=1, n_comp=2, t=T):
        self.log_n, self.L, self.K, self.batch, self.t = log_n, L, K, batch, t
        self.N = 1 << log_n
        self.Lq = L - K
        self.lv = self.Lq if level is None else level   # limbs of the call's ciphertexts
        self.level = level
        self.n_rot, self.n_terms, self.n_steps, self.n_groups, self.n_comp = n_rot, n_terms, n_steps, n_groups, n_comp
        self.dnum = -(-self.Lq // K) if K else L

    def __repr__(self):
        return "N%d-L%d-K%d-b%d%s" % (self.N, self.L, self.K, self.batch, "" if self.level is None else "-l%d" % self.level)


class Buf:
    def __init__(self, name, role, items, limbs, count=None, host=False):
        self.name, self.role, self.items, self.limbs, self.count, self.host = name, role, items, limbs, count, host

    def words(self, s):
        return self.items(s) * self.limbs(s) * s.N

    def names(self, s):
        return [self.name] if self.count is None else ["%s.%d" % (self.name, i) for i in range(self.count(s))]


class Row:
    def __init__(self, fn, bufs, run, ref, aliases=(), gen=None, multi=False, note=""):
        self.fn, self.bufs, self.run, self.ref = fn, bufs, run, ref
        self.aliases, self.gen, self.multi, self.note = list(aliases), gen or {}, multi, note

    @property
    def host(self):
        return any(b.host for b in self.bufs)

    def outputs(self):
        return [b for b in self.bufs if b.role in (OUTPUT, INPLACE)]


# ---- sizes ----------------------------------------------------------------------------------------------------------------------

ALL = lambda s: s.L                          # every limb of the context
LV = lambda s: s.lv                          # the call's ciphertext limbs
LV1 = lambda s: s.lv - 1                     # one level down (rescale)
ONE = lambda s: 1
BATCH = lambda s: s.batch
CT = lambda s: 2 * s.batch                   # a batch of ciphertexts, as polynomials
PERLIMB_KEY = lambda s: 2 * s.L              # [L][2][L][N]
GROUPED_KEY = lambda s: 2 * s.dnum           # [dnum][2][L][N]


def dev(name, role, items, limbs=LV, count=None):
    return Buf(name, role, items, limbs, count)


def hst(name, role, items, limbs=LV):
    return Buf(name, role, items, limbs, host=True)


# ---- references ---------------------------------------------------------------------------------------------------------------

def cts(x, name, s, limbs=None):
    return x[name].reshape(-1, 2, limbs or s.lv, s.N)


def level_oracle(R, s):
    """the oracle of the call's basis: the context's at the top, {q_0 .. q_{l-1}, p_0 .. p_{K-1}} at level l"""
    if s.level is None or s.level == s.Lq:
        return R.o
    m = list(R.o.moduli)
    return R.sub(m[:s.level] + m[s.Lq:])


def level_key(s, key):
    key = key.reshape(s.dnum, 2, s.L, s.N)
    return key if s.level is None or s.level == s.Lq else pr.restrict_key(key, s.Lq, s.K, s.level)


def q_oracle(R, o, s):
    """the oracle over the ciphertext moduli of oracle o (K special primes last)"""
    return R.sub(list(o.moduli)[:o.L - s.K])


def table(x, name, s, limbs=None):
    n = len([k for k in x if k.startswith(name + ".")])
    return [cts(x, "%s.%d" % (name, i), s, limbs) for i in range(n)]


def gal(s, r):
    """the Galois element of rotation r of a case: rotations by 1, 2, ... slots, the last of several the conjugation"""
    return 2 * s.N - 1 if r == s.n_rot - 1 and s.n_rot > 1 else pow(5, r + 1, 2 * s.N)


def gals(s):
    return [gal(s, r) for r in range(s.n_rot)]


# ---- rows: device buffers -----------------------------------------------------------------------------------------------------

def _elementwise(fn, call, oracle_fn):
    return Row(fn, [dev("a", OPERAND, CT, ALL), dev("b", OPERAND, CT, ALL), dev("out", OUTPUT, CT, ALL)],
               lambda c, s, p: getattr(c, call)(p["a"], p["b"], p["out"], 2 * s.batch),
               lambda R, s, x: {"out": getattr(R.o, oracle_fn)(x["a"], x["b"])},
               aliases=[("out", "a"), ("out", "b"), ("out", "a", "b")])


def _keyswitch_family():
    rows = []
    key = lambda: dev("key", KEY, PERLIMB_KEY, ALL)
    rows.append(Row("dpfhe_keyswitch", [dev("d", OPERAND, BATCH, ALL), key(), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.keyswitch(p["d"], p["key"], p["out"], s.batch),
                    lambda R, s, x: {"out": np.stack([np.stack(R.o.keyswitch(d, x["key"].reshape(s.L, 2, s.L, s.N))) for d in x["d"]])}))
    rows.append(Row("dpfhe_ct_mul_relin", [dev("a", OPERAND, CT, ALL), dev("b", OPERAND, CT, ALL), key(), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.ct_mul_relin(p["a"], p["b"], p["key"], p["out"], s.batch),
                    lambda R, s, x: {"out": R.o.ct_mul_relin(cts(x, "a", s), cts(x, "b", s), x["key"].reshape(s.L, 2, s.L, s.N))}))
    rows.append(Row("dpfhe_rotate", [dev("ct", OPERAND, CT, ALL), key(), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.rotate(p["ct"], gal(s, 0), p["key"], p["out"], s.batch),
                    lambda R, s, x: {"out": R.o.rotate(cts(x, "ct", s), gal(s, 0), x["key"].reshape(s.L, 2, s.L, s.N))}))
    rows.append(Row("dpfhe_rotate_steps", [dev("ct", OPERAND, CT, ALL), key(), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.rotate_steps(p["ct"], -3, p["key"], p["out"], s.batch),
                    lambda R, s, x: {"out": R.o.rotate(cts(x, "ct", s), R.o.galois_elt(-3), x["key"].reshape(s.L, 2, s.L, s.N))}))
    rows.append(Row("dpfhe_rotate_hoisted",
                    [dev("ct", OPERAND, CT, ALL), dev("gks", KEY, PERLIMB_KEY, ALL, count=lambda s: s.n_rot),
                     dev("out", OUTPUT, lambda s: s.n_rot * 2 * s.batch, ALL)],
                    lambda c, s, p: c.rotate_hoisted(p["ct"], gals(s), p["gks"], p["out"], s.batch),
                    lambda R, s, x: {"out": np.stack([R.o.rotate(cts(x, "ct", s), g, k.reshape(s.L, 2, s.L, s.N))
                                                      for g, k in zip(gals(s), table(x, "gks", s))])}))
    return rows


def _grouped_family():
    """the hybrid (K = 1) and grouped calls, their level forms, the hoisted rotations, summed rotations, inner products and
    multiply-and-rescale: keys [dnum][2][L][N], ciphertexts [batch][2][lv][N]"""
    rows = []
    key = lambda: dev("key", KEY, GROUPED_KEY, ALL)

    def mk(fn, bufs, run, ref):
        rows.append(Row(fn, bufs, run, ref))

    for form, K1 in (("hybrid", True), ("grouped", False)):
        ks = (lambda c, s, p: c.keyswitch_hybrid(p["d"], p["key"], p["out"], s.batch, 0)) if K1 else \
             (lambda c, s, p: c.keyswitch_grouped(s.K, p["d"], p["key"], p["out"], s.batch, 0))
        mk("dpfhe_keyswitch_" + form, [dev("d", OPERAND, BATCH), key(), dev("out", OUTPUT, CT)], ks,
           lambda R, s, x: {"out": np.stack([np.stack(R.o.keyswitch_grouped(s.K, d, x["key"].reshape(s.dnum, 2, s.L, s.N), 0))
                                             for d in x["d"]])})
        mul = (lambda c, s, p: c.ct_mul_relin_hybrid(p["a"], p["b"], p["key"], p["out"], s.batch, T)) if K1 else \
              (lambda c, s, p: c.ct_mul_relin_grouped(s.K, p["a"], p["b"], p["key"], p["out"], s.batch, T))
        mk("dpfhe_ct_mul_relin_" + form, [dev("a", OPERAND, CT), dev("b", OPERAND, CT), key(), dev("out", OUTPUT, CT)], mul,
           lambda R, s, x: {"out": R.o.ct_mul_relin_grouped(s.K, cts(x, "a", s), cts(x, "b", s), x["key"].reshape(s.dnum, 2, s.L, s.N), T)})
        rot = (lambda c, s, p: c.rotate_hybrid(p["ct"], gal(s, 0), p["key"], p["out"], s.batch, T)) if K1 else \
              (lambda c, s, p: c.rotate_grouped(s.K, p["ct"], gal(s, 0), p["key"], p["out"], s.batch, T))
        mk("dpfhe_rotate_" + form, [dev("ct", OPERAND, CT), key(), dev("out", OUTPUT, CT)], rot,
           lambda R, s, x: {"out": R.o.rotate_grouped(s.K, cts(x, "ct", s), gal(s, 0), x["key"].reshape(s.dnum, 2, s.L, s.N), T)})

    gks = lambda: dev("gks", KEY, GROUPED_KEY, ALL, count=lambda s: s.n_rot)
    pairs = lambda: [dev("as", OPERAND, CT, count=lambda s: s.n_terms), dev("bs", OPERAND, CT, count=lambda s: s.n_terms)]

    def lv_call(name):   # the level form of a call at s.level, the top-level form otherwise
        return lambda c, s: (getattr(c, name + "_level"), (s.K, s.level)) if s.level is not None else (getattr(c, name), (s.K,))

    for lvl in ("", "_level"):
        def rows_at(lvl=lvl):
            def call(name):
                return lambda c, s: (getattr(c, name + lvl), (s.K, s.lv) if lvl else (s.K,))

            def mul_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": o.ct_mul_relin_grouped(s.K, cts(x, "a", s), cts(x, "b", s), level_key(s, x["key"]), T)}

            def rot_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": o.rotate_grouped(s.K, cts(x, "ct", s), gal(s, 0), level_key(s, x["key"]), T)}

            def hoist_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": o.rotate_hoisted_grouped(s.K, cts(x, "ct", s), gals(s), np.stack([level_key(s, k) for k in table(x, "gks", s, s.L)]), T)}

            def sum_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": slot_sum_ref.rotate_sum(o, s.K, cts(x, "ct", s), gals(s), np.stack([level_key(s, k) for k in table(x, "gks", s, s.L)]), T)}

            def dot_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": ct_dot_ref.ct_dot(o, q_oracle(R, o, s), s.K, table(x, "as", s), table(x, "bs", s), level_key(s, x["key"]), T)}

            def rs_ref(R, s, x):
                o = level_oracle(R, s)
                return {"out": mrr.mul_rescale(o, s.K, table(x, "as", s), table(x, "bs", s), level_key(s, x["key"]), T)}

            def pairs_run(name, single):
                def run(c, s, p):
                    f, head = call(name)(c, s)
                    if single:
                        f(*head, p["as.0"], p["bs.0"], p["key"], p["out"], s.batch, T)
                    else:
                        f(*head, [p["as.%d" % i] for i in range(s.n_terms)], [p["bs.%d" % i] for i in range(s.n_terms)], p["key"], p["out"], s.batch, T)
                return run

            if lvl:
                mk("dpfhe_ct_mul_relin_grouped_level", [dev("a", OPERAND, CT), dev("b", OPERAND, CT), key(), dev("out", OUTPUT, CT)],
                   lambda c, s, p: c.ct_mul_relin_grouped_level(s.K, s.lv, p["a"], p["b"], p["key"], p["out"], s.batch, T), mul_ref)
                mk("dpfhe_rotate_grouped_level", [dev("ct", OPERAND, CT), key(), dev("out", OUTPUT, CT)],
                   lambda c, s, p: c.rotate_grouped_level(s.K, s.lv, p["ct"], gal(s, 0), p["key"], p["out"], s.batch, T), rot_ref)
            mk("dpfhe_rotate_hoisted_grouped" + lvl, [dev("ct", OPERAND, CT), gks(), dev("out", OUTPUT, lambda s: s.n_rot * 2 * s.batch)],
               lambda c, s, p: call("rotate_hoisted_grouped")(c, s)[0](*call("rotate_hoisted_grouped")(c, s)[1], p["ct"], gals(s), p["gks"],
                                                                      p["out"], s.batch, T), hoist_ref)
            mk("dpfhe_rotate_sum_grouped" + lvl, [dev("ct", OPERAND, CT), gks(), dev("out", OUTPUT, CT)],
               lambda c, s, p: call("rotate_sum_grouped")(c, s)[0](*call("rotate_sum_grouped")(c, s)[1], p["ct"], gals(s), p["gks"],
                                                                  p["out"], s.batch, T), sum_ref)
            mk("dpfhe_ct_dot_grouped" + lvl, pairs() + [key(), dev("out", OUTPUT, CT)], pairs_run("ct_dot_grouped", False), dot_ref)
            mk("dpfhe_ct_mul_relin_rescale_grouped" + lvl,
               [dev("as", OPERAND, CT, count=ONE), dev("bs", OPERAND, CT, count=ONE), key(), dev("out", OUTPUT, CT, LV1)],
               pairs_run("ct_mul_relin_rescale_grouped", True), rs_ref)
            mk("dpfhe_ct_dot_rescale_grouped" + lvl, pairs() + [key(), dev("out", OUTPUT, CT, LV1)], pairs_run("ct_dot_rescale_grouped", False),
               rs_ref)
        rows_at()
    return rows


def _plain_rows():
    rows = []
    rows.append(Row("dpfhe_ct_mul_plain", [dev("ct", OPERAND, CT, ALL), dev("pt", OPERAND, ONE, ALL), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.ct_mul_plain(p["ct"], p["pt"], p["out"], s.batch),
                    lambda R, s, x: {"out": R.o.ct_mul_plain(cts(x, "ct", s, s.L), x["pt"][0])}, aliases=[("out", "ct")]))
    rows.append(Row("dpfhe_ct_mul_plain_acc", [dev("ct", OPERAND, CT, ALL), dev("pt", OPERAND, ONE, ALL), dev("acc", INPLACE, CT, ALL)],
                    lambda c, s, p: c.ct_mul_plain_acc(p["ct"], p["pt"], p["acc"], s.batch),
                    lambda R, s, x: {"acc": R.o.poly_add(x["acc"].reshape(-1, s.L, s.N),
                                                         R.o.ct_mul_plain(cts(x, "ct", s, s.L), x["pt"][0]).reshape(-1, s.L, s.N))}))
    rows.append(Row("dpfhe_ct_mul_plain_inner",
                    [dev("steps", OPERAND, lambda s: s.n_steps * 2 * s.batch, ALL), dev("pts", OPERAND, lambda s: s.n_groups * s.n_steps, ALL),
                     dev("out", OUTPUT, lambda s: s.n_groups * 2 * s.batch, ALL)],
                    lambda c, s, p: c.ct_mul_plain_inner(p["steps"], p["pts"], p["out"], s.n_steps, s.n_groups, s.batch),
                    lambda R, s, x: {"out": R.o.ct_mul_plain_inner(x["steps"].reshape(s.n_steps, s.batch, 2, s.L, s.N),
                                                                   x["pts"].reshape(s.n_groups, s.n_steps, s.L, s.N))}))
    rows.append(Row("dpfhe_ct_lincomb", [dev("cts", OPERAND, CT, ALL, count=lambda s: s.n_terms), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.ct_lincomb(p["cts"], COEFFS[:s.n_terms], -7, p["out"], s.batch),
                    lambda R, s, x: {"out": pr.lincomb(R.o.moduli, table(x, "cts", s, s.L), COEFFS[:s.n_terms], -7)},
                    aliases=[("out", "cts.0"), ("out", "cts.1")]))
    rows.append(Row("dpfhe_ct_add_plain", [dev("ct", OPERAND, CT, ALL), dev("pt", OPERAND, ONE, ALL), dev("out", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.ct_add_plain(p["ct"], p["pt"], p["out"], s.batch),
                    lambda R, s, x: {"out": pr.lincomb(R.o.moduli, [cts(x, "ct", s, s.L)], [1], 0, x["pt"][0])}, aliases=[("out", "ct")]))
    rows.append(Row("dpfhe_mod_switch_down", [dev("in", OPERAND, CT, ALL), dev("out", OUTPUT, CT, lambda s: s.L - 1)],
                    lambda c, s, p: c.mod_switch_down(p["in"], p["out"], 2 * s.batch, T),
                    lambda R, s, x: {"out": R.o.mod_switch_down(x["in"], T)}))
    rows.append(Row("dpfhe_mod_down_special", [dev("in", OPERAND, CT, ALL), dev("out", OUTPUT, CT, lambda s: s.L - s.K)],
                    lambda c, s, p: c.mod_down_special(s.K, p["in"], p["out"], 2 * s.batch, T),
                    lambda R, s, x: {"out": R.o.mod_down_special(s.K, x["in"], T)}))
    rows.append(Row("dpfhe_ntt_fwd", [dev("data", INPLACE, CT, ALL)], lambda c, s, p: c.ntt_fwd(p["data"], 2 * s.batch),
                    lambda R, s, x: {"data": R.o.ntt_fwd(x["data"])}))
    rows.append(Row("dpfhe_ntt_inv", [dev("data", INPLACE, CT, ALL)], lambda c, s, p: c.ntt_inv(p["data"], 2 * s.batch),
                    lambda R, s, x: {"data": R.o.ntt_inv(x["data"])}))
    rows.append(Row("dpfhe_ct_tensor", [dev("a", OPERAND, CT, ALL), dev("b", OPERAND, CT, ALL), dev("d", OUTPUT, lambda s: 3 * s.batch, ALL)],
                    lambda c, s, p: c.ct_tensor(p["a"], p["b"], p["d"], s.batch),
                    lambda R, s, x: {"d": R.o.ct_tensor(cts(x, "a", s, s.L), cts(x, "b", s, s.L))}))
    rows.append(Row("dpfhe_fill_uniform", [dev("data", OUTPUT, CT, ALL)], lambda c, s, p: c.fill_uniform(99, p["data"], 2 * s.batch, 5),
                    lambda R, s, x: {"data": R.o.fill_uniform(99, 2 * s.batch, 5)}))
    return rows


COEFFS = [3, -1, 1 << 40, -(1 << 62), 0, 12345]


def _key_rows():
    """key generation, encryption and decryption (t = 65537, a uniform-residue secret: the generators read it as given)"""
    rows = []
    sk = lambda: dev("sk", KEY, ONE, ALL)
    rows.append(Row("dpfhe_secret_keygen", [dev("sk", OUTPUT, ONE, ALL)], lambda c, s, p: c.generate_secret(SEED, p["sk"]),
                    lambda R, s, x: {"sk": keys_ref.secret(R.o, SEED)}))
    rows.append(Row("dpfhe_relin_keygen", [sk(), dev("key", OUTPUT, lambda s: 2 * (s.dnum if s.K else s.L), ALL)],
                    lambda c, s, p: c.generate_relin_key(s.K, T, p["sk"], SEED, p["key"]),
                    lambda R, s, x: {"key": keys_ref.relin_key(R.o, s.K, T, x["sk"][0], SEED)}))
    rows.append(Row("dpfhe_galois_keygen", [sk(), dev("keys", OUTPUT, lambda s: s.n_rot * 2 * (s.dnum if s.K else s.L), ALL)],
                    lambda c, s, p: c.generate_galois_keys(s.K, T, p["sk"], gals(s), SEED, p["keys"]),
                    lambda R, s, x: {"keys": keys_ref.galois_keys(R.o, s.K, T, x["sk"][0], SEED, gals(s))}))
    rows.append(Row("dpfhe_encrypt", [sk(), dev("pt", OPERAND, BATCH, ALL), dev("ct", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.encrypt(T, p["sk"], SEED, 11, p["pt"], p["ct"], s.batch),
                    lambda R, s, x: {"ct": keys_ref.encrypt(R.o, T, x["sk"][0], SEED, 11, x["pt"])}))
    rows.append(Row("dpfhe_decrypt", [sk(), dev("ct", OPERAND, lambda s: s.n_comp * s.batch, ALL), dev("pt", OUTPUT, BATCH, ALL)],
                    lambda c, s, p: c.decrypt(p["sk"], p["ct"], s.n_comp, p["pt"], s.batch),
                    lambda R, s, x: {"pt": keys_ref.decrypt(R.o, x["sk"][0], x["ct"].reshape(s.batch, s.n_comp, s.L, s.N))}))
    rows.append(Row("dpfhe_public_keygen", [sk(), dev("pk", OUTPUT, lambda s: 2, ALL)], lambda c, s, p: c.public_keygen(T, p["sk"], SEED, p["pk"]),
                    lambda R, s, x: {"pk": public_key_ref.public_keygen(R.o, T, x["sk"][0], SEED)}))
    rows.append(Row("dpfhe_encrypt_public", [dev("pk", KEY, lambda s: 2, ALL), dev("pt", OPERAND, BATCH, ALL), dev("ct", OUTPUT, CT, ALL)],
                    lambda c, s, p: c.encrypt_public(T, p["pk"], SEED, 3, p["pt"], p["ct"], s.batch),
                    lambda R, s, x: {"ct": public_key_ref.encrypt_public(R.o, T, x["pk"].reshape(2, s.L, s.N), SEED, 3, x["pt"])}))
    return rows


# slot buffers: N words per vector (N/2 complex doubles, or [2][N/2] int64 BGV slots)
SLOTS = lambda s: s.batch


def ckks_slots(s, rng):
    z = rng.uniform(-1, 1, s.batch * s.N).astype(np.float64)
    return z.view(np.uint64).reshape(s.batch, 1, s.N)


def bgv_slots(s, rng):
    return rng.integers(-(1 << 40), 1 << 40, size=(s.batch, 1, s.N), dtype=np.int64).view(np.uint64)


def _encoder_rows():
    rows = []
    rows.append(Row("dpfhe_ckks_encode", [dev("slots", OPERAND, SLOTS, ONE), dev("pt", OUTPUT, BATCH, ALL)],
                    lambda c, s, p: c._chk(c._l.dpfhe_ckks_encode(c._h, C.c_void_p(p["slots"]), C.c_void_p(p["pt"]), s.batch, SCALE, _stream())),
                    lambda R, s, x: {"pt": ckks_ref.encode(R.o, x["slots"].view(np.complex128).reshape(s.batch, s.N // 2), SCALE)},
                    gen={"slots": ckks_slots}))
    rows.append(Row("dpfhe_ckks_decode", [dev("pt", OPERAND, BATCH, ALL), dev("slots", OUTPUT, SLOTS, ONE)],
                    lambda c, s, p: c._chk(c._l.dpfhe_ckks_decode(c._h, C.c_void_p(p["pt"]), C.c_void_p(p["slots"]), s.batch, SCALE, _stream())),
                    lambda R, s, x: {"slots": ckks_ref.decode(R.o, x["pt"], SCALE).view(np.uint64)}))
    rows.append(Row("dpfhe_bgv_encode", [dev("slots", OPERAND, SLOTS, ONE), dev("pt", OUTPUT, BATCH, ALL)],
                    lambda c, s, p: c.bgv_encode(p["slots"], p["pt"], s.batch, T_SLOTS),
                    lambda R, s, x: {"pt": bgv_ref.encode(R.o, x["slots"].view(np.int64).reshape(s.batch, 2, s.N // 2), T_SLOTS)},
                    gen={"slots": bgv_slots}))
    rows.append(Row("dpfhe_bgv_decode", [dev("pt", OPERAND, BATCH, ALL), dev("slots", OUTPUT, SLOTS, ONE)],
                    lambda c, s, p: c.bgv_decode(p["pt"], p["slots"], s.batch, T_SLOTS),
                    lambda R, s, x: {"slots": bgv_ref.decode(R.o, x["pt"], T_SLOTS)}))
    return rows


def _stream():
    import torch
    h = torch.cuda.current_stream().cuda_stream
    return C.c_void_p(h if h else 1)


# ---- rows: host buffers ---------------------------------------------------------------------------------------------------------
# A host form takes the buffers of its device form as host arrays (tables of device pointers become one array [n][...]) and gives
# the same result; the batch is pipelined in chunks.

def _host_rows(device):
    rows = []

    def like(fn, dev_fn, run, bufs=None, ref=None, gen=None):
        d = device[dev_fn]
        hb = bufs or [Buf(b.name, b.role, b.items, b.limbs, host=True) for b in d.bufs]
        rows.append(Row(fn, hb, run, ref or d.ref, gen=gen or d.gen))

    like("dpfhe_ntt_fwd_host", "dpfhe_ntt_fwd", lambda c, s, p: c.ntt_fwd_host(p["data"]))
    like("dpfhe_ntt_inv_host", "dpfhe_ntt_inv", lambda c, s, p: c.ntt_inv_host(p["data"]))
    like("dpfhe_ct_mul_relin_host", "dpfhe_ct_mul_relin", lambda c, s, p: c.ct_mul_relin_host(p["a"], p["b"], p["key"], p["out"]))
    like("dpfhe_ct_mul_plain_host", "dpfhe_ct_mul_plain", lambda c, s, p: c.ct_mul_plain_host(p["ct"], p["pt"], p["out"]))
    like("dpfhe_rotate_host", "dpfhe_rotate", lambda c, s, p: c.rotate_host(p["ct"], gal(s, 0), p["key"], p["out"]))
    like("dpfhe_ct_add_plain_host", "dpfhe_ct_add_plain", lambda c, s, p: c.ct_add_plain_host(p["ct"], p["pt"], p["out"]))
    like("dpfhe_mod_switch_down_host", "dpfhe_mod_switch_down", lambda c, s, p: c.mod_switch_down_host(p["in"], p["out"], T))
    like("dpfhe_mod_down_special_host", "dpfhe_mod_down_special", lambda c, s, p: c.mod_down_special_host(s.K, p["in"], p["out"], T))
    like("dpfhe_ct_mul_relin_hybrid_host", "dpfhe_ct_mul_relin_hybrid", lambda c, s, p: c.ct_mul_relin_hybrid_host(p["a"], p["b"], p["key"], p["out"], T))
    like("dpfhe_rotate_hybrid_host", "dpfhe_rotate_hybrid", lambda c, s, p: c.rotate_hybrid_host(p["ct"], gal(s, 0), p["key"], p["out"], T))
    like("dpfhe_ct_mul_relin_grouped_host", "dpfhe_ct_mul_relin_grouped",
         lambda c, s, p: c.ct_mul_relin_grouped_host(s.K, p["a"], p["b"], p["key"], p["out"], T))
    like("dpfhe_rotate_grouped_host", "dpfhe_rotate_grouped", lambda c, s, p: c.rotate_grouped_host(s.K, p["ct"], gal(s, 0), p["key"], p["out"], T))

    def unpack(name, s, limbs=None):   # the host array [n][batch][2][lv][N] as the device row's table
        def f(x):
            y = dict(x)
            v = y.pop(name).reshape(-1, s.batch * 2 * (limbs or s.lv) * s.N)
            for i in range(v.shape[0]):
                y["%s.%d" % (name, i)] = v[i]
            return y
        return f

    def via(dev_fn, *names, limbs=None):
        return lambda R, s, x: device[dev_fn].ref(R, s, _chain(x, [unpack(n, s, limbs(s) if limbs else None) for n in names]))

    def terms(p, s, name):   # the host form counts the pairs by the array's first axis
        return p[name].reshape(s.n_terms, -1)

    gks_h = lambda: hst("gks", KEY, lambda s: s.n_rot * 2 * s.dnum, ALL)
    like("dpfhe_rotate_sum_grouped_host", "dpfhe_rotate_sum_grouped",
         lambda c, s, p: c.rotate_sum_grouped_host(s.K, p["ct"], gals(s), p["gks"], p["out"], T),
         bufs=[hst("ct", OPERAND, CT), gks_h(), hst("out", OUTPUT, CT)], ref=via("dpfhe_rotate_sum_grouped", "gks", limbs=ALL))
    pair_h = lambda: [hst("as", OPERAND, lambda s: s.n_terms * 2 * s.batch), hst("bs", OPERAND, lambda s: s.n_terms * 2 * s.batch)]
    key_h = lambda: hst("key", KEY, GROUPED_KEY, ALL)
    like("dpfhe_ct_dot_grouped_host", "dpfhe_ct_dot_grouped", lambda c, s, p: c.ct_dot_grouped_host(s.K, terms(p, s, "as"), terms(p, s, "bs"), p["key"], p["out"], T),
         bufs=pair_h() + [key_h(), hst("out", OUTPUT, CT)], ref=via("dpfhe_ct_dot_grouped", "as", "bs"))
    like("dpfhe_ct_mul_relin_rescale_grouped_host", "dpfhe_ct_mul_relin_rescale_grouped",
         lambda c, s, p: c.ct_mul_relin_rescale_grouped_host(s.K, p["as"], p["bs"], p["key"], p["out"], T),
         bufs=[hst("as", OPERAND, CT), hst("bs", OPERAND, CT), key_h(), hst("out", OUTPUT, CT, LV1)],
         ref=via("dpfhe_ct_mul_relin_rescale_grouped", "as", "bs"))
    like("dpfhe_ct_dot_rescale_grouped_host", "dpfhe_ct_dot_rescale_grouped",
         lambda c, s, p: c.ct_dot_rescale_grouped_host(s.K, terms(p, s, "as"), terms(p, s, "bs"), p["key"], p["out"], T),
         bufs=pair_h() + [key_h(), hst("out", OUTPUT, CT, LV1)], ref=via("dpfhe_ct_dot_rescale_grouped", "as", "bs"))
    like("dpfhe_ct_mul_relin_rescale_grouped_level_host", "dpfhe_ct_mul_relin_rescale_grouped_level",
         lambda c, s, p: c.ct_mul_relin_rescale_grouped_level_host(s.K, s.lv, p["as"], p["bs"], p["key"], p["out"], T),
         bufs=[hst("as", OPERAND, CT), hst("bs", OPERAND, CT), key_h(), hst("out", OUTPUT, CT, LV1)],
         ref=via("dpfhe_ct_mul_relin_rescale_grouped_level", "as", "bs"))
    like("dpfhe_ct_dot_rescale_grouped_level_host", "dpfhe_ct_dot_rescale_grouped_level",
         lambda c, s, p: c.ct_dot_rescale_grouped_level_host(s.K, s.lv, terms(p, s, "as"), terms(p, s, "bs"), p["key"], p["out"], T),
         bufs=pair_h() + [key_h(), hst("out", OUTPUT, CT, LV1)], ref=via("dpfhe_ct_dot_rescale_grouped_level", "as", "bs"))
    like("dpfhe_ckks_encode_host", "dpfhe_ckks_encode", lambda c, s, p: c.ckks_encode_host(p["slots"].view(np.complex128), p["pt"], SCALE))
    like("dpfhe_ckks_decode_host", "dpfhe_ckks_decode", lambda c, s, p: c.ckks_decode_host(p["pt"], p["slots"].view(np.complex128), SCALE))
    like("dpfhe_bgv_encode_host", "dpfhe_bgv_encode", lambda c, s, p: c.bgv_encode_host(p["slots"].view(np.int64), p["pt"], T_SLOTS))
    like("dpfhe_bgv_decode_host", "dpfhe_bgv_decode", lambda c, s, p: c.bgv_decode_host(p["pt"], p["slots"].view(np.int64), T_SLOTS))
    like("dpfhe_secret_keygen_host", "dpfhe_secret_keygen", lambda c, s, p: c.generate_secret_host(SEED, p["sk"]))
    like("dpfhe_relin_keygen_host", "dpfhe_relin_keygen", lambda c, s, p: c.generate_relin_key_host(s.K, T, p["sk"], SEED, p["key"]))
    like("dpfhe_galois_keygen_host", "dpfhe_galois_keygen", lambda c, s, p: c.generate_galois_keys_host(s.K, T, p["sk"], gals(s), SEED, p["keys"]))
    like("dpfhe_encrypt_host", "dpfhe_encrypt", lambda c, s, p: c.encrypt_host(T, p["sk"], SEED, 11, p["pt"], p["ct"]))
    like("dpfhe_decrypt_host", "dpfhe_decrypt", lambda c, s, p: c.decrypt_host(p["sk"], p["ct"], s.n_comp, p["pt"]))
    like("dpfhe_public_keygen_host", "dpfhe_public_keygen", lambda c, s, p: c.public_keygen_host(T, p["sk"], SEED, p["pk"]))
    like("dpfhe_encrypt_public_host", "dpfhe_encrypt_public", lambda c, s, p: c.encrypt_public_host(T, p["pk"], SEED, 3, p["pt"], p["ct"]))
    return rows


def _chain(x, fs):
    for f in fs:
        x = f(x)
    return x


# ---- rows: several GPUs in one process ----------------------------------------------------------------------------------------

def _multi_rows(device):
    rows = []
    d = device["dpfhe_ct_mul_relin"]
    hb = lambda row: [Buf(b.name, b.role, b.items, b.limbs, host=True) for b in row.bufs]
    rows.append(Row("dpfhe_multi_ct_mul_relin_host", hb(d), lambda m, s, p: m.ct_mul_relin_host(p["a"], p["b"], p["key"], p["out"]), d.ref,
                    multi=True))
    g = device["dpfhe_ct_mul_relin_grouped"]
    rows.append(Row("dpfhe_multi_ct_mul_relin_grouped_host", hb(g),
                    lambda m, s, p: m.ct_mul_relin_grouped_host(s.K, p["a"], p["b"], p["key"], p["out"], T), g.ref, multi=True))
    r = device["dpfhe_rotate"]
    rows.append(Row("dpfhe_multi_rotate_host", hb(r), lambda m, s, p: m.rotate_host(p["ct"], gal(s, 0), p["key"], p["out"]), r.ref, multi=True))

    def gather(m, s, p):
        """two shards on the devices of the multi-context; every shard's operands are rows of the placed a and b, the key placed
        once and shared (all shards are on one device when it is listed twice)"""
        ct = 2 * s.L * s.N * 8
        firsts = [m.shard(s.batch, r) for r in range(m.n)]
        m.ct_mul_relin_gather([p["a"] + f * ct for f, _ in firsts], [p["b"] + f * ct for f, _ in firsts], [p["key"]] * m.n, p["out"], 0, s.batch)
    rows.append(Row("dpfhe_multi_ct_mul_relin_gather", list(d.bufs), gather, d.ref, multi=True,
                    note="shards of one device listed twice: the root buffer gathers both"))
    return rows


# ---- rows: library objects ------------------------------------------------------------------------------------------------------
# create: the caller's host arrays (diagonals, keys) are OPERANDs that must stay unchanged; apply / apply_host: the object's
# ciphertexts.  The object rows' run creates the object from the placed host arrays, applies it and closes it.

def _object_rows():
    rows = []
    baby, n_diags = 2, 4

    def linear_ref(R, s, x):
        o = level_oracle(R, s)
        oq = q_oracle(R, o, s) if s.K else o
        ct = cts(x, "ct", s)
        diags = x["diags"].reshape(n_diags, s.lv, s.N)
        if s.K:
            kb = [level_key(s, k) for k in x["gk_baby"].reshape(baby - 1, -1)]
            kg = level_key(s, x["gk_giant"])
            steps = [ct] + list(o.rotate_hoisted_grouped(s.K, ct, [pow(5, b, 2 * s.N) for b in range(1, baby)], np.stack(kb), s.t))
            rot = lambda y: o.rotate_grouped(s.K, y, pow(5, baby, 2 * s.N), kg, s.t)
        else:
            kb = x["gk_baby"].reshape(baby - 1, s.L, 2, s.L, s.N)
            kg = x["gk_giant"].reshape(s.L, 2, s.L, s.N)
            steps = [ct] + [o.rotate(ct, pow(5, b, 2 * s.N), kb[b - 1]) for b in range(1, baby)]
            rot = lambda y: o.rotate(y, pow(5, baby, 2 * s.N), kg)
        giant = n_diags // baby
        inner = oq.ct_mul_plain_inner(np.stack(steps), diags.reshape(giant, baby, s.lv, s.N))
        acc = inner[giant - 1]
        for g in range(giant - 2, -1, -1):
            acc = oq.poly_add(rot(acc), inner[g])
        return {"out": acc}

    def linear_bufs(host_apply):
        bufs = [hst("diags", OPERAND, lambda s: n_diags),
                hst("gk_baby", KEY, lambda s: (baby - 1) * (2 * s.dnum if s.K else 2 * s.L), ALL),
                hst("gk_giant", KEY, lambda s: 2 * s.dnum if s.K else 2 * s.L, ALL)]
        mk = hst if host_apply else dev
        return bufs + [mk("ct", OPERAND, CT), mk("out", OUTPUT, CT)]

    def linear_run(host_apply):
        def run(c, s, p):
            from deeppowers_b200 import LinearLayer
            diags = p["diags"].reshape(n_diags, -1)
            if s.K:
                layer = LinearLayer.grouped(c, s.K, diags, baby, p["gk_baby"], p["gk_giant"], s.t, s.level)
            else:
                layer = LinearLayer(c, diags, baby, p["gk_baby"], p["gk_giant"])
            try:
                layer.apply_host(p["ct"], p["out"]) if host_apply else layer.apply(p["ct"], p["out"], s.batch)
                c.synchronize()
            finally:
                layer.close()
        return run

    for fn, host_apply in (("dpfhe_linear_create", False), ("dpfhe_linear_apply", False), ("dpfhe_linear_apply_host", True),
                           ("dpfhe_linear_create_grouped", False), ("dpfhe_linear_create_grouped_level", False)):
        rows.append(Row(fn, linear_bufs(host_apply), linear_run(host_apply), linear_ref))

    coeffs = [3, 0, 5, 1]

    def polyeval_ref(R, s, x):
        chain = pr.Chain(R.oracle_mod, s.log_n, list(R.o.moduli), s.K)
        return {"out": pr.polyeval(chain, T, coeffs, cts(x, "ct", s), x["key"].reshape(s.dnum, 2, s.L, s.N))}

    def polyeval_run(host_apply):
        def run(c, s, p):
            from deeppowers_b200 import PolyEval
            pe = PolyEval(c, s.K, T, coeffs, p["key"])
            try:
                pe.apply_host(p["ct"], p["out"]) if host_apply else pe.apply(p["ct"], p["out"], s.batch)
                c.synchronize()
            finally:
                pe.close()
        return run

    D = 2   # ceil(log2 3)
    for fn, host_apply in (("dpfhe_polyeval_create_grouped", False), ("dpfhe_polyeval_apply", False), ("dpfhe_polyeval_apply_host", True)):
        mk = hst if host_apply else dev
        rows.append(Row(fn, [hst("key", KEY, GROUPED_KEY, ALL), mk("ct", OPERAND, CT), mk("out", OUTPUT, CT, lambda s: s.Lq - D)],
                        polyeval_run(host_apply), polyeval_ref))

    stride, radices = 1, [3]

    def slotsum_ref(R, s, x):
        o = level_oracle(R, s)
        keys = np.stack([level_key(s, k) for k in x["gks"].reshape(-1, s.dnum * 2 * s.L * s.N)])
        return {"out": slot_sum_ref.slot_sum(o, s.K, cts(x, "ct", s), stride, radices, keys, s.t)}

    def slotsum_run(host_apply):
        def run(c, s, p):
            from deeppowers_b200 import SlotSum
            ss = SlotSum.grouped(c, s.K, stride, radices, p["gks"], s.t, s.level)
            try:
                ss.apply_host(p["ct"], p["out"]) if host_apply else ss.apply(p["ct"], p["out"], s.batch)
                c.synchronize()
            finally:
                ss.close()
        return run

    n_steps = sum(r - 1 for r in radices)
    for fn, host_apply in (("dpfhe_slotsum_create_grouped", False), ("dpfhe_slotsum_apply", False), ("dpfhe_slotsum_apply_host", True),
                           ("dpfhe_slotsum_create_grouped_level", False)):
        mk = hst if host_apply else dev
        rows.append(Row(fn, [hst("gks", KEY, lambda s: n_steps * 2 * s.dnum, ALL), mk("ct", OPERAND, CT), mk("out", OUTPUT, CT)],
                        slotsum_run(host_apply), slotsum_ref))
    return rows


def _ckks_polyeval_row():
    import ckks_polyeval_ref as cpr
    coeffs = [0.5, -0.25, 0.125]

    def ref(R, s, x):
        return {"out": cpr.polyeval(pr.Chain(R.oracle_mod, s.log_n, list(R.o.moduli), s.K), coeffs, SCALE, cts(x, "ct", s),
                                    x["key"].reshape(s.dnum, 2, s.L, s.N), SCALE)}

    def run(c, s, p):
        from deeppowers_b200 import PolyEval
        pe = PolyEval.ckks(c, s.K, coeffs, SCALE, p["key"])
        try:
            pe.apply(p["ct"], p["out"], s.batch)
            c.synchronize()
        finally:
            pe.close()
    return Row("dpfhe_polyeval_create_ckks", [hst("key", KEY, GROUPED_KEY, ALL), dev("ct", OPERAND, CT), dev("out", OUTPUT, CT, lambda s: s.Lq - 2)],
               run, ref)


def build_rows():
    device = {}
    for r in (_keyswitch_family() + _grouped_family() + _plain_rows() + _key_rows() + _encoder_rows()
              + [_elementwise("dpfhe_poly_mul_pointwise", "poly_mul_pointwise", "poly_mul_pointwise"),
                 _elementwise("dpfhe_poly_add", "poly_add", "poly_add")]):
        device[r.fn] = r
    rows = dict(device)
    for r in _host_rows(device) + _multi_rows(device) + _object_rows() + [_ckks_polyeval_row()]:
        rows[r.fn] = r
    return rows


# entry points with a d_ or h_ buffer parameter that take no part in a call's memory contract
EXEMPT = {
    "dpfhe_get_root_powers": "copies a table of the context to the caller; no device buffer",
    "dpfhe_device_alloc": "returns memory; reads and writes none",
    "dpfhe_device_free": "releases memory; reads and writes none",
    "dpfhe_ipc_export": "exports a handle of an allocation; reads and writes none of its words",
    "dpfhe_ipc_close": "unmaps an opened allocation; reads and writes none of its words",
    "dpfhe_ipc_open": "maps another process's allocation; reads and writes none of its words",
}


def header_functions(text):
    """{name: [parameter names]} of every dpfhe_* function declared in the text of dpfhe.h"""
    import re
    body = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    body = re.sub(r"#[^\n]*", " ", body)
    out = {}
    for m in re.finditer(r"\b(dpfhe_\w+)\s*\(([^;{]*?)\)\s*;", body, flags=re.S):
        params = []
        for p in m.group(2).split(","):
            p = p.strip()
            if not p or p == "void":
                continue
            name = re.findall(r"(\w+)\s*(?:\[[^\]]*\])?\s*$", p)
            if name:
                params.append(name[0])
        out[m.group(1)] = params
    return out


def buffer_functions(text):
    """the dpfhe_* functions of the header with a device (d_*) or host (h_*) buffer parameter"""
    return sorted(f for f, ps in header_functions(text).items() if any(p.startswith(("d_", "h_")) for p in ps))
