"""Seeded call programs on one context (test infrastructure; imports no torch).

`program(seed, shape, n_steps)` draws, from numpy.random.default_rng(seed) alone, a list of steps for one context shape
(log_n, L).  A step is one of:

  call     one row of memory_contract, level_contract, seeded_contract or compact_contract (the dpfhe_multi_* rows excluded) at
           a Shape the context realises, with a batch, a stream (0: torch's legacy default stream, 1: S1, 2: S2), an input seed and
           optionally a chain: one operand is the output of an earlier call of the program with the same words;
  trim     dpfhe_context_trim;
  sync     dpfhe_synchronize;
  create / apply / destroy
           a library object (linear layer, polynomial evaluator or slot sum, top-level or level form) made from one object row,
           applied to device buffers between other steps and destroyed later.

Every program contains, whatever its seed, the transitions that only a sequence of calls on one context can exercise
(`check_guarantees` tells which ones a program lacks):
  growth     each DeviceScratch of the context (SCRATCH) grows straight after a smaller call of another family, and is first
             reused after a trim that released it;
  bgv_t      the BGV tables change their plaintext modulus in both directions while a decode at the old modulus is still queued on
             another stream;
  levels     a level call at every (K, l) the context allows, before and after a trim, each next to a top-level call of the same K;
  keyless    a keyless level call at every l;
  host       a host form between two device calls on two different streams;
  chain      a chained operand on another stream than the step that produced it;
  object     an object applied after a trim and after a scratch was regrown by another family since.

`footprint(steps, shape)` bounds the device memory of a program: its guarded device arena and the context's scratch."""
import numpy as np

import compact_contract
import level_contract
import memory_contract as mc
import seeded_contract

T_PAIR = (65537, 786433)     # two BGV plaintext moduli: primes below 2^31, 1 mod 2N up to N = 2^17
SMS = 132                    # streaming multiprocessors of an H100 SXM: the persistent grid of the round batch
GUARD_MIN = 8192             # guard words around every buffer, as tests/test_gpu_memory_contract.py places them
BUDGET = 4 << 30             # device bytes of one program
SCRATCH = ("ms_tau", "hoist_U", "hoist_zero", "hoistg", "enc_work", "compact_work", "stage_in", "stage_out", "stage_key")


def all_rows():
    """{fn: Row} of the four contract tables, without the rows of several GPUs"""
    rows = {}
    for table in (mc.build_rows(), level_contract.build_rows(), seeded_contract.build_rows(), compact_contract.build_rows()):
        rows.update({fn: r for fn, r in table.items() if not r.multi})
    return rows


ROWS = all_rows()

KS_PERLIMB = ["dpfhe_keyswitch", "dpfhe_ct_mul_relin", "dpfhe_rotate", "dpfhe_rotate_steps", "dpfhe_rotate_hoisted"]
KS_HYBRID = ["dpfhe_keyswitch_hybrid", "dpfhe_ct_mul_relin_hybrid", "dpfhe_rotate_hybrid"]
KS_GROUPED = ["dpfhe_keyswitch_grouped", "dpfhe_ct_mul_relin_grouped", "dpfhe_rotate_grouped", "dpfhe_rotate_hoisted_grouped",
              "dpfhe_rotate_sum_grouped", "dpfhe_ct_dot_grouped", "dpfhe_ct_mul_relin_rescale_grouped", "dpfhe_ct_dot_rescale_grouped"]
KS_LEVEL = ["dpfhe_ct_mul_relin_grouped_level", "dpfhe_rotate_grouped_level", "dpfhe_rotate_hoisted_grouped_level",
            "dpfhe_rotate_sum_grouped_level", "dpfhe_ct_dot_grouped_level", "dpfhe_ct_mul_relin_rescale_grouped_level",
            "dpfhe_ct_dot_rescale_grouped_level"]
PLAIN = ["dpfhe_ct_mul_plain", "dpfhe_ct_mul_plain_acc", "dpfhe_ct_mul_plain_inner", "dpfhe_ct_lincomb", "dpfhe_ct_add_plain",
         "dpfhe_mod_switch_down", "dpfhe_ntt_fwd", "dpfhe_ntt_inv", "dpfhe_ct_tensor", "dpfhe_fill_uniform", "dpfhe_poly_mul_pointwise",
         "dpfhe_poly_add"]
KEYS = ["dpfhe_secret_keygen", "dpfhe_relin_keygen", "dpfhe_galois_keygen", "dpfhe_encrypt", "dpfhe_decrypt", "dpfhe_public_keygen",
        "dpfhe_encrypt_public"]
ENCODERS = ["dpfhe_ckks_encode", "dpfhe_ckks_decode"]
BGV_SLOTS = ["dpfhe_bgv_encode", "dpfhe_bgv_decode"]          # at mc.T_SLOTS, a modulus of N = 4096 only
KEYLESS = [fn for fn, r in level_contract.build_rows().items() if not fn.startswith("dpfhe_polyeval")]
SEEDED = list(seeded_contract.build_rows())
COMPACT = list(compact_contract.build_rows())
HOST_KS = ["dpfhe_ct_mul_relin_host", "dpfhe_rotate_host", "dpfhe_ct_mul_relin_hybrid_host", "dpfhe_rotate_hybrid_host",
           "dpfhe_ct_mul_relin_grouped_host", "dpfhe_rotate_grouped_host", "dpfhe_rotate_sum_grouped_host", "dpfhe_ct_dot_grouped_host",
           "dpfhe_ct_mul_relin_rescale_grouped_host", "dpfhe_ct_dot_rescale_grouped_host",
           "dpfhe_ct_mul_relin_rescale_grouped_level_host", "dpfhe_ct_dot_rescale_grouped_level_host"]
HOST_OTHER = ["dpfhe_ntt_fwd_host", "dpfhe_ntt_inv_host", "dpfhe_ct_mul_plain_host", "dpfhe_ct_add_plain_host", "dpfhe_mod_switch_down_host",
              "dpfhe_mod_down_special_host", "dpfhe_ckks_encode_host", "dpfhe_ckks_decode_host", "dpfhe_encrypt_host", "dpfhe_decrypt_host",
              "dpfhe_encrypt_public_host", "dpfhe_relin_keygen_host", "dpfhe_galois_keygen_host", "dpfhe_public_keygen_host"]
OBJECTS = ["dpfhe_linear_create_grouped", "dpfhe_linear_create_grouped_level", "dpfhe_slotsum_create_grouped",
           "dpfhe_slotsum_create_grouped_level", "dpfhe_polyeval_create_grouped", "dpfhe_polyeval_create_grouped_level"]


class Step:
    """one step; `kw` are the Shape's parameters besides the context's (K, level, batch, t, n_rot, n_terms)"""

    def __init__(self, kind, fn=None, kw=None, stream=0, seed=0, chain=None, obj=None):
        self.kind, self.fn, self.kw, self.stream, self.seed, self.chain, self.obj = kind, fn, dict(kw or {}), stream, seed, chain, obj

    def shape(self, log_n, L, sms=SMS):
        kw = dict(self.kw)
        if kw.get("batch") == "round":
            kw["batch"] = round_batch(L, kw.get("K", 0), kw.get("level"), sms)
        return mc.Shape(log_n, L, kw.get("K", 0), kw.get("batch", 1), kw.get("level"), n_rot=kw.get("n_rot", 2),
                        n_terms=kw.get("n_terms", 2), t=kw.get("t", mc.T))

    def key(self):
        return (self.kind, self.fn, tuple(sorted(self.kw.items())), self.stream, self.seed, self.chain, self.obj)

    def __repr__(self):
        bits = [self.kind] + ([self.fn] if self.fn else []) + ["%s=%s" % kv for kv in sorted(self.kw.items())]
        if self.kind in ("call", "apply"):
            bits.append("stream=%s" % ("legacy", "S1", "S2")[self.stream])
        if self.chain:
            bits.append("chain=%s" % (self.chain,))
        if self.obj is not None:
            bits.append("obj=%d" % self.obj)
        return "<" + " ".join(bits) + ">"


def round_batch(L, K, level, sms=SMS):
    """one ciphertext past a full round of the persistent grid (tests/test_gpu_ks_16384.grid, uncapped): groups of the call's basis"""
    group = (L - K if level is None else level) + K
    G = min(3 * sms, 4 * sms) // group * group
    return G // group + 1


def family(fn):
    """the entry point without its host and level suffixes: calls of two families run different code on the same scratch"""
    for suf in ("_level_host", "_host", "_level"):
        if fn.endswith(suf):
            return fn[:-len(suf)]
    return fn


def valid_levels(L, K):
    """the levels of the level calls with K special primes below the top: K <= l < L - K (2K <= L)"""
    return list(range(K, L - K)) if 2 * K <= L else []


def level_pairs(L):
    return [(K, l) for K in (1, 2, 3) for l in valid_levels(L, K)]


def host_chunk(item_bytes, n_items, sms=SMS):
    """the items of one host-pipeline chunk (deeppowers_b200/csrc/abi.cu pick_chunk)"""
    c = max(1, (64 << 20) // item_bytes)
    if c < sms <= n_items:
        c = sms
    return min(c, n_items)


def short_chunk_batch(log_n, L):
    """a batch of ciphertexts [2][L][N] whose last host-pipeline chunk holds one"""
    c = (64 << 20) // (16 * L << log_n)
    b = c + 1
    assert host_chunk(16 * L << log_n, b) == c, "the batch reaches a full wave: pick another row"
    return b


# ---- scratch model --------------------------------------------------------------------------------------------------------------
# the bytes of each scratch a call reserves, for the calls the guarantees rely on (deeppowers_b200/csrc/abi.cu: the reserve() of
# each entry point); a call missing here may still use a scratch, so the checks only look at the steps around a growth

UNSIZED = -1   # a step that may use the scratch by an amount the model does not size


def touches(step):
    """the scratch a step may use, from its entry point's name (deeppowers_b200/csrc/abi.cu: the users of each reserve())"""
    if step.kind in ("create", "apply") or step.fn.startswith(("dpfhe_linear", "dpfhe_polyeval", "dpfhe_slotsum")):
        return set(SCRATCH)          # the objects' own paths: any of them
    fn, out = step.fn, set()
    if "mod_switch" in fn or "mod_down_special" in fn or "compact_ciphertexts" in fn:
        out.add("ms_tau")
    if "rotate_hoisted" in fn and "grouped" not in fn:
        out |= {"hoist_U", "hoist_zero"}
    if "hoisted_grouped" in fn or "rotate_sum" in fn:
        out.add("hoistg")
    if "encode" in fn or "decode" in fn:
        out.add("enc_work")
    if "compact" in fn:
        out.add("compact_work")
    if ROWS[fn].host:
        out |= {"stage_in", "stage_out", "stage_key"}
    return out


def scratch_use(step, log_n, L):
    """{scratch: bytes it needs} of a step, UNSIZED where the model does not know"""
    if step.kind not in ("call", "create", "apply"):
        return {}
    u = {X: UNSIZED for X in touches(step)}
    u.update(_sized(step, log_n, L))
    return u


def _sized(step, log_n, L):
    if step.kind != "call":
        return {}
    s, fn, N = step.shape(log_n, L), step.fn, 1 << log_n
    b, w = s.batch, 8
    u = {}
    if fn in ("dpfhe_mod_switch_down", "dpfhe_mod_switch_down_level"):
        u["ms_tau"] = 2 * b * N * w
    elif fn == "dpfhe_mod_down_special":
        u["ms_tau"] = 2 * b * s.K * N * w
    elif fn == "dpfhe_rotate_hoisted":
        u["hoist_U"], u["hoist_zero"] = b * L * L * N * w, b * 4
    elif fn == "dpfhe_linear_create":
        u["hoist_U"], u["hoist_zero"] = L * L * N * w, 4      # the per-limb layer applied to one ciphertext: one chunk of one
    elif fn in ("dpfhe_rotate_hoisted_grouped", "dpfhe_rotate_sum_grouped"):
        Lb = L if s.level is None else s.level + s.K
        dnum = -(-(Lb - s.K) // s.K)
        u["hoistg"] = b * (dnum * Lb * N + 2 * Lb * N + 2 * s.K * N) * w
    elif fn in ("dpfhe_ckks_encode", "dpfhe_bgv_encode"):
        u["enc_work"] = b * N * w
    elif fn in ("dpfhe_ckks_decode", "dpfhe_bgv_decode"):
        u["enc_work"] = b * L * N * w
    elif fn in ("dpfhe_ckks_decode_level", "dpfhe_bgv_decode_level"):
        u["enc_work"] = b * s.lv * N * w
    elif fn == "dpfhe_decrypt_compact":
        u["compact_work"] = 2 * b * N * w
    elif fn == "dpfhe_compact_ciphertexts":
        l = s.lv
        u["compact_work"] = 2 * b * N * ((l - 1) + max(0, l - 2)) * w if l >= 2 else 2 * b * N * w
        if l >= 2:
            u["ms_tau"] = 2 * b * N * w
    elif fn == "dpfhe_ct_add_plain_host":
        item = 2 * L * N * w
        c = host_chunk(item, b)
        u["stage_in"], u["stage_out"], u["stage_key"] = c * item, c * item, L * N * w
    elif fn == "dpfhe_ct_mul_relin_host":
        item = 2 * L * N * w
        c = host_chunk(item, b)
        u["stage_in"], u["stage_out"], u["stage_key"] = 2 * c * item, c * item, 2 * L * L * N * w
    return u


def growth_pairs(log_n, L):
    """{scratch: (smaller call, larger call of another family)}: (fn, kw) each"""
    K = 2 if 2 * 2 <= L else 1
    lc = min(3, L)
    pairs = {
        "ms_tau": (("dpfhe_mod_switch_down", dict(batch=1)), ("dpfhe_mod_down_special", dict(K=K, batch=2))),
        "hoist_U": (("dpfhe_linear_create", dict(batch=1)), ("dpfhe_rotate_hoisted", dict(batch=3))),
        "hoistg": (("dpfhe_rotate_hoisted_grouped", dict(K=K, batch=1)), ("dpfhe_rotate_sum_grouped", dict(K=K, batch=3))),
        "enc_work": (("dpfhe_ckks_encode", dict(batch=1)), ("dpfhe_bgv_decode_level", dict(level=L - 1, batch=2))),
        "compact_work": (("dpfhe_decrypt_compact", dict(batch=1)), ("dpfhe_compact_ciphertexts", dict(level=lc, batch=2))),
        "stage_in": (("dpfhe_ct_add_plain_host", dict(batch=1)), ("dpfhe_ct_mul_relin_host", dict(batch=3))),
    }
    pairs["hoist_zero"] = pairs["hoist_U"]
    pairs["stage_out"] = pairs["stage_key"] = pairs["stage_in"]
    return pairs


# ---- shapes ---------------------------------------------------------------------------------------------------------------------

def shapes(fn, log_n, L):
    """the Shape parameters (K, level) at which a row runs on the context (log_n, L): [] when it does not"""
    Ks = [K for K in (2, 3) if 2 * K <= L]
    if fn in KS_PERLIMB or fn in PLAIN or fn in ENCODERS or fn in ("dpfhe_ct_mul_relin_host", "dpfhe_rotate_host", "dpfhe_ntt_fwd_host",
                                                                   "dpfhe_ntt_inv_host", "dpfhe_ct_mul_plain_host", "dpfhe_ct_add_plain_host",
                                                                   "dpfhe_mod_switch_down_host", "dpfhe_ckks_encode_host", "dpfhe_ckks_decode_host",
                                                                   "dpfhe_linear_create"):
        return [dict(K=0)]
    if fn in BGV_SLOTS:
        return [dict(K=0)] if log_n == 12 else []
    if fn in KEYS or fn in ("dpfhe_encrypt_host", "dpfhe_decrypt_host", "dpfhe_encrypt_public_host", "dpfhe_public_keygen_host"):
        return [dict(K=K) for K in [0] + Ks] if "keygen" in fn and fn not in ("dpfhe_secret_keygen", "dpfhe_public_keygen",
                                                                                "dpfhe_public_keygen_host") else [dict(K=0)]
    if fn in ("dpfhe_relin_keygen_host", "dpfhe_galois_keygen_host"):
        return [dict(K=K) for K in [0] + Ks]
    if fn in KS_HYBRID or fn in ("dpfhe_ct_mul_relin_hybrid_host", "dpfhe_rotate_hybrid_host"):
        return [dict(K=1)]
    if fn in ("dpfhe_mod_down_special", "dpfhe_mod_down_special_host"):
        return [dict(K=K) for K in [1] + Ks]
    if fn in KS_GROUPED or fn in ("dpfhe_ct_mul_relin_grouped_host", "dpfhe_rotate_grouped_host", "dpfhe_rotate_sum_grouped_host",
                                  "dpfhe_ct_dot_grouped_host", "dpfhe_ct_mul_relin_rescale_grouped_host", "dpfhe_ct_dot_rescale_grouped_host"):
        return [dict(K=K) for K in Ks]
    if fn in KS_LEVEL or fn in ("dpfhe_ct_mul_relin_rescale_grouped_level_host", "dpfhe_ct_dot_rescale_grouped_level_host"):
        rescale = "rescale" in fn
        return [dict(K=K, level=l) for K, l in level_pairs(L) if l >= 2 or not rescale]
    if fn in KEYLESS:
        lo = 2 if "mod_switch" in fn else 1
        return [dict(K=0, level=l) for l in range(lo, L + 1)]
    if fn in SEEDED:
        if "keygen" in fn or "switch_keys" in fn:
            return [dict(K=K) for K in [0] + Ks]
        if fn.endswith(("_level", "_level_host")):
            return [dict(K=0, level=l) for l in range(1, L + 1)]
        return [dict(K=0)]
    if fn in COMPACT:
        if fn in ("dpfhe_compact_ciphertexts", "dpfhe_download_compact_ciphertexts"):
            return [dict(K=0, level=l) for l in range(1, L + 1)]
        return [dict(K=0)]
    if fn in ("dpfhe_linear_create_grouped", "dpfhe_slotsum_create_grouped"):
        return [dict(K=K) for K in Ks]
    if fn in ("dpfhe_linear_create_grouped_level", "dpfhe_slotsum_create_grouped_level"):
        return [dict(K=K, level=l) for K, l in level_pairs(L) if K >= 2]
    # degree 3 takes D = 2 levels: at most min(Lq - 1, Lq - K + 1) below Lq ciphertext limbs
    if fn == "dpfhe_polyeval_create_grouped":
        return [dict(K=K) for K in Ks if min(L - K - 1, L - 2 * K + 1) >= 2]
    if fn == "dpfhe_polyeval_create_grouped_level":
        return [dict(K=K, level=l) for K, l in level_pairs(L) if K >= 2 and min(l - 1, l - K + 1) >= 2]
    return []


def pool(log_n, L):
    """[(fn, kw)] of every row and shape the filler calls draw from (the object rows are drawn as objects)"""
    names = (KS_PERLIMB + KS_HYBRID + KS_GROUPED + KS_LEVEL + PLAIN + ["dpfhe_mod_down_special"] + KEYS + ENCODERS + BGV_SLOTS + KEYLESS
             + SEEDED + COMPACT + HOST_KS + HOST_OTHER)
    if log_n == 14:   # N = 16384: the key-switch families and compaction
        names = KS_PERLIMB + KS_HYBRID + KS_GROUPED + KS_LEVEL + ["dpfhe_mod_down_special"] + COMPACT + ["dpfhe_ct_mul_relin_hybrid_host"]
    return [(fn, kw) for fn in names for kw in shapes(fn, log_n, L)]


def chainable(producer, p_name, consumer, c_name, log_n, L):
    """an output of the producer may be the consumer's operand: same words and rows of residues under the same moduli"""
    pr, cr = ROWS[producer.fn], ROWS[consumer.fn]
    pb = next(b for b in pr.bufs if b.name == p_name)
    cb = next(b for b in cr.bufs if b.name == c_name)
    if pb.role != mc.OUTPUT or cb.role != mc.OPERAND or pb.count is not None or cb.count is not None or pb.host or cb.host:
        return False
    if p_name in pr.gen or c_name in cr.gen or producer.fn in GENERATED_OUT:
        return False
    ps, cs = producer.shape(log_n, L), consumer.shape(log_n, L)
    return pb.words(ps) == cb.words(cs) and pb.limbs(ps) == cb.limbs(cs)


# outputs that are not residues of the rows' moduli: slots, compact words
GENERATED_OUT = {"dpfhe_ckks_decode", "dpfhe_bgv_decode", "dpfhe_ckks_decode_level", "dpfhe_bgv_decode_level", "dpfhe_compact_ciphertexts",
                 "dpfhe_decrypt_compact", "dpfhe_secret_keygen", "dpfhe_relin_keygen_seeded", "dpfhe_galois_keygen_seeded",
                 "dpfhe_encrypt_seeded", "dpfhe_encrypt_seeded_level", "dpfhe_decrypt", "dpfhe_decrypt_level"}


# ---- the generator --------------------------------------------------------------------------------------------------------------

class _Builder:
    def __init__(self, rng, log_n, L):
        self.rng, self.log_n, self.L = rng, log_n, L
        self.steps = []
        self.pool = pool(log_n, L)

    def seed(self):
        return int(self.rng.integers(0, 1 << 31))

    def stream(self, other_than=None):
        s = [x for x in (0, 1, 2) if x != other_than]
        return int(s[self.rng.integers(0, len(s))])

    def t(self):
        return int(T_PAIR[self.rng.integers(0, 2)])

    def call(self, fn, kw, stream=None, chain=None):
        kw = dict(kw)
        if fn == "dpfhe_rotate_sum_grouped_host":   # its row's reference splits the key table in pieces of one batch: one per digit
            kw["batch"] = -(-(self.L - kw["K"]) // kw["K"])
        kw.setdefault("batch", int(self.rng.integers(1, 4)))
        kw.setdefault("t", self.t())
        self.steps.append(Step("call", fn, kw, self.stream() if stream is None else stream, self.seed(), chain))
        return len(self.steps) - 1

    def filler(self):
        fn, kw = self.pool[self.rng.integers(0, len(self.pool))]
        i = self.call(fn, kw)
        self.try_chain(i)
        return i

    def try_chain(self, i, force_other_stream=False):
        """chains one operand of step i to the output of an earlier call when one fits"""
        st = self.steps[i]
        for j in self.rng.permutation(i):
            p = self.steps[int(j)]
            if p.kind != "call" or (force_other_stream and p.stream == st.stream):
                continue
            for pb in ROWS[p.fn].outputs():
                for cb in ROWS[st.fn].bufs:
                    if chainable(p, pb.name, st, cb.name, self.log_n, self.L):
                        st.chain = (int(j), pb.name, cb.name)
                        return True
        return False

    def growth(self):
        pairs = []
        for small, big in growth_pairs(self.log_n, self.L).values():
            if (small, big) not in pairs:
                pairs.append((small, big))
        # the per-limb linear layer's row comes last: an object row may use any scratch by an amount the model does not size
        order = [pairs[int(k)] for k in self.rng.permutation(len(pairs))]
        order.sort(key=lambda p: p[0][0] == "dpfhe_linear_create")
        for small, big in order:
            self.call(small[0], small[1])
            self.call(big[0], big[1])

    def bgv_t(self):
        """encode and decode at one t on two streams, then at the other t and back, each change behind a queued decode"""
        a, b = (T_PAIR if self.rng.integers(0, 2) else T_PAIR[::-1])
        e_st = self.stream()
        d_st = self.stream(other_than=e_st)
        for t in (a, b, a):
            l = int(self.rng.integers(1, self.L + 1))
            kw = dict(level=l, t=t, batch=int(self.rng.integers(1, 3)))
            e = self.call("dpfhe_bgv_encode_level", kw, stream=e_st)
            self.call("dpfhe_bgv_decode_level", kw, stream=d_st, chain=(e, "pt", "pt"))

    def levels(self):
        pairs = level_pairs(self.L)
        for k in self.rng.permutation(len(pairs)):
            K, l = pairs[int(k)]
            top = KS_HYBRID if K == 1 else ["dpfhe_ct_mul_relin_grouped", "dpfhe_rotate_grouped", "dpfhe_rotate_sum_grouped",
                                            "dpfhe_ct_mul_relin_rescale_grouped"]
            lv = [fn for fn in KS_LEVEL if l >= 2 or "rescale" not in fn]
            order = [("top", K), ("level", K, l)] if self.rng.integers(0, 2) else [("level", K, l), ("top", K)]
            for o in order:
                if o[0] == "top":
                    self.call(top[self.rng.integers(0, len(top))], dict(K=K))
                else:
                    self.call(lv[self.rng.integers(0, len(lv))], dict(K=K, level=l))

    def keyless(self):
        for l in range(1, self.L + 1):
            fns = [fn for fn in KEYLESS if shapes(fn, self.log_n, self.L) and l >= (2 if "mod_switch" in fn else 1)]
            self.call(fns[self.rng.integers(0, len(fns))], dict(K=0, level=l))

    def host_between(self):
        a = self.stream()
        self.call("dpfhe_ct_add_plain", dict(K=0), stream=a)
        host = [fn for fn, kw in self.pool if ROWS[fn].host]
        fn = host[self.rng.integers(0, len(host))]
        self.call(fn, shapes(fn, self.log_n, self.L)[0])
        self.call("dpfhe_ntt_fwd", dict(K=0), stream=self.stream(other_than=a))

    def chain_across(self):
        K = 2 if 2 * 2 <= self.L else 1
        fn = "dpfhe_ct_mul_relin_grouped" if K == 2 else "dpfhe_ct_mul_relin_hybrid"
        rot = "dpfhe_rotate_grouped" if K == 2 else "dpfhe_rotate_hybrid"
        b = int(self.rng.integers(1, 4))
        p = self.call(fn, dict(K=K, batch=b))
        self.call(rot, dict(K=K, batch=b), stream=self.stream(other_than=self.steps[p].stream), chain=(p, "out", "ct"))

    def short_host(self):
        self.call("dpfhe_ct_add_plain_host", dict(K=0, batch=short_chunk_batch(self.log_n, self.L)))

    def create(self, obj):
        cands = [(fn, kw) for fn in OBJECTS for kw in shapes(fn, self.log_n, self.L)]
        fn, kw = cands[self.rng.integers(0, len(cands))]
        kw = dict(kw, batch=1, t=mc.T)
        self.steps.append(Step("create", fn, kw, 0, self.seed(), obj=obj))

    def apply(self, obj):
        c = next(s for s in self.steps if s.kind == "create" and s.obj == obj)
        kw = dict(c.kw, batch=int(self.rng.integers(1, 4)))
        self.steps.append(Step("apply", c.fn, kw, self.stream(), self.seed(), obj=obj))

    def destroy(self, obj):
        self.steps.append(Step("destroy", obj=obj))


def program(seed, shape, n_steps):
    """the steps of one program on a context (log_n, L): the guaranteed transitions in seeded order, filler calls between them"""
    log_n, L = shape
    b = _Builder(np.random.default_rng(seed), log_n, L)

    def fill(n):
        for _ in range(n):
            b.filler()
            if b.rng.integers(0, 8) == 0:
                b.steps.append(Step("sync"))

    n_fill = max(0, n_steps - 80) // 4
    b.growth()
    b.create(0)
    b.create(1)
    phase_a = [b.bgv_t, b.levels, b.host_between, b.chain_across, b.keyless, lambda: b.apply(0), b.short_host]
    for k in b.rng.permutation(len(phase_a)):
        phase_a[int(k)]()
        fill(int(b.rng.integers(0, 2)))
    fill(n_fill)
    if log_n == 14:
        b.call("dpfhe_rotate_hybrid", dict(K=1, batch="round"))
    b.steps.append(Step("trim"))
    b.growth()
    b.apply(0)
    b.apply(1)
    phase_b = [b.levels, b.keyless, b.bgv_t, b.chain_across, b.host_between]
    for k in b.rng.permutation(len(phase_b)):
        phase_b[int(k)]()
        fill(int(b.rng.integers(0, 2)))
    fill(n_fill)
    b.destroy(1)
    fill(2)
    b.steps.append(Step("trim"))
    b.apply(0)
    b.destroy(0)
    fill(n_fill)
    return b.steps


# ---- the guarantees -------------------------------------------------------------------------------------------------------------

def _uses(steps, shape):
    return [scratch_use(s, *shape) for s in steps]


def growth_steps(steps, shape):
    """({scratch: [steps that grow it straight after a smaller call of another family]},
    {scratch: [steps that first use it after a trim that released it]})"""
    uses = _uses(steps, shape)
    grown, regrown = {X: [] for X in SCRATCH}, {X: [] for X in SCRATCH}
    for X in SCRATCH:
        since, used_before, first_after_trim = 0, False, False     # since: the largest use since the last trim
        for i, s in enumerate(steps):
            if s.kind == "trim":
                used_before, since, first_after_trim = used_before or since > 0, 0, True
                continue
            u = uses[i].get(X, 0)
            if not u:
                continue
            if u == UNSIZED:    # from here on nothing is known to grow until the next trim
                used_before, first_after_trim, since = True, False, float("inf")
                continue
            if first_after_trim and used_before:
                regrown[X].append(i)
            first_after_trim = False
            prev = steps[i - 1] if i else None
            if (u > since and prev is not None and prev.kind == "call" and 0 < uses[i - 1].get(X, 0) < u
                    and family(prev.fn) != family(s.fn)):
                grown[X].append(i)
            since = max(since, u)
    return grown, regrown


def check_guarantees(steps, shape):
    """[names of the guaranteed transitions the program lacks]"""
    log_n, L = shape
    missing = []
    uses = _uses(steps, shape)
    calls = [i for i, s in enumerate(steps) if s.kind == "call"]

    # growth straight after a smaller call of another family; first reuse after a trim that released it
    grown, regrown = growth_steps(steps, shape)
    for X in SCRATCH:
        if not grown[X]:
            missing.append("growth of %s after a smaller call of another family" % X)
        if not regrown[X]:
            missing.append("growth of %s after a trim" % X)

    # the BGV tables: t changes both ways, each behind a decode of the old t queued on another stream (no synchronisation between)
    def bgv_t(s):
        return mc.T_SLOTS if s.fn in BGV_SLOTS else s.kw["t"]

    bgv = set(BGV_SLOTS) | {"dpfhe_bgv_encode_level", "dpfhe_bgv_decode_level"}
    seen, last = set(), None
    for s in steps:
        if s.kind in ("sync", "trim", "create", "destroy") or (s.kind == "call" and ROWS[s.fn].host):
            last = None
        elif s.kind == "call" and s.fn in bgv:
            if last is not None and "decode" in last.fn and bgv_t(last) != bgv_t(s) and last.stream != s.stream:
                seen.add((bgv_t(last), bgv_t(s)))
            last = s
    if not any(a < b for a, b in seen) or not any(a > b for a, b in seen):
        missing.append("a BGV t change in both directions behind a queued decode")

    # a level call at every (K, l) before and after a trim, next to a top-level call of the same K
    trims = [i for i, s in enumerate(steps) if s.kind == "trim"]
    first_trim = trims[0] if trims else len(steps)

    def top_k(s):
        return s.kind == "call" and s.kw.get("level") is None and s.fn in KS_HYBRID + KS_GROUPED + KS_PERLIMB

    for K, l in level_pairs(L):
        for lo, hi, when in ((0, first_trim, "before"), (first_trim, len(steps), "after")):
            ok = False
            for i in range(lo, hi):
                s = steps[i]
                if s.kind == "call" and s.fn in KS_LEVEL and s.kw.get("K") == K and s.kw.get("level") == l:
                    nb = [steps[j] for j in (i - 1, i + 1) if lo <= j < hi]
                    ok = ok or any(top_k(n) and n.kw.get("K") == K for n in nb)
            if not ok:
                missing.append("level call at (K=%d, l=%d) %s a trim" % (K, l, when))

    # a keyless level call at every l
    for l in range(1, L + 1):
        if not any(steps[i].fn in KEYLESS and steps[i].kw.get("level") == l for i in calls):
            missing.append("keyless level call at l=%d" % l)

    # a host form between device calls on two different streams
    if not any(ROWS[steps[i].fn].host and 0 < i < len(steps) - 1 and all(steps[j].kind == "call" and not ROWS[steps[j].fn].host
                                                                          for j in (i - 1, i + 1))
               and steps[i - 1].stream != steps[i + 1].stream for i in calls):
        missing.append("a host form between device calls on two streams")

    # a host form whose last pipeline chunk is short
    def short(s):
        if s.kind != "call" or s.fn != "dpfhe_ct_add_plain_host":
            return False
        b = s.shape(log_n, L).batch
        c = host_chunk(16 * L << log_n, b)
        return b > c and b % c != 0
    if not any(short(steps[i]) for i in calls):
        missing.append("a host form with a short last chunk")

    # a chained operand on another stream than its producer
    if not any(steps[i].chain and not ROWS[steps[i].fn].host and steps[steps[i].chain[0]].stream != steps[i].stream for i in calls):
        missing.append("a chained step on another stream")

    # an object applied after a trim and after a scratch grew by a call since
    ok = False
    for i, s in enumerate(steps):
        if s.kind != "apply":
            continue
        c = next(j for j, x in enumerate(steps) if x.kind == "create" and x.obj == s.obj)
        tr = [j for j in trims if c < j < i]
        if not tr:
            continue
        big = {}
        for j in range(tr[-1] + 1, i):
            for X, u in uses[j].items():
                if u > big.get(X, 0):
                    if big.get(X, 0) and steps[j].kind == "call":
                        ok = True
                    big[X] = u
    if not ok:
        missing.append("an object applied after a trim and a scratch regrowth")
    return missing


# ---- memory ---------------------------------------------------------------------------------------------------------------------

def guard_words(row, s):
    per_ct = max(2 * b.limbs(s) * s.N for b in row.outputs())
    return max(GUARD_MIN, 2 * per_ct)


def device_buffers(step, log_n, L, sms=SMS):
    """[(name, words)] of a step's device buffers (a create: none; an apply: the object row's device buffers)"""
    if step.kind not in ("call", "apply"):
        return []
    row, s = ROWS[step.fn], step.shape(log_n, L, sms)
    return [(n, b.words(s)) for b in row.bufs if not b.host for n in b.names(s)]


def footprint(steps, shape, sms=SMS):
    """an upper bound of a program's device bytes: its arena (every buffer between guards) and every scratch at its largest use"""
    log_n, L = shape
    words = 0
    for st in steps:
        if st.kind not in ("call", "apply"):
            continue
        G = guard_words(ROWS[st.fn], st.shape(log_n, L, sms))
        words += sum(G + w + 32 for n, w in device_buffers(st, log_n, L, sms))
    scratch = {}
    for u in _uses(steps, shape):
        for X, v in u.items():
            scratch[X] = max(scratch.get(X, 0), v)   # UNSIZED counts nothing: the allowance below covers it
    # the context's own tables, key companions and digit slots, and the scratch the model does not size: a generous allowance
    return 8 * words + sum(scratch.values()) * 3 + (256 << 20)
