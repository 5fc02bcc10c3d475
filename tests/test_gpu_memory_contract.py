"""What every call of the C ABI writes, and what it must leave alone (DESIGN.md §3): each row of tests/memory_contract.py, with
every buffer of the call placed in one arena between guard words, on the GPU:

1. the outputs equal the reference bit for bit;
2. every guard word is unchanged;
3. every operand and key is bit-identical to its snapshot;
4. with the outputs pre-filled with all-ones words (above every modulus) and, in a second run, with random words, the result is the
   same: no output word is read before it is written (in-place buffers are exempt);

the exact aliases the header permits give the bits of the separate placement, and every output placed over any other buffer of
its call by one 16-byte pair, at that buffer's start and at its end, is rejected with DPFHE_ERR_INVALID, the arena unchanged and
no launch issued.  Argument checks the other files exercise are repeated here against a whole guarded arena.

Placement: each buffer starts 16 bytes past a 256-byte boundary (the 16-byte rule of CHECK_PTR, and the least alignment the
kernels need: the TMA tensor maps of the inverse transform and the bulk prefetches of the key-switch kernels want 16 bytes) and is
followed and preceded by seeded random guard words, at least 64 KiB and at least two ciphertexts of the call's output, so that a
store one row or one ciphertext off lands in a guard.  Host forms place their numpy arrays the same way inside one guarded array,
and run a batch whose last chunk is short.

Shapes: the rows at N = 4096; the key-switch families also at N = 8192 and N = 16384, with batch 1 and one ciphertext past a full
round of the persistent grid (test_gpu_ks_16384.grid); grouped keys with a ragged last digit (Lq = 5, K = 2) and a level call at
level 3 (one whole digit and a short one).  Contexts are made and closed per test; expected results are computed once per input
set.  The file's 403 cases take 3 min 21 s on an H100 80GB HBM3 (SXM, 700 W power limit) with an 8-core host."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import memory_contract as mc  # noqa: E402
from memory_contract import INPLACE, KEY, OPERAND, OUTPUT, Shape  # noqa: E402
from test_gpu_ks_16384 import UNCAPPED, grid  # noqa: E402
from test_gpu_parity import dp  # noqa: E402,F401  (a fixture)

ROWS = mc.build_rows()
GUARD_MIN = 8192            # words: 64 KiB
ALL_ONES = -1               # int64 view of 2^64 - 1, above every modulus
_REF = {}


class Refs:
    """the oracle of the context and oracles over other moduli, made on demand"""

    def __init__(self, oracle_mod, log_n, L):
        self.oracle_mod, self.log_n = oracle_mod, log_n
        self.o = oracle_mod.Oracle(log_n, L)
        self._sub = {}

    def sub(self, moduli):
        key = tuple(int(q) for q in moduli)
        if key not in self._sub:
            self._sub[key] = self.oracle_mod.Oracle(self.log_n, len(key), list(key))
        return self._sub[key]


# ---- placement ------------------------------------------------------------------------------------------------------------------

def entries(row, s):
    """[(name, words, role)] of every placed buffer"""
    return [(n, b.words(s), b.role) for b in row.bufs for n in b.names(s)]


def guard_words(row, s):
    per_ct = max(2 * b.limbs(s) * s.N for b in row.outputs())
    return max(GUARD_MIN, 2 * per_ct)


def up(x):
    """the next word offset 16 bytes past a 256-byte boundary"""
    return x + (2 - x) % 32


def layout(row, s, alias=(), over=None):
    """{name: (offset, words)} and the arena's words.  alias: names sharing the first one's placement; over = (output, other,
    'start' | 'end'): the output overlaps the other buffer by one 16-byte pair there (holes of the output's size around it keep it
    clear of every other buffer)"""
    G = guard_words(row, s)
    ents = entries(row, s)
    words = dict((n, w) for n, w, _ in ents)
    at, cur = {}, 0
    for n, w, _ in ents:
        if n in alias[1:] or (over and n == over[0]):
            continue
        if n == (alias[0] if alias else None):
            w = max(words[a] for a in alias)
        if over and n == over[1]:
            cur += words[over[0]]
        cur = up(cur + G)
        at[n] = (cur, w)
        cur += w
        if over and n == over[1]:
            cur += words[over[0]]
    for a in alias[1:]:
        at[a] = (at[alias[0]][0], words[a])
    if over:
        o, x, where = over
        xo, xw = at[x]
        ow = words[o]
        at[o] = (xo - ow + 2, ow) if where == "start" else (xo + xw - 2, ow)
    return at, up(cur + G) + 32


def inputs(row, R, s, rng):
    """the input words of every operand, key and in-place buffer: canonical residues under the moduli of its rows"""
    x = {}
    q = np.array(R.o.moduli, dtype=np.uint64)
    for b in row.bufs:
        if b.role == OUTPUT:
            continue
        for n in b.names(s):
            if b.name in row.gen:
                x[n] = row.gen[b.name](s, rng).reshape(-1)
                continue
            rows = b.items(s) * b.limbs(s)
            mods = np.tile(q[:b.limbs(s)], b.items(s))
            x[n] = (rng.integers(0, 1 << 63, size=(rows, s.N), dtype=np.uint64) % mods[:, None]).reshape(-1)
    return x


def reference(row, R, s, x):
    shaped = {n: v.reshape(-1, _limbs(row, s, n), s.N) if not _raw(row, n) else v for n, v in x.items()}
    return {n: np.ascontiguousarray(v).reshape(-1).astype(np.uint64, copy=False) for n, v in row.ref(R, s, shaped).items()}


def _buf(row, n):
    return next(b for b in row.bufs if b.name == n.split(".")[0])


def _raw(row, n):
    return _buf(row, n).name in row.gen


def _limbs(row, s, n):
    return _buf(row, n).limbs(s)


class Arena:
    """one arena (a CUDA tensor, or a numpy array for host rows) with the buffers of a call placed in it"""

    def __init__(self, row, s, at, total, seed, device):
        self.row, self.s, self.at, self.host = row, s, at, row.host
        g = np.random.default_rng(seed).integers(0, 1 << 63, size=total, dtype=np.uint64) | np.uint64(1 << 63)
        self.dev = None if all(b.host for b in row.bufs) else torch.from_numpy(g.view(np.int64)).to(device)
        self.harr = g.copy() if any(b.host for b in row.bufs) else None
        if self.dev is not None:
            assert self.dev.data_ptr() % 256 == 0

    def _where(self, n):
        return self.harr if _buf(self.row, n).host else self.dev

    def write(self, n, words):
        o, w = self.at[n]
        tgt = self._where(n)
        if tgt is self.harr:
            tgt[o:o + w] = words
        else:
            tgt[o:o + w] = torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint64).view(np.int64)).to(tgt.device)

    def ptrs(self):
        p = {}
        for b in self.row.bufs:
            for n in b.names(self.s):
                o, w = self.at[n]
                p[n] = self.harr[o:o + w] if b.host else self.dev.data_ptr() + 8 * o
            if b.count is not None:
                p[b.name] = [p[n] for n in b.names(self.s)]
        return p

    def snapshot(self):
        return (None if self.dev is None else self.dev.cpu().numpy().view(np.uint64).copy(),
                None if self.harr is None else self.harr.copy())

    def region(self, snap, n):
        o, w = self.at[n]
        d, h = snap
        return (h if _buf(self.row, n).host else d)[o:o + w]


def compare_outside(row, arena, before, after, written):
    """every word outside the regions of `written` is unchanged (guards, operands, keys)"""
    for k in (0, 1):
        if before[k] is None:
            continue
        host_side = k == 1
        keep = np.ones(before[k].shape[0], dtype=bool)
        for n in written:
            if _buf(row, n).host == host_side:
                o, w = arena.at[n]
                keep[o:o + w] = False
        bad = np.flatnonzero(before[k][keep] != after[k][keep])
        if bad.size:
            idx = np.flatnonzero(keep)[bad[:4]]
            owner = [_owner(arena, int(i), host_side) for i in idx]
            raise AssertionError("%s: %d words outside the outputs changed, first at %s" % (row.fn, bad.size, owner))


def _owner(arena, i, host_side):
    for n, (o, w) in arena.at.items():
        if _buf(arena.row, n).host == host_side and o <= i < o + w:
            return "%s+%d" % (n, i - o)
    near = min(((abs(i - o), n, i - o) if i < o else (abs(i - o - w), n, i - o - w + 1) for n, (o, w) in arena.at.items()
                if _buf(arena.row, n).host == host_side))
    return "guard %s %+d words" % (near[1], near[2])


# ---- the four properties ----------------------------------------------------------------------------------------------------------

def run_case(row, c, R, s, seed, alias=()):
    rng = np.random.default_rng(seed)
    key = (row.fn, repr(s), s.n_rot, s.n_terms, s.n_steps, s.n_groups, seed, alias)
    if key not in _REF:
        x = inputs(row, R, s, rng)
        for a in alias[1:]:                      # buffers sharing a placement share their words
            if a in x and alias[0] in x:
                x[a] = x[alias[0]]
        for a in alias:
            if a in x:
                for b in alias:
                    if b != a and _buf(row, b).role != OUTPUT:
                        x[b] = x[a]
        _REF.clear()
        _REF[key] = (x, reference(row, R, s, x))
    x, want = _REF[key]
    at, total = layout(row, s, alias)
    written = [b.name if b.count is None else n for b in row.outputs() for n in b.names(s)]
    for fill in ("ones", "random"):
        arena = Arena(row, s, at, total, seed + 1, "cuda")
        for n, v in x.items():
            if n not in alias or _buf(row, n).role != OUTPUT:
                arena.write(n, v)
        for n in written:
            if n in alias or _buf(row, n).role == INPLACE:
                continue
            w = at[n][1]
            arena.write(n, np.full(w, np.uint64(2**64 - 1)) if fill == "ones" else rng.integers(0, 1 << 64, size=w, dtype=np.uint64))
        before = arena.snapshot()
        row.run(c, s, arena.ptrs())
        torch.cuda.synchronize()
        after = arena.snapshot()
        for n in written:
            got = arena.region(after, n)
            if not np.array_equal(got, want[n]):
                bad = np.flatnonzero(got != want[n])
                per_ct = 2 * _limbs(row, s, n) * s.N
                raise AssertionError("%s %s (%s fill, alias %s): %d words of %s differ, ciphertexts %s" %
                                     (row.fn, s, fill, alias, bad.size, n, sorted(set((bad // per_ct).tolist()))[:8]))
        compare_outside(row, arena, before, after, list(written) + [a for a in alias if a not in written])
        if alias:
            break


@pytest.fixture
def make(dp, oracle_mod, monkeypatch):
    """make(s, env={}, multi=False) -> (context, Refs); contexts closed when the test ends, after torch's cached blocks went back"""
    made = []
    torch.cuda.empty_cache()

    def get(s, env=None, multi=False):
        for k, v in (env or {}).items():
            monkeypatch.setenv(k, v)
        c = dp.MultiContext(s.log_n, s.L, devices=[0, 0]) if multi else dp.Context(s.log_n, s.L)
        made.append(c)
        return c, Refs(oracle_mod, s.log_n, s.L)

    yield get
    for c in made:
        c.close()
    _REF.clear()
    torch.cuda.empty_cache()


# ---- cases ----------------------------------------------------------------------------------------------------------------------

KS_PERLIMB = ["dpfhe_keyswitch", "dpfhe_ct_mul_relin", "dpfhe_rotate", "dpfhe_rotate_steps", "dpfhe_rotate_hoisted"]
KS_HYBRID = ["dpfhe_keyswitch_hybrid", "dpfhe_ct_mul_relin_hybrid", "dpfhe_rotate_hybrid"]
KS_GROUPED = ["dpfhe_keyswitch_grouped", "dpfhe_ct_mul_relin_grouped", "dpfhe_rotate_grouped", "dpfhe_rotate_hoisted_grouped",
              "dpfhe_rotate_sum_grouped", "dpfhe_ct_dot_grouped", "dpfhe_ct_mul_relin_rescale_grouped", "dpfhe_ct_dot_rescale_grouped"]
KS_LEVEL = ["dpfhe_ct_mul_relin_grouped_level", "dpfhe_rotate_grouped_level", "dpfhe_rotate_hoisted_grouped_level",
            "dpfhe_rotate_sum_grouped_level", "dpfhe_ct_dot_grouped_level", "dpfhe_ct_mul_relin_rescale_grouped_level",
            "dpfhe_ct_dot_rescale_grouped_level"]


def ks_shape(fn, log_n, batch=1, **kw):
    if fn in KS_PERLIMB:
        return Shape(log_n, 2, 0, batch, n_rot=2, **kw)
    if fn in KS_HYBRID:
        return Shape(log_n, 3, 1, batch, **kw)
    level = 3 if fn in KS_LEVEL else None
    base = dict(n_rot=2, n_terms=3)
    base.update(kw)
    return Shape(log_n, 7, 2, batch, level=level, **base)


def round_batch(s):
    """one ciphertext past a full round of the persistent grid: groups of every limb of the call's basis (the fused kernel: the
    ciphertext limbs, which are all of the context's)"""
    groups, rounds = grid(s.lv + s.K, UNCAPPED)
    b = groups + 1
    assert grid(s.lv + s.K, b) == (groups, 2)
    return b


KS_CASES = [(fn, log_n, b) for fn in KS_PERLIMB + KS_HYBRID + KS_GROUPED + KS_LEVEL for log_n in (12, 13, 14)
            for b in ((1, "round") if log_n == 12 else ("round",))]


def with_batch(s, b):
    if b == "round":
        b = round_batch(s)
    return Shape(s.log_n, s.L, s.K, b, s.level, s.n_rot, s.n_terms, s.n_steps, s.n_groups, s.n_comp, s.t)


@pytest.mark.parametrize("fn,log_n,batch", KS_CASES)
def test_key_switch_families(make, fn, log_n, batch):
    s = with_batch(ks_shape(fn, log_n), batch)
    c, R = make(s)
    run_case(ROWS[fn], c, R, s, 1000 + log_n)


@pytest.mark.parametrize("fn,kw", [("dpfhe_rotate_sum_grouped", dict(n_rot=15)), ("dpfhe_rotate_sum_grouped_level", dict(n_rot=15)),
                                   ("dpfhe_ct_dot_grouped", dict(n_terms=64)), ("dpfhe_ct_dot_rescale_grouped_level", dict(n_terms=64))])
def test_many_rotations_and_pairs(make, fn, kw):
    """15 summed rotations, 64 operand pairs"""
    s = ks_shape(fn, 12, 2, **kw)
    c, R = make(s)
    run_case(ROWS[fn], c, R, s, 2000)


OTHER = {
    "dpfhe_poly_mul_pointwise": Shape(12, 2, batch=3), "dpfhe_poly_add": Shape(12, 2, batch=3),
    "dpfhe_ct_tensor": Shape(12, 2, batch=3), "dpfhe_ct_mul_plain": Shape(12, 2, batch=3),
    "dpfhe_ct_mul_plain_acc": Shape(12, 2, batch=3), "dpfhe_ct_mul_plain_inner": Shape(12, 2, batch=3, n_steps=3, n_groups=2),
    "dpfhe_ct_lincomb": Shape(12, 2, batch=3, n_terms=3), "dpfhe_ct_add_plain": Shape(12, 2, batch=3),
    "dpfhe_mod_switch_down": Shape(12, 3, batch=3), "dpfhe_mod_down_special": Shape(12, 5, 2, batch=3),
    "dpfhe_ntt_fwd": Shape(12, 2, batch=3), "dpfhe_ntt_inv": Shape(12, 2, batch=3), "dpfhe_fill_uniform": Shape(12, 2, batch=3),
    "dpfhe_secret_keygen": Shape(12, 3), "dpfhe_relin_keygen": Shape(12, 5, 2), "dpfhe_galois_keygen": Shape(12, 5, 2, n_rot=3),
    "dpfhe_encrypt": Shape(12, 2, batch=3), "dpfhe_decrypt": Shape(12, 2, batch=3, n_comp=3), "dpfhe_public_keygen": Shape(12, 2),
    "dpfhe_encrypt_public": Shape(12, 2, batch=3), "dpfhe_ckks_encode": Shape(12, 2, batch=3), "dpfhe_ckks_decode": Shape(12, 2, batch=3),
    "dpfhe_bgv_encode": Shape(12, 2, batch=2), "dpfhe_bgv_decode": Shape(12, 2, batch=2),
}
OTHER_EXTRA = [("dpfhe_relin_keygen", Shape(12, 3, 0)), ("dpfhe_galois_keygen", Shape(12, 3, 0, n_rot=3)),
               ("dpfhe_ntt_inv", Shape(13, 2, batch=3)), ("dpfhe_decrypt", Shape(12, 2, batch=3, n_comp=2))]


@pytest.mark.parametrize("fn,s", list(OTHER.items()) + OTHER_EXTRA, ids=lambda v: repr(v) if isinstance(v, Shape) else v)
def test_other_device_calls(make, fn, s):
    c, R = make(s)
    run_case(ROWS[fn], c, R, s, 3000)


ALIAS_CASES = [(fn, a) for fn, row in sorted(ROWS.items()) for a in row.aliases]


@pytest.mark.parametrize("fn,alias", ALIAS_CASES)
def test_permitted_aliases(make, fn, alias):
    """the output on an input it may alias: the bits of the separate placement, every guard and every other buffer unchanged"""
    s = OTHER[fn]
    c, R = make(s)
    run_case(ROWS[fn], c, R, s, 4000, alias)


# ---- host forms ---------------------------------------------------------------------------------------------------------------

HOST = {fn: row for fn, row in ROWS.items() if row.host and not row.multi and fn.endswith("_host") and
        not fn.startswith(("dpfhe_linear", "dpfhe_polyeval", "dpfhe_slotsum"))}


def host_shape(fn):
    dev_fn = fn[:-len("_host")]
    if dev_fn in OTHER:
        s = OTHER[dev_fn]
        return Shape(s.log_n, s.L, s.K, max(s.batch, 3), s.level, s.n_rot, s.n_terms, s.n_steps, s.n_groups, s.n_comp)
    return ks_shape(dev_fn, 12, 3)


@pytest.mark.parametrize("fn", sorted(HOST))
def test_host_forms(make, fn):
    s = host_shape(fn)
    c, R = make(s)
    run_case(ROWS[fn], c, R, s, 5000)


def test_host_form_with_short_last_chunk(make):
    """513 ciphertexts at N = 4096 with two limbs: a 64 MiB chunk holds 512 (abi.cu pick_chunk), the last holds one"""
    s = Shape(12, 2, batch=513)
    c, R = make(s)
    run_case(ROWS["dpfhe_ct_mul_plain_host"], c, R, s, 5100)


@pytest.mark.parametrize("fn", ["dpfhe_rotate_hoisted", "dpfhe_rotate_hoisted_grouped", "dpfhe_rotate_sum_grouped"])
def test_hoisting_scratch_in_chunks(make, fn):
    """DPFHE_HOIST_CAP_MB=1: chunks of a few ciphertexts of the hoisted rotations' scratch, the last one short"""
    s = ks_shape(fn, 12, 11)
    c, R = make(s, {"DPFHE_HOIST_CAP_MB": "1"})
    run_case(ROWS[fn], c, R, s, 5200)


# ---- library objects --------------------------------------------------------------------------------------------------------------

OBJECTS = [("dpfhe_linear_create", Shape(12, 2, batch=3), {}),
           ("dpfhe_linear_apply_host", Shape(12, 2, batch=0), {"DPFHE_LINEAR_CHUNK_ROUNDS": "1"}),
           ("dpfhe_linear_create_grouped", Shape(12, 7, 2, batch=3), {}),
           ("dpfhe_linear_create_grouped_level", Shape(12, 7, 2, batch=3, level=3), {}),
           ("dpfhe_polyeval_create_grouped", Shape(12, 5, 2, batch=3), {}),
           ("dpfhe_polyeval_apply_host", Shape(12, 5, 2, batch=5), {"DPFHE_POLYEVAL_CHUNK": "2"}),
           ("dpfhe_polyeval_create_ckks", Shape(12, 5, 2, batch=3, t=0), {}),
           ("dpfhe_slotsum_create_grouped", Shape(12, 7, 2, batch=3), {}),
           ("dpfhe_slotsum_apply_host", Shape(12, 7, 2, batch=5), {"DPFHE_SLOTSUM_CHUNK": "2"}),
           ("dpfhe_slotsum_create_grouped_level", Shape(12, 7, 2, batch=3, level=3), {})]
OBJECTS += [("dpfhe_linear_apply", OBJECTS[0][1], {}), ("dpfhe_polyeval_apply", OBJECTS[4][1], {}),
            ("dpfhe_slotsum_apply", OBJECTS[7][1], {})]


@pytest.mark.parametrize("fn,s,env", OBJECTS, ids=[o[0] for o in OBJECTS])
def test_library_objects(make, fn, s, env):
    """create from guarded host arrays (which stay unchanged), apply (device or host buffers), destroy"""
    if s.batch == 0:   # one ciphertext past a chunk of one grid round of the per-limb layer
        s = Shape(s.log_n, s.L, s.K, grid(s.L, UNCAPPED)[0] + 1)
    c, R = make(s, env)
    run_case(ROWS[fn], c, R, s, 6000)


# ---- several GPUs in one process ----------------------------------------------------------------------------------------------

MULTI = [("dpfhe_multi_ct_mul_relin_host", Shape(12, 2, batch=5)), ("dpfhe_multi_ct_mul_relin_grouped_host", Shape(12, 7, 2, batch=5)),
         ("dpfhe_multi_rotate_host", Shape(12, 2, batch=5)), ("dpfhe_multi_ct_mul_relin_gather", Shape(12, 2, batch=5))]


@pytest.mark.parametrize("fn,s", MULTI, ids=[m[0] for m in MULTI])
def test_multi_device_calls(make, fn, s):
    """device 0 listed twice: two shards, the gather's root buffer between guards"""
    c, R = make(s, multi=True)
    run_case(ROWS[fn], c, R, s, 7000)


# ---- overlaps -----------------------------------------------------------------------------------------------------------------------

def overlap_cases():
    out = []
    for fn, row in sorted(ROWS.items()):
        if row.host or row.multi:
            continue
        s = OTHER.get(fn) or ks_shape(fn, 12, 2)
        names = [n for b in row.bufs for n in b.names(s)]
        for b in row.outputs():
            for o in b.names(s):
                for x in names:
                    if x != o:
                        out += [(fn, o, x, "start"), (fn, o, x, "end")]
    return out


@pytest.mark.parametrize("fn,out,other,where", overlap_cases())
def test_overlapping_output_is_rejected(make, fn, out, other, where):
    """the output over one 16-byte pair of another buffer of the call: DPFHE_ERR_INVALID, nothing written, nothing launched"""
    row = ROWS[fn]
    s = OTHER.get(fn) or ks_shape(fn, 12, 2)
    c, R = make(s)
    at, total = layout(row, s, over=(out, other, where))
    arena = Arena(row, s, at, total, 8000, "cuda")
    x = inputs(row, R, s, np.random.default_rng(8001))
    for n, v in x.items():
        if n != out:
            arena.write(n, v)
    torch.cuda.synchronize()
    before, launches = arena.snapshot(), c.launch_count()
    with pytest.raises(RuntimeError, match="overlap|must be"):
        row.run(c, s, arena.ptrs())
    torch.cuda.synchronize()
    assert c.launch_count() == launches
    after = arena.snapshot()
    assert np.array_equal(before[0], after[0]), "%s: a rejected call wrote into the arena" % fn


# ---- rejected calls -----------------------------------------------------------------------------------------------------------------

def _rejections(c, s, p):
    """the argument errors the other files exercise, each with every buffer placed"""
    K = s.K
    yield "null key", lambda: c.ct_mul_relin_grouped(K, p["a"], p["b"], 0, p["out"], s.batch, mc.T)
    yield "misaligned output", lambda: c.ct_mul_relin_grouped(K, p["a"], p["b"], p["key"], p["out"] + 8, s.batch, mc.T)
    yield "n_special", lambda: c.ct_mul_relin_grouped(4, p["a"], p["b"], p["key"], p["out"], s.batch, mc.T)
    yield "t above a special prime", lambda: c.ct_mul_relin_grouped(K, p["a"], p["b"], p["key"], p["out"], s.batch, c.moduli[-1])
    yield "level", lambda: c.ct_mul_relin_grouped_level(K, 1, p["a"], p["b"], p["key"], p["out"], s.batch, mc.T)
    yield "galois element", lambda: c.rotate_grouped(K, p["a"], 4, p["key"], p["out"], s.batch, mc.T)
    yield "n_terms", lambda: c.ct_dot_grouped(K, [p["a"]] * 65, [p["b"]] * 65, p["key"], p["out"], s.batch, mc.T)
    yield "n_rot", lambda: c.rotate_sum_grouped(K, p["a"], [5] * 16, [p["key"]] * 16, p["out"], s.batch, mc.T)
    yield "output on the input", lambda: c.ct_mul_relin_grouped(K, p["a"], p["b"], p["key"], p["a"], s.batch, mc.T)


def test_rejected_calls_leave_the_arena_untouched(make):
    row = ROWS["dpfhe_ct_mul_relin_grouped"]
    s = ks_shape("dpfhe_ct_mul_relin_grouped", 12, 3)
    c, R = make(s)
    at, total = layout(row, s)
    arena = Arena(row, s, at, total, 9000, "cuda")
    for n, v in inputs(row, R, s, np.random.default_rng(9001)).items():
        arena.write(n, v)
    torch.cuda.synchronize()
    before = arena.snapshot()
    p = arena.ptrs()
    for what, call in _rejections(c, s, p):
        launches = c.launch_count()
        with pytest.raises(RuntimeError):
            call()
        torch.cuda.synchronize()
        assert c.launch_count() == launches, what
        assert np.array_equal(arena.snapshot()[0], before[0]), what
