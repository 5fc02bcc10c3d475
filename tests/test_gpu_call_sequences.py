"""Call sequences on one context (tests/call_program.py): the memory-contract rows back to back on three streams, with trims,
BGV plaintext-modulus changes, level calls at every (K, l), growing scratch and objects that live across other calls.

Each program runs on one context and one guarded arena: every step's buffers are placed as tests/test_gpu_memory_contract.py places
one call's (Arena, layout), one after another, so a store into a neighbour lands in a guard or in another step's buffer.  The
expected results are computed first, with each row's own reference (chained operands take their producer's expected output).
The inputs are written and synchronised once; the program is then issued without host synchronisation, except in the steps that
synchronise by contract (host forms, object rows, sync, trim).  After one synchronisation at the end every output equals its
reference bit for bit, and every operand, key and guard word is unchanged.  At every step where the program guarantees that a
scratch buffer grows, dpfhe_context_device_bytes grew.  After the objects are destroyed, a trim brings dpfhe_context_device_bytes
back to its value at creation plus what a trim keeps by design: the hoisted-rotation constants and the special-prime accumulator
rows of the hybrid, grouped and multiply-and-rescale kernels (kept_after_trim).

A failing program reports its seed, the first failing step, the five steps before it and the first differing words, then replays
itself on a new context up to that step with dpfhe_synchronize after every step: a step that still fails points at context state,
one that passes at the ordering between streams.  Keeping the BGV tables of the first plaintext modulus when t changes fails the
N = 4096 program at its first encode after a change, and the serialised replay fails there too.

One program per context: N = 4096 with L = 7 (390 steps), N = 8192 with L = 6 (302 steps, DPFHE_EPOCH_LIMIT=40 so that the
round numbering of the persistent kernels restarts many times) and N = 16384 with L = 4 (181 steps, one batch past a full grid
round); two programs on two contexts interleaved from one thread, and two from two threads.  The file's 5 tests take 79 s on an
H100 80GB HBM3 (SXM, 700 W power limit) with an 8-core host; the largest program (N = 16384) peaks at 2.34 GiB of device memory,
arena and context together."""
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import call_program as cp  # noqa: E402
import memory_contract as mc  # noqa: E402
from test_gpu_ks_16384 import UNCAPPED, grid, sms  # noqa: E402
from test_gpu_memory_contract import Refs, inputs, reference, up  # noqa: E402
from test_gpu_parity import dp  # noqa: E402,F401  (a fixture)

PROGRAMS = [("n4096", (12, 7), 11, 400, {}), ("n8192", (13, 6), 12, 320, {"DPFHE_EPOCH_LIMIT": "40"}), ("n16384", (14, 4), 13, 200, {})]


# ---- the objects: made as the rows of memory_contract._object_rows / level_contract._polyeval_level_rows make them ----------------

def make_object(c, fn, s, p):
    from deeppowers_b200 import LinearLayer, PolyEval, SlotSum
    if fn.startswith("dpfhe_linear"):
        return LinearLayer.grouped(c, s.K, p["diags"].reshape(4, -1), 2, p["gk_baby"], p["gk_giant"], s.t, s.level)
    if fn.startswith("dpfhe_slotsum"):
        return SlotSum.grouped(c, s.K, 1, [3], p["gks"], s.t, s.level)
    if fn == "dpfhe_polyeval_create_grouped":
        return PolyEval(c, s.K, mc.T, [3, 0, 5, 1], p["key"])
    if fn == "dpfhe_polyeval_create_grouped_level":
        return PolyEval(c, s.K, mc.T, [3, 0, 5, 1], p["key"], level=s.lv)
    raise ValueError(fn)


# ---- placement ----------------------------------------------------------------------------------------------------------------------

class Plan:
    """every step's buffers placed in one device arena and one host arena, each buffer between guards; a chained operand shares its
    producer's output placement.  x[i] / want[i]: the inputs and expected outputs of step i"""

    def __init__(self, steps, shape, R, sms_):
        self.steps, self.shape, self.sms = steps, shape, sms_
        log_n, L = shape
        self.at = [dict() for _ in steps]          # step -> {name: (host?, offset, words)}
        cur = {False: 0, True: 0}
        for i, st in enumerate(steps):
            if st.kind not in ("call", "apply", "create"):
                continue
            row, s = cp.ROWS[st.fn], st.shape(log_n, L, sms_)
            G = cp.guard_words(row, s)
            for b in row.bufs:
                if st.kind == "create" and not b.host or st.kind == "apply" and b.host:
                    continue
                for n in b.names(s):
                    if st.chain and n == st.chain[2]:
                        self.at[i][n] = self.at[st.chain[0]][st.chain[1]]
                        continue
                    o = up(cur[b.host] + G)
                    self.at[i][n] = (b.host, o, b.words(s))
                    cur[b.host] = o + b.words(s)
        self.total = {h: up(cur[h] + cp.GUARD_MIN) + 32 for h in (False, True)}
        self.x, self.want = self._references(R)

    def _references(self, R):
        log_n, L = self.shape
        x, want = [None] * len(self.steps), [None] * len(self.steps)
        futs = {}

        def one(i):
            st = self.steps[i]
            row, s = cp.ROWS[st.fn], st.shape(log_n, L, self.sms)
            xi = inputs(row, R, s, np.random.default_rng(st.seed))
            if st.chain:
                j, pn, cn = st.chain
                futs[j].result()
                xi[cn] = want[j][pn]
            if st.kind == "apply":
                c = next(k for k, y in enumerate(self.steps) if y.kind == "create" and y.obj == st.obj)
                futs[c].result()
                xi.update({n: v for n, v in x[c].items() if n in self.at[c]})
            x[i] = xi
            if st.kind != "create":
                want[i] = reference(row, R, s, xi)

        with ThreadPoolExecutor(8) as pool:
            for i, st in enumerate(self.steps):
                if st.kind in ("call", "apply", "create"):
                    futs[i] = pool.submit(one, i)
            for f in futs.values():
                f.result()
        return x, want

    def arenas(self, seed):
        """(initial, expected) words of the device and the host arena: guards and output fill random, inputs placed"""
        init, exp = {}, {}
        for h in (False, True):
            g = np.random.default_rng(seed + h).integers(0, 1 << 63, size=self.total[h], dtype=np.uint64) | np.uint64(1 << 63)
            init[h], exp[h] = g, g.copy()
        for i, st in enumerate(self.steps):
            for n, (h, o, w) in self.at[i].items():
                if st.chain and n == st.chain[2]:
                    continue
                if self.x[i] is not None and n in self.x[i]:
                    init[h][o:o + w] = self.x[i][n]
                    exp[h][o:o + w] = self.x[i][n]
        for i, st in enumerate(self.steps):
            if self.want[i] is None:
                continue
            for n, v in self.want[i].items():
                h, o, w = self.at[i][n]
                exp[h][o:o + w] = v
        return init, exp

    def owner(self, h, idx):
        """(step, buffer or 'guard before <buffer>') of arena word idx"""
        best = None
        for i, m in enumerate(self.at):
            for n, (hh, o, w) in m.items():
                if hh != h:
                    continue
                if o <= idx < o + w:
                    return i, "%s+%d" % (n, idx - o)
                d = o - idx if idx < o else idx - o - w + 1
                if best is None or d < best[0]:
                    best = (d, i, "guard %+d words from %s" % (idx - o if idx < o else idx - o - w + 1, n))
        return best[1], best[2]


# ---- execution -------------------------------------------------------------------------------------------------------------------

class Runner:
    """one program on one context: its plan, arenas, streams and live objects"""

    def __init__(self, name, c, plan, seed):
        self.name, self.c, self.plan, self.seed = name, c, plan, seed
        self.steps, self.shape = plan.steps, plan.shape
        self.streams = [torch.cuda.default_stream(), torch.cuda.Stream(), torch.cuda.Stream()]
        self.objs, self.peak, self.grew = {}, 0, {}

    def load(self):
        init, self.exp = self.plan.arenas(self.seed)
        self.dev = torch.from_numpy(init[False].view(np.int64)).cuda()
        self.host = init[True].copy()
        assert self.dev.data_ptr() % 256 == 0
        torch.cuda.synchronize()
        self.base = self.c.device_bytes()
        self.peak = self.base + self.dev.numel() * 8

    def ptrs(self, i):
        p = {}
        st = self.steps[i]
        row = cp.ROWS[st.fn]
        for n, (h, o, w) in self.plan.at[i].items():
            p[n] = self.host[o:o + w] if h else self.dev.data_ptr() + 8 * o
        s = st.shape(*self.shape, sms())
        for b in row.bufs:
            if b.count is not None and all(n in p for n in b.names(s)):
                p[b.name] = [p[n] for n in b.names(s)]
        return p

    def step(self, i):
        st, c = self.steps[i], self.c
        before = c.device_bytes()
        if st.kind == "trim":
            c._chk(c._l.dpfhe_context_trim(c._h))
        elif st.kind == "sync":
            c.synchronize()
        elif st.kind == "create":
            self.objs[st.obj] = make_object(c, st.fn, st.shape(*self.shape, sms()), self.ptrs(i))
        elif st.kind == "destroy":
            self.objs.pop(st.obj).close()
        else:
            s = st.shape(*self.shape, sms())
            p = self.ptrs(i)
            with torch.cuda.stream(self.streams[st.stream]):
                if st.kind == "apply":
                    self.objs[st.obj].apply(p["ct"], p["out"], s.batch)
                else:
                    cp.ROWS[st.fn].run(c, s, p)
        self.grew[i] = c.device_bytes() > before
        self.peak = max(self.peak, c.device_bytes() + self.dev.numel() * 8)

    def run(self, upto=None, serial=False):
        for i in range(len(self.steps) if upto is None else upto + 1):
            self.step(i)
            if serial:
                self.c.synchronize()

    def finish(self):
        for o in self.objs.values():
            o.close()
        self.objs.clear()

    def mismatches(self, upto=None):
        """[(step, where, got, want)] of every differing word, by step"""
        torch.cuda.synchronize()
        got = {False: self.dev.cpu().numpy().view(np.uint64), True: self.host}
        out = []
        for h in (False, True):
            bad = np.flatnonzero(got[h] != self.exp[h])
            for k in bad[:4096]:
                i, where = self.plan.owner(h, int(k))
                if upto is None or i <= upto:
                    out.append((i, where, int(got[h][k]), int(self.exp[h][k])))
        return sorted(out, key=lambda m: m[0])

    def report(self, bad):
        i = bad[0][0]
        s = self.steps[i]
        lines = ["%s seed %d: step %d %r (shape %r) fails" % (self.name, self.seed, i, s,
                                                              s.shape(*self.shape, sms()) if s.fn else None)]
        lines += ["  step %d: %r" % (j, self.steps[j]) for j in range(max(0, i - 5), i)]
        lines += ["  %s: got %#x, want %#x" % (w, g, e) for k, w, g, e in bad if k == i][:8]
        return i, "\n".join(lines)


def run_program(name, dp, oracle_mod, shape, seed, n_steps, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    steps = cp.program(seed, shape, n_steps)
    assert not cp.check_guarantees(steps, shape)
    plan = Plan(steps, shape, Refs(oracle_mod, *shape), sms())
    c = dp.Context(*shape)
    r = Runner(name, c, plan, seed)
    try:
        check_round_batches(r)
        r.load()
        r.run()
        torch.cuda.synchronize()
        finish_and_check(r, oracle_mod, dp, env)
    finally:
        r.finish()
        c.close()
    return r


def check_round_batches(r):
    for st in r.steps:
        if st.kind == "call" and st.kw.get("batch") == "round":
            s = st.shape(*r.shape, sms())
            groups, _ = grid(s.lv + s.K, UNCAPPED)
            assert s.batch == groups + 1 and grid(s.lv + s.K, s.batch) == (groups, 2)


def finish_and_check(r, oracle_mod, dp, env):
    bad = r.mismatches()
    if bad:
        i, text = r.report(bad)
        verdict = replay(r, i, dp, env)
        pytest.fail(text + "\n" + verdict)
    assert not r.objs
    grown, regrown = cp.growth_steps(r.steps, r.shape)
    for X in cp.SCRATCH:   # the growths the program guarantees happened: the context's device bytes grew at those steps
        for i in grown[X] + regrown[X]:
            assert r.grew[i], "%s: %s did not grow at step %d %r" % (r.name, X, i, r.steps[i])
    r.c._chk(r.c._l.dpfhe_context_trim(r.c._h))
    assert r.c.device_bytes() - r.base in kept_after_trim(r.steps, r.shape)
    assert r.peak < cp.BUDGET, r.peak


def kept_after_trim(steps, shape):
    """the device bytes a context keeps through a trim once the program ran (deeppowers_b200/csrc/abi.cu): the hoisted-rotation
    constants M, kprime and delta (ensure_hoist_consts) after a per-limb hoisted rotation, the special-prime accumulator rows of
    the hybrid and grouped kernels (ensure_hyb) after their first call, the dropped limb's rows of multiply-and-rescale
    (ensure_tau_drop) after its first call; [allowed totals]"""
    log_n, L = shape
    N, slots = 1 << log_n, 4 * sms()
    fns = {s.fn for s in steps if s.kind in ("call", "create", "apply")}
    hoist = 8 * (3 * L * N + L * L) if fns & {"dpfhe_rotate_hoisted", "dpfhe_linear_create"} else 0
    hyb = (slots // 2 + 1) * 6 * N * 8 + slots * 4 * N * 8
    tau = (slots // 3 + 1) * 4 * N * 8
    if any("rescale" in fn for fn in fns):
        return [hoist + hyb + tau]
    return [hoist + hyb, hoist + hyb + tau]


def replay(r, upto, dp, env):
    """the program up to step `upto` on a new context, synchronised after every step: does the step still fail?"""
    c = dp.Context(*r.shape)
    q = Runner(r.name + " (serialised replay)", c, r.plan, r.seed)
    try:
        q.load()
        q.run(upto, serial=True)
        bad = [m for m in q.mismatches(upto) if m[0] == upto]
    finally:
        q.finish()
        c.close()
    return ("serialised replay: step %d still fails: context state" % upto if bad else
            "serialised replay: step %d passes: ordering between streams" % upto)


# ---- one program per context -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,shape,seed,n_steps,env", PROGRAMS, ids=[p[0] for p in PROGRAMS])
def test_program(dp, oracle_mod, monkeypatch, name, shape, seed, n_steps, env):
    torch.cuda.empty_cache()
    t0 = time.time()
    r = run_program(name, dp, oracle_mod, shape, seed, n_steps, monkeypatch, env)
    print("%s: %d steps, peak %.2f GiB, %.1f s" % (name, len(r.steps), r.peak / 2**30, time.time() - t0))
    torch.cuda.empty_cache()


def test_two_contexts_interleaved(dp, oracle_mod):
    """two programs on two contexts of one device, issued step by step in turn from one thread"""
    torch.cuda.empty_cache()
    rs = []
    try:
        for name, shape, seed in (("a", (12, 7), 21), ("b", (13, 6), 22)):
            steps = cp.program(seed, shape, 0)
            rs.append(Runner(name, dp.Context(*shape), Plan(steps, shape, Refs(oracle_mod, *shape), sms()), seed))
        for r in rs:
            r.load()
        n = max(len(r.steps) for r in rs)
        for i in range(n):
            for r in rs:
                if i < len(r.steps):
                    r.step(i)
        torch.cuda.synchronize()
        for r in rs:
            finish_and_check(r, oracle_mod, dp, {})
    finally:
        for r in rs:
            r.finish()
            r.c.close()
    torch.cuda.empty_cache()


def test_two_contexts_two_threads(dp, oracle_mod):
    """two programs, each on its own context driven by its own host thread"""
    torch.cuda.empty_cache()
    rs = []
    try:
        for name, shape, seed in (("a", (12, 7), 31), ("b", (13, 6), 32)):
            steps = cp.program(seed, shape, 0)
            rs.append(Runner(name, dp.Context(*shape), Plan(steps, shape, Refs(oracle_mod, *shape), sms()), seed))
        for r in rs:
            r.load()
        errors = []

        def drive(r):
            try:
                r.run()
            except BaseException as e:  # noqa: BLE001  (re-raised by the test thread)
                errors.append(e)

        ts = [threading.Thread(target=drive, args=(r,)) for r in rs]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        if errors:
            raise errors[0]
        torch.cuda.synchronize()
        for r in rs:
            finish_and_check(r, oracle_mod, dp, {})
    finally:
        for r in rs:
            r.finish()
            r.c.close()
    torch.cuda.empty_cache()
