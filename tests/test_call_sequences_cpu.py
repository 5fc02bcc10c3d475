"""The call programs of tests/call_program.py, without a GPU: a seed gives one program; every call is a row of the contract tables at
a shape the context realises and that the tables' own well-formedness checks accept; every program the GPU file runs has each
guaranteed transition and stays within its device-memory budget; and removing any one guarantee from a program is noticed."""
import pytest

import call_program as cp
import memory_contract as mc

# the programs of tests/test_gpu_call_sequences.py: (shape, seed, n_steps)
GPU_PROGRAMS = [((12, 7), 11, 400), ((13, 6), 12, 320), ((14, 4), 13, 200), ((12, 7), 21, 0), ((13, 6), 22, 0), ((12, 7), 31, 0),
                ((13, 6), 32, 0)]
IDS = ["N%d-L%d-seed%d" % (1 << p[0][0], p[0][1], p[1]) for p in GPU_PROGRAMS]


@pytest.mark.parametrize("shape,seed,n", GPU_PROGRAMS, ids=IDS)
def test_same_seed_same_program(shape, seed, n):
    a, b = cp.program(seed, shape, n), cp.program(seed, shape, n)
    assert [s.key() for s in a] == [s.key() for s in b]
    assert [s.key() for s in a] != [s.key() for s in cp.program(seed + 1, shape, n)]


def _well_formed(fn, row, s):
    """the checks of test_{memory,level,seeded,compact}_contract_cpu.py::test_rows_are_well_formed at one shape"""
    names = [n for b in row.bufs for n in b.names(s)]
    assert len(names) == len(set(names)), fn
    assert row.outputs(), fn
    assert all(b.role in (mc.OPERAND, mc.KEY, mc.OUTPUT, mc.INPLACE) for b in row.bufs), fn
    assert all(b.words(s) > 0 for b in row.bufs), (fn, s)
    for b in row.bufs:
        if b.name in ("key", "pk", "sk") and b.role != mc.OUTPUT:
            assert b.role == mc.KEY, (fn, b.name)
    if fn in cp.SEEDED or fn in cp.COMPACT:
        assert len(row.outputs()) == 1, fn


@pytest.mark.parametrize("shape,seed,n", GPU_PROGRAMS, ids=IDS)
def test_every_call_is_a_realisable_row(shape, seed, n):
    log_n, L = shape
    for i, st in enumerate(cp.program(seed, shape, n)):
        if st.kind not in ("call", "create", "apply"):
            continue
        assert st.fn in cp.ROWS and not cp.ROWS[st.fn].multi, st
        s = st.shape(log_n, L)
        assert (s.log_n, s.L) == shape
        assert {"K": s.K, "level": s.level} in [dict(K=d["K"], level=d.get("level")) for d in cp.shapes(st.fn, log_n, L)], (i, st)
        assert s.K in (0, 1, 2, 3) and 2 * s.K <= L and 1 <= s.lv <= L
        assert s.t in cp.T_PAIR and (s.t - 1) % (2 * s.N) == 0
        assert s.batch >= 1 and st.stream in (0, 1, 2)
        _well_formed(st.fn, cp.ROWS[st.fn], s)
        if st.chain:
            j, pn, cn = st.chain
            assert j < i and cp.chainable(cp.program(seed, shape, n)[j], pn, st, cn, log_n, L)


@pytest.mark.parametrize("shape,seed,n", GPU_PROGRAMS, ids=IDS)
def test_every_guarantee_holds(shape, seed, n):
    assert cp.check_guarantees(cp.program(seed, shape, n), shape) == []


@pytest.mark.parametrize("shape,seed,n", GPU_PROGRAMS, ids=IDS)
def test_footprint_under_budget(shape, seed, n):
    steps = cp.program(seed, shape, n)
    assert cp.footprint(steps, shape) < cp.BUDGET
    assert cp.footprint(steps, shape, sms=cp.SMS) >= 8 * sum(w for st in steps for _, w in cp.device_buffers(st, *shape))


def test_objects_live_across_steps():
    for shape, seed, n in GPU_PROGRAMS:
        steps = cp.program(seed, shape, n)
        for o in {s.obj for s in steps if s.kind == "create"}:
            at = [i for i, s in enumerate(steps) if s.obj == o]
            kinds = [steps[i].kind for i in at]
            assert kinds[0] == "create" and kinds[-1] == "destroy" and kinds.count("apply") >= 1
            assert any(steps[k].kind == "call" for k in range(at[0], at[-1]))


def test_round_batch_is_one_past_a_grid_round():
    """the N = 16384 program has one key-switch batch one ciphertext past a full round of the persistent grid"""
    steps = cp.program(13, (14, 4), 200)
    r = [s for s in steps if s.kw.get("batch") == "round"]
    assert len(r) == 1
    s = r[0].shape(14, 4)
    group = s.lv + s.K
    assert (s.batch - 1) * group <= 3 * cp.SMS < s.batch * group


# every guarantee, removed from the program (its steps replaced by no-ops, which keeps the chains' indices): the check notices
def _without(pred):
    return lambda steps: [cp.Step("noop") if s.kind != "noop" and pred(s) else s for s in steps]


def _call(fns=None, **kw):
    return lambda s: s.kind == "call" and (fns is None or s.fn in fns) and all(f(s) for f in kw.values())


MUTATIONS = {
    "growth": _without(_call(["dpfhe_mod_down_special"])),
    "trim": _without(lambda s: s.kind == "trim"),
    "bgv_t": _without(_call(["dpfhe_bgv_decode_level", "dpfhe_bgv_decode"])),
    "levels": _without(_call(cp.KS_LEVEL, at_k=lambda s: s.kw.get("level") == s.kw.get("K"))),
    "keyless": _without(_call(cp.KEYLESS, at_1=lambda s: s.kw.get("level") == 1)),
    "host": _without(_call(host=lambda s: cp.ROWS[s.fn].host)),
    "short_chunk": _without(_call(["dpfhe_ct_add_plain_host"], big=lambda s: s.kw["batch"] > 3)),
    "chain": lambda steps: [cp.Step(s.kind, s.fn, s.kw, s.stream, s.seed, None, s.obj) for s in steps],
    "object": _without(lambda s: s.kind == "apply"),
}


@pytest.mark.parametrize("what", sorted(MUTATIONS))
def test_a_missing_guarantee_is_noticed(what):
    for shape, seed, n in GPU_PROGRAMS[:3]:
        steps = cp.program(seed, shape, n)
        assert cp.check_guarantees(MUTATIONS[what](steps), shape), (what, shape)
