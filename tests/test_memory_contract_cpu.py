"""The role table of tests/memory_contract.py against include/dpfhe.h: every entry point with a device (d_*) or host (h_*) buffer
parameter has a row or a reason to have none, so that a call added later cannot slip past the memory-contract tests."""
import os

import pytest

import memory_contract as mc

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dpfhe.h")


@pytest.fixture(scope="module")
def header():
    with open(HEADER) as f:
        return f.read()


@pytest.fixture(scope="module")
def rows():
    return mc.build_rows()


def test_parser_sees_the_buffer_parameters(header):
    fns = mc.header_functions(header)
    assert fns["dpfhe_ct_mul_relin"] == ["ctx", "d_a", "d_b", "d_evk", "d_out", "batch", "stream"]
    assert fns["dpfhe_ipc_open"] == ["ctx", "handle", "d_out"]
    assert "dpfhe_launch_count" in fns and "dpfhe_launch_count" not in mc.buffer_functions(header)
    assert len(mc.buffer_functions(header)) > 80


def test_every_buffer_call_has_a_row_or_a_reason(header, rows):
    need = set(mc.buffer_functions(header))
    missing = sorted(need - set(rows) - set(mc.EXEMPT))
    assert not missing, "entry points without a memory-contract row: %s" % missing
    assert not set(rows) & set(mc.EXEMPT)
    stale = sorted((set(rows) | set(mc.EXEMPT)) - set(mc.header_functions(header)))
    assert not stale, "rows of functions the header no longer declares: %s" % stale
    assert all(mc.EXEMPT.values())


@pytest.mark.parametrize("s", [mc.Shape(12, 2, 0, 3, n_rot=2, n_terms=3), mc.Shape(13, 7, 2, 5, level=3, n_rot=2, n_terms=3)], ids=repr)
def test_rows_are_well_formed(rows, s):
    """every row has an output, distinct buffer names and aliases that name its own buffers: an output with an operand"""
    for fn, row in rows.items():
        names = [n for b in row.bufs for n in b.names(s)]
        assert len(names) == len(set(names)), fn
        assert row.outputs(), fn
        assert all(b.role in (mc.OPERAND, mc.KEY, mc.OUTPUT, mc.INPLACE) for b in row.bufs), fn
        assert not s.K or all(b.words(s) > 0 for b in row.bufs), fn   # the objects need special primes
        for alias in row.aliases:
            roles = [next(b.role for b in row.bufs if b.name == a.split(".")[0]) for a in alias]
            assert roles[0] == mc.OUTPUT and all(r == mc.OPERAND for r in roles[1:]), (fn, alias)


def test_aliases_are_those_of_the_header(rows):
    got = {fn: sorted(r.aliases) for fn, r in rows.items() if r.aliases}
    assert got == {"dpfhe_poly_mul_pointwise": sorted([("out", "a"), ("out", "b"), ("out", "a", "b")]),
                   "dpfhe_poly_add": sorted([("out", "a"), ("out", "b"), ("out", "a", "b")]),
                   "dpfhe_ct_mul_plain": [("out", "ct")], "dpfhe_ct_add_plain": [("out", "ct")],
                   "dpfhe_ct_lincomb": [("out", "cts.0"), ("out", "cts.1")]}


def test_keys_are_keys(rows):
    """the buffers every work item reads for the whole launch carry the key role, which the overlap tests pair with each output"""
    for fn, row in rows.items():
        for b in row.bufs:
            if b.name in ("key", "gks", "gk_baby", "gk_giant", "pk", "sk") and b.role != mc.OUTPUT:   # keygen writes them
                assert b.role == mc.KEY, (fn, b.name)
