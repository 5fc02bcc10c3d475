"""include/dpfhe_level.h against its memory-contract rows (tests/level_contract.py) and its bindings, without a GPU: dpfhe.h includes it;
every entry point with a device (d_*) or host (h_*) buffer has a row, and every row an entry point; the rows are well formed and the
keys carry the key role; the Python binding table of the header (deeppowers_b200/_lib.py: LEVEL_SYMBOLS) is exactly what it declares,
and libdpfhe.so exports it.  The same checks as tests/test_memory_contract_cpu.py and tests/test_host_logic.py make for dpfhe.h, so that
a call of the level header cannot slip past the memory-contract tests either."""
import os
import re

import pytest

import level_contract as lc
import memory_contract as mc

INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")


@pytest.fixture(scope="module")
def header():
    with open(os.path.join(INCLUDE, "dpfhe_level.h")) as f:
        return f.read()


@pytest.fixture(scope="module")
def rows():
    return lc.build_rows()


def test_dpfhe_h_includes_the_level_header(header):
    with open(os.path.join(INCLUDE, "dpfhe.h")) as f:
        core = f.read()
    assert '#include "dpfhe_level.h"' in core
    assert not set(mc.header_functions(core)) & set(mc.header_functions(header)), "an entry point declared in both headers"


def test_every_buffer_call_has_a_row(header, rows):
    need = set(mc.buffer_functions(header))
    assert len(need) == 20
    assert not sorted(need - set(rows)), "entry points without a memory-contract row: %s" % sorted(need - set(rows))
    assert not sorted(set(rows) - set(mc.header_functions(header))), "rows of functions the header does not declare"


@pytest.mark.parametrize("s", [mc.Shape(12, 4, 0, 3, level=2, n_terms=3), mc.Shape(13, 7, 2, 5, level=3, n_terms=3)], ids=repr)
def test_rows_are_well_formed(rows, s):
    for fn, row in rows.items():
        names = [n for b in row.bufs for n in b.names(s)]
        assert len(names) == len(set(names)), fn
        assert row.outputs(), fn
        assert all(b.role in (mc.OPERAND, mc.KEY, mc.OUTPUT, mc.INPLACE) for b in row.bufs), fn
        assert not row.aliases, fn
        for b in row.bufs:
            if b.name in ("key", "pk", "sk"):
                assert b.role == mc.KEY, (fn, b.name)


def test_bindings_are_the_header(header):
    import deeppowers_b200
    from deeppowers_b200 import _lib
    declared = set(re.findall(r"\b(dpfhe_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", " ", header, flags=re.S)))
    assert declared == set(_lib.LEVEL_SYMBOLS), declared ^ set(_lib.LEVEL_SYMBOLS)
    assert not declared & set(_lib.SYMBOLS)
    lib = deeppowers_b200.load_library()
    for name in sorted(declared):
        assert hasattr(lib, name), name
