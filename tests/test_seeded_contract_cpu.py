"""include/dpfhe_seeded.h against its memory-contract rows (tests/seeded_contract.py) and its bindings, without a GPU: dpfhe.h includes
it; every entry point with a device (d_*) or host (h_*) buffer has a row, and every row an entry point; the rows are well formed and
the secret carries the key role; the Python binding table of the header (deeppowers_b200/_lib.py: SEEDED_SYMBOLS) is exactly what it
declares, and libdpfhe.so exports it.  The checks tests/test_level_contract_cpu.py makes for dpfhe_level.h."""
import os
import re

import pytest

import memory_contract as mc
import seeded_contract as scn

INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")


@pytest.fixture(scope="module")
def header():
    with open(os.path.join(INCLUDE, "dpfhe_seeded.h")) as f:
        return f.read()


@pytest.fixture(scope="module")
def rows():
    return scn.build_rows()


def test_dpfhe_h_includes_the_seeded_header(header):
    with open(os.path.join(INCLUDE, "dpfhe.h")) as f:
        core = f.read()
    with open(os.path.join(INCLUDE, "dpfhe_level.h")) as f:
        level = f.read()
    assert '#include "dpfhe_seeded.h"' in core
    for other in (core, level):
        assert not set(mc.header_functions(other)) & set(mc.header_functions(header)), "an entry point declared in two headers"


def test_every_buffer_call_has_a_row(header, rows):
    need = set(mc.buffer_functions(header))
    assert len(need) == 15
    assert not sorted(need - set(rows)), "entry points without a memory-contract row: %s" % sorted(need - set(rows))
    assert not sorted(set(rows) - set(mc.header_functions(header))), "rows of functions the header does not declare"
    assert set(mc.header_functions(header)) - need == {"dpfhe_seeded_public_seed"}


@pytest.mark.parametrize("s", [mc.Shape(12, 3, 0, 3, n_rot=3), mc.Shape(13, 6, 2, 2, level=3, n_rot=2)], ids=repr)
def test_rows_are_well_formed(rows, s):
    for fn, row in rows.items():
        names = [n for b in row.bufs for n in b.names(s)]
        assert len(names) == len(set(names)), fn
        assert len(row.outputs()) == 1, fn
        assert all(b.role in (mc.OPERAND, mc.KEY, mc.OUTPUT) for b in row.bufs), fn
        assert not row.aliases, fn
        assert row.host == fn.endswith("_host") or "upload" in fn, fn
        for b in row.bufs:
            if b.name == "sk":
                assert b.role == mc.KEY, (fn, b.name)


def test_bindings_are_the_header(header):
    import deeppowers_b200
    from deeppowers_b200 import _lib
    declared = set(re.findall(r"\b(dpfhe_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", " ", header, flags=re.S)))
    assert declared == set(_lib.SEEDED_SYMBOLS), declared ^ set(_lib.SEEDED_SYMBOLS)
    assert not declared & (set(_lib.SYMBOLS) | set(_lib.LEVEL_SYMBOLS))
    lib = deeppowers_b200.load_library()
    for name in sorted(declared):
        assert hasattr(lib, name), name
