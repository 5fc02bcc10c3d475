"""include/dpfhe_compact.h against its memory-contract rows (tests/compact_contract.py) and its bindings, without a GPU: dpfhe.h includes
it; every entry point with a device (d_*) or host (h_*) buffer has a row, and every row an entry point; the rows are well formed and
the secret carries the key role; the Python binding table of the header (deeppowers_b200/_lib.py: COMPACT_SYMBOLS) is exactly what it
declares, and libdpfhe.so exports it.  The checks tests/test_seeded_contract_cpu.py makes for dpfhe_seeded.h."""
import os
import re

import pytest

import compact_contract as ccn
import memory_contract as mc

INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")


@pytest.fixture(scope="module")
def header():
    with open(os.path.join(INCLUDE, "dpfhe_compact.h")) as f:
        return f.read()


@pytest.fixture(scope="module")
def rows():
    return ccn.build_rows()


def test_dpfhe_h_includes_the_compact_header(header):
    with open(os.path.join(INCLUDE, "dpfhe.h")) as f:
        core = f.read()
    assert '#include "dpfhe_compact.h"' in core
    for other in ("dpfhe.h", "dpfhe_level.h", "dpfhe_seeded.h"):
        with open(os.path.join(INCLUDE, other)) as f:
            text = f.read()
        assert not set(mc.header_functions(text)) & set(mc.header_functions(header)), "an entry point declared in two headers"


def test_every_buffer_call_has_a_row(header, rows):
    need = set(mc.buffer_functions(header))
    assert len(need) == 4
    assert need == set(rows) == set(mc.header_functions(header))


@pytest.mark.parametrize("s", [mc.Shape(12, 3, 0, 3), mc.Shape(13, 6, 2, 2, level=3)], ids=repr)
def test_rows_are_well_formed(rows, s):
    for fn, row in rows.items():
        names = [n for b in row.bufs for n in b.names(s)]
        assert len(names) == len(set(names)), fn
        assert len(row.outputs()) == 1, fn
        assert all(b.role in (mc.OPERAND, mc.KEY, mc.OUTPUT) for b in row.bufs), fn
        assert not row.aliases, fn
        assert row.host == fn.endswith("_host") or "download" in fn, fn
        for b in row.bufs:
            if b.name == "sk":
                assert b.role == mc.KEY, (fn, b.name)
        out = row.outputs()[0]
        # a compact ciphertext of ccn.BITS bits is N bits / 32 words: one [N] row per ciphertext
        if out.name == "cct":
            assert out.words(s) == s.batch * s.N * ccn.BITS // 32, fn


def test_bindings_are_the_header(header):
    import deeppowers_b200
    from deeppowers_b200 import _lib
    declared = set(re.findall(r"\b(dpfhe_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", " ", header, flags=re.S)))
    assert declared == set(_lib.COMPACT_SYMBOLS), declared ^ set(_lib.COMPACT_SYMBOLS)
    assert not declared & (set(_lib.SYMBOLS) | set(_lib.LEVEL_SYMBOLS) | set(_lib.SEEDED_SYMBOLS))
    lib = deeppowers_b200.load_library()
    for name in sorted(declared):
        assert hasattr(lib, name), name
