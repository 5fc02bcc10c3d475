"""The memory contract of the entry points of include/dpfhe_compact.h (DESIGN.md §2.24): one row per entry point, in the form of
tests/memory_contract.py's rows and run by the same harness (tests/test_gpu_memory_contract.py: run_case, the arena between guard
words).  The rows use bits = 32, so that a compact ciphertext is N words, one polynomial's worth of the harness's sizes.  The
references are tests/compact_ref.py's restatement.  The download takes a device input and gives a host output: its row places the
input in the device arena and the output in the host arena, and the harness checks the guard words and the unchanged input on both
sides.  The decryption rows take a ternary secret and random packed words.  Test infrastructure."""
import numpy as np

import compact_ref as cr
import keys_ref as kr
from memory_contract import BATCH, CT, KEY, ONE, OPERAND, OUTPUT, SEED, T, ALL, Row, dev, hst

BITS = 32


def _secret(s, rng):
    import oracle
    return kr.secret(oracle.Oracle(s.log_n, s.L), SEED)


def _words(s, rng):
    return rng.integers(0, 1 << 64, size=(s.batch, 2, s.N * BITS // 64), dtype=np.uint64)


def _compact_ref(R, s, x):
    return {"cct": cr.compact(R.oracle_mod, R.o, s.lv, BITS, T, x["ct"])}


def _decrypt_ref(R, s, x):
    sk = np.asarray(x["sk"]).reshape(s.L, s.N)
    return {"pt": cr.decrypt(R.o, BITS, T, sk, np.asarray(x["cct"]).reshape(s.batch, 2, -1))}


def build_rows():
    """{function name: Row} of every buffer entry point of dpfhe_compact.h"""
    gen = {"sk": _secret, "cct": _words}
    rows = [
        Row("dpfhe_compact_ciphertexts", [dev("ct", OPERAND, CT), dev("cct", OUTPUT, BATCH, ONE)],
            lambda c, s, p: c.compact_ciphertexts(s.lv, BITS, T, p["ct"], p["cct"], s.batch), _compact_ref),
        Row("dpfhe_download_compact_ciphertexts", [dev("ct", OPERAND, CT), hst("cct", OUTPUT, BATCH, ONE)],
            lambda c, s, p: c.download_compact_ciphertexts(s.lv, BITS, T, p["ct"], p["cct"], s.batch), _compact_ref,
            note="device input in the device arena, host output in the host arena"),
        Row("dpfhe_decrypt_compact", [dev("sk", KEY, ONE, ALL), dev("cct", OPERAND, BATCH, ONE), dev("pt", OUTPUT, BATCH, ONE)],
            lambda c, s, p: c.decrypt_compact(BITS, T, p["sk"], p["cct"], p["pt"], s.batch), _decrypt_ref, gen=gen),
        Row("dpfhe_decrypt_compact_host", [hst("sk", KEY, ONE, ALL), hst("cct", OPERAND, BATCH, ONE), hst("pt", OUTPUT, BATCH, ONE)],
            lambda c, s, p: c.decrypt_compact_host(BITS, T, p["sk"], p["cct"], p["pt"]), _decrypt_ref, gen=gen),
    ]
    return {r.fn: r for r in rows}
