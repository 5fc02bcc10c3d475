"""The memory contract of the entry points of include/dpfhe_level.h (DESIGN.md §2.22): one row per entry point that takes device or host
buffers, in the form of tests/memory_contract.py's rows and run by the same harness (tests/test_gpu_memory_contract.py: run_case, the
arena between guard words).  The keyless level calls are referred to the oracle over the prefix basis q_0 .. q_{lv-1}; the
polynomial evaluators at a level to the restatements on {q_0 .. q_{lv-1}, p_0 .. p_{K-1}} with the restricted key.  Test
infrastructure."""
import ctypes as C

import numpy as np

import bgv_ref
import ckks_ref
import keys_ref
import polyeval_ref as pr
import public_key_ref
from memory_contract import (ALL, BATCH, COEFFS, CT, GROUPED_KEY, KEY, LV1, ONE, OPERAND, OUTPUT, SCALE, SEED, SLOTS, T, Buf, Row, _stream,
                             bgv_slots, ckks_slots, cts, dev, hst, level_key, table)


def prefix_oracle(R, s):
    """the oracle of a keyless level call's basis: the first lv moduli q_0 .. q_{lv-1} (DESIGN.md §2.22)"""
    return R.o if s.lv == s.L else R.sub(list(R.o.moduli)[:s.lv])


def _prefix_rows():
    """the keyless calls at level lv on the top-level context: the call on a context over the first lv moduli.  The secret is its
    first lv rows; the public key is the top-level one [2][L][N].  The BGV encoders take the case's t (65537 by default: 1 mod 2N at
    every N)"""
    rows = []
    rows.append(Row("dpfhe_ckks_encode_level", [dev("slots", OPERAND, SLOTS, ONE), dev("pt", OUTPUT, BATCH)],
                    lambda c, s, p: c._chk(c._l.dpfhe_ckks_encode_level(c._h, s.lv, C.c_void_p(p["slots"]), C.c_void_p(p["pt"]), s.batch, SCALE,
                                                                        _stream())),
                    lambda R, s, x: {"pt": ckks_ref.encode(prefix_oracle(R, s), x["slots"].view(np.complex128).reshape(s.batch, s.N // 2), SCALE)},
                    gen={"slots": ckks_slots}))
    rows.append(Row("dpfhe_ckks_decode_level", [dev("pt", OPERAND, BATCH), dev("slots", OUTPUT, SLOTS, ONE)],
                    lambda c, s, p: c._chk(c._l.dpfhe_ckks_decode_level(c._h, s.lv, C.c_void_p(p["pt"]), C.c_void_p(p["slots"]), s.batch, SCALE,
                                                                        _stream())),
                    lambda R, s, x: {"slots": ckks_ref.decode(prefix_oracle(R, s), x["pt"], SCALE).view(np.uint64)}))
    rows.append(Row("dpfhe_bgv_encode_level", [dev("slots", OPERAND, SLOTS, ONE), dev("pt", OUTPUT, BATCH)],
                    lambda c, s, p: c.bgv_encode_level(s.lv, p["slots"], p["pt"], s.batch, s.t),
                    lambda R, s, x: {"pt": bgv_ref.encode(prefix_oracle(R, s), x["slots"].view(np.int64).reshape(s.batch, 2, s.N // 2), s.t)},
                    gen={"slots": bgv_slots}))
    rows.append(Row("dpfhe_bgv_decode_level", [dev("pt", OPERAND, BATCH), dev("slots", OUTPUT, SLOTS, ONE)],
                    lambda c, s, p: c.bgv_decode_level(s.lv, p["pt"], p["slots"], s.batch, s.t),
                    lambda R, s, x: {"slots": bgv_ref.decode(prefix_oracle(R, s), x["pt"], s.t)}))
    sk = lambda: dev("sk", KEY, ONE)
    rows.append(Row("dpfhe_encrypt_level", [sk(), dev("pt", OPERAND, BATCH), dev("ct", OUTPUT, CT)],
                    lambda c, s, p: c.encrypt_level(s.lv, T, p["sk"], SEED, 11, p["pt"], p["ct"], s.batch),
                    lambda R, s, x: {"ct": keys_ref.encrypt(prefix_oracle(R, s), T, x["sk"][0], SEED, 11, x["pt"])}))
    rows.append(Row("dpfhe_decrypt_level", [sk(), dev("ct", OPERAND, lambda s: s.n_comp * s.batch), dev("pt", OUTPUT, BATCH)],
                    lambda c, s, p: c.decrypt_level(s.lv, p["sk"], p["ct"], s.n_comp, p["pt"], s.batch),
                    lambda R, s, x: {"pt": keys_ref.decrypt(prefix_oracle(R, s), x["sk"][0], x["ct"].reshape(s.batch, s.n_comp, s.lv, s.N))}))
    rows.append(Row("dpfhe_encrypt_public_level", [dev("pk", KEY, lambda s: 2, ALL), dev("pt", OPERAND, BATCH), dev("ct", OUTPUT, CT)],
                    lambda c, s, p: c.encrypt_public_level(s.lv, T, p["pk"], SEED, 3, p["pt"], p["ct"], s.batch),
                    lambda R, s, x: {"ct": public_key_ref.encrypt_public(prefix_oracle(R, s), T,
                                                                         np.ascontiguousarray(x["pk"].reshape(2, s.L, s.N)[:, :s.lv]), SEED, 3, x["pt"])}))
    rows.append(Row("dpfhe_ct_mul_plain_level", [dev("ct", OPERAND, CT), dev("pt", OPERAND, ONE), dev("out", OUTPUT, CT)],
                    lambda c, s, p: c.ct_mul_plain_level(s.lv, p["ct"], p["pt"], p["out"], s.batch),
                    lambda R, s, x: {"out": prefix_oracle(R, s).ct_mul_plain(cts(x, "ct", s), x["pt"][0])}))
    rows.append(Row("dpfhe_ct_lincomb_level", [dev("cts", OPERAND, CT, count=lambda s: s.n_terms), dev("out", OUTPUT, CT)],
                    lambda c, s, p: c.ct_lincomb_level(s.lv, p["cts"], COEFFS[:s.n_terms], -7, p["out"], s.batch),
                    lambda R, s, x: {"out": pr.lincomb(list(R.o.moduli)[:s.lv], table(x, "cts", s), COEFFS[:s.n_terms], -7)}))
    rows.append(Row("dpfhe_ct_add_plain_level", [dev("ct", OPERAND, CT), dev("pt", OPERAND, ONE), dev("out", OUTPUT, CT)],
                    lambda c, s, p: c.ct_add_plain_level(s.lv, p["ct"], p["pt"], p["out"], s.batch),
                    lambda R, s, x: {"out": pr.lincomb(list(R.o.moduli)[:s.lv], [cts(x, "ct", s)], [1], 0, x["pt"][0])}))
    rows.append(Row("dpfhe_mod_switch_down_level", [dev("in", OPERAND, CT), dev("out", OUTPUT, CT, LV1)],
                    lambda c, s, p: c.mod_switch_down_level(s.lv, p["in"], p["out"], 2 * s.batch, s.t),
                    lambda R, s, x: {"out": prefix_oracle(R, s).mod_switch_down(x["in"], s.t)}))
    return rows


def _prefix_host_rows(device):
    """the host forms of the keyless level calls: the buffers of the device form as host arrays"""
    rows = []

    def like(fn, run):
        d = device[fn[:-len("_host")]]
        rows.append(Row(fn, [Buf(b.name, b.role, b.items, b.limbs, host=True) for b in d.bufs], run, d.ref, gen=d.gen))

    like("dpfhe_ckks_encode_level_host", lambda c, s, p: c.ckks_encode_level_host(s.lv, p["slots"].view(np.complex128), p["pt"], SCALE))
    like("dpfhe_ckks_decode_level_host", lambda c, s, p: c.ckks_decode_level_host(s.lv, p["pt"], p["slots"].view(np.complex128), SCALE))
    like("dpfhe_bgv_encode_level_host", lambda c, s, p: c.bgv_encode_level_host(s.lv, p["slots"].view(np.int64), p["pt"], s.t))
    like("dpfhe_bgv_decode_level_host", lambda c, s, p: c.bgv_decode_level_host(s.lv, p["pt"], p["slots"].view(np.int64), s.t))
    like("dpfhe_encrypt_level_host", lambda c, s, p: c.encrypt_level_host(s.lv, T, p["sk"], SEED, 11, p["pt"], p["ct"]))
    like("dpfhe_decrypt_level_host", lambda c, s, p: c.decrypt_level_host(s.lv, p["sk"], p["ct"], s.n_comp, p["pt"]))
    like("dpfhe_encrypt_public_level_host", lambda c, s, p: c.encrypt_public_level_host(s.lv, T, p["pk"], SEED, 3, p["pt"], p["ct"]))
    return rows


def _polyeval_level_rows():
    """the polynomial evaluators at level lv (DESIGN.md §2.22): the top-level object on {q_0 .. q_{lv-1}, p_0 .. p_{K-1}} with the
    restricted key; BGV p = 3 + 5x^2 + x^3 (D = 2), CKKS a quadratic (D = 1)"""
    import ckks_polyeval_ref as cpr
    coeffs, ccoeffs = [3, 0, 5, 1], [0.5, -0.25, 0.125]

    def chain(R, s):
        m = list(R.o.moduli)
        return pr.Chain(R.oracle_mod, s.log_n, m[:s.lv] + m[s.Lq:], s.K)

    def bgv_run(c, s, p):
        from deeppowers_b200 import PolyEval
        pe = PolyEval(c, s.K, T, coeffs, p["key"], level=s.lv)
        try:
            pe.apply(p["ct"], p["out"], s.batch)
            c.synchronize()
        finally:
            pe.close()

    def ckks_run(c, s, p):
        from deeppowers_b200 import PolyEval
        pe = PolyEval.ckks(c, s.K, ccoeffs, SCALE, p["key"], level=s.lv)
        try:
            pe.apply(p["ct"], p["out"], s.batch)
            c.synchronize()
        finally:
            pe.close()

    return [Row("dpfhe_polyeval_create_grouped_level", [hst("key", KEY, GROUPED_KEY, ALL), dev("ct", OPERAND, CT), dev("out", OUTPUT, CT, lambda s: s.lv - 2)],
                bgv_run, lambda R, s, x: {"out": pr.polyeval(chain(R, s), T, coeffs, cts(x, "ct", s), level_key(s, x["key"]))}),
            Row("dpfhe_polyeval_create_ckks_level", [hst("key", KEY, GROUPED_KEY, ALL), dev("ct", OPERAND, CT), dev("out", OUTPUT, CT, lambda s: s.lv - 2)],
                ckks_run, lambda R, s, x: {"out": cpr.polyeval(chain(R, s), ccoeffs, SCALE, cts(x, "ct", s), level_key(s, x["key"]), SCALE)})]


def build_rows():
    """{function name: Row} of every buffer entry point of dpfhe_level.h"""
    device = {r.fn: r for r in _prefix_rows()}
    rows = dict(device)
    for r in _prefix_host_rows(device) + _polyeval_level_rows():
        rows[r.fn] = r
    return rows
