"""The memory contract of the entry points of include/dpfhe_seeded.h (DESIGN.md §2.23): one row per entry point that takes device or host
buffers, in the form of tests/memory_contract.py's rows and run by the same harness (tests/test_gpu_memory_contract.py: run_case, the
arena between guard words).  The references are tests/seeded_ref.py's restatement, over the prefix basis q_0 .. q_{lv-1} for the
level forms.  The two uploads take a host input and give a device output; their rows place both in a host arena, and the call writes
into a device tensor of its own whose words are copied back into the arena's output.  Test infrastructure."""
import numpy as np

import seeded_ref as sr
from memory_contract import ALL, BATCH, CT, KEY, ONE, OPERAND, OUTPUT, SEED, T, Row, dev, gals, hst

ITEM0 = (1 << 32) - 1   # item numbers of the ciphertext rows cross 2^32
A_SEED = sr.public_seed(SEED)
DIG = lambda s: s.n_rot * s.dnum          # the b rows of n_rot keys [n_rot][dnum][L][N]
KEYS = lambda s: 2 * s.n_rot * s.dnum     # n_rot keys [n_rot][dnum][2][L][N]


def prefix_oracle(R, s):
    return R.o if s.lv == s.L else R.sub(list(R.o.moduli)[:s.lv])


def items(s):
    """the item numbers of a case's keys: the relinearisation key (0), then Galois elements"""
    return [0] + gals(s)[:s.n_rot - 1]


def _key_ref(R, s, sk):
    sk = np.ascontiguousarray(sk.reshape(s.L, s.N))
    its = items(s)
    out = [sr.relin_key_seeded(R.o, s.K, T, sk, SEED)]
    if len(its) > 1:
        out += list(sr.galois_keys_seeded(R.o, s.K, T, sk, SEED, its[1:]))
    return np.stack(out)


def _via_device(c, p, name, shape, call):
    """runs call(device output tensor) and copies its words into the host arena's output p[name]"""
    import torch
    out = torch.empty(shape, dtype=torch.int64, device="cuda")
    call(out)
    torch.cuda.synchronize()
    p[name][...] = out.cpu().numpy().view(np.uint64).reshape(p[name].shape)


def build_rows():
    """{function name: Row} of every buffer entry point of dpfhe_seeded.h"""
    sk = lambda: dev("sk", KEY, ONE, ALL)
    hsk = lambda: hst("sk", KEY, ONE, ALL)
    enc_ref = lambda R, s, x: {"c0": sr.encrypt_seeded(prefix_oracle(R, s), T, x["sk"][0], SEED, ITEM0, x["pt"])[:, 0]}
    exp_ref = lambda R, s, x: {"ct": sr.expand_ciphertexts(prefix_oracle(R, s), A_SEED, ITEM0, x["c0"])}
    kexp_ref = lambda R, s, x: {"keys": sr.expand_switch_keys(R.o, s.K, A_SEED, items(s), x["b"])}
    rows = [
        Row("dpfhe_encrypt_seeded", [sk(), dev("pt", OPERAND, BATCH), dev("c0", OUTPUT, BATCH)],
            lambda c, s, p: c.encrypt_seeded(T, p["sk"], SEED, ITEM0, p["pt"], p["c0"], s.batch), enc_ref),
        Row("dpfhe_encrypt_seeded_level", [sk(), dev("pt", OPERAND, BATCH), dev("c0", OUTPUT, BATCH)],
            lambda c, s, p: c.encrypt_seeded_level(s.lv, T, p["sk"], SEED, ITEM0, p["pt"], p["c0"], s.batch), enc_ref),
        Row("dpfhe_encrypt_seeded_host", [hsk(), hst("pt", OPERAND, BATCH), hst("c0", OUTPUT, BATCH)],
            lambda c, s, p: c.encrypt_seeded_host(T, p["sk"], SEED, ITEM0, p["pt"], p["c0"]), enc_ref),
        Row("dpfhe_encrypt_seeded_level_host", [hsk(), hst("pt", OPERAND, BATCH), hst("c0", OUTPUT, BATCH)],
            lambda c, s, p: c.encrypt_seeded_level_host(s.lv, T, p["sk"], SEED, ITEM0, p["pt"], p["c0"]), enc_ref),
        Row("dpfhe_expand_ciphertexts", [dev("c0", OPERAND, BATCH), dev("ct", OUTPUT, CT)],
            lambda c, s, p: c.expand_ciphertexts(A_SEED, ITEM0, p["c0"], p["ct"], s.batch), exp_ref),
        Row("dpfhe_expand_ciphertexts_level", [dev("c0", OPERAND, BATCH), dev("ct", OUTPUT, CT)],
            lambda c, s, p: c.expand_ciphertexts_level(s.lv, A_SEED, ITEM0, p["c0"], p["ct"], s.batch), exp_ref),
        Row("dpfhe_upload_seeded_ciphertexts", [hst("c0", OPERAND, BATCH), hst("ct", OUTPUT, CT)],
            lambda c, s, p: _via_device(c, p, "ct", (s.batch, 2, s.lv, s.N), lambda o: c.upload_seeded_ciphertexts(A_SEED, ITEM0, p["c0"], o)),
            exp_ref, note="device output through a tensor of its own"),
        Row("dpfhe_upload_seeded_ciphertexts_level", [hst("c0", OPERAND, BATCH), hst("ct", OUTPUT, CT)],
            lambda c, s, p: _via_device(c, p, "ct", (s.batch, 2, s.lv, s.N),
                                        lambda o: c.upload_seeded_ciphertexts_level(s.lv, A_SEED, ITEM0, p["c0"], o)),
            exp_ref, note="device output through a tensor of its own"),
        Row("dpfhe_relin_keygen_seeded", [sk(), dev("b", OUTPUT, lambda s: s.dnum, ALL)],
            lambda c, s, p: c.generate_relin_key_seeded(s.K, T, p["sk"], SEED, p["b"]),
            lambda R, s, x: {"b": _key_ref(R, s, x["sk"])[0, :, 0]}),
        Row("dpfhe_relin_keygen_seeded_host", [hsk(), hst("b", OUTPUT, lambda s: s.dnum, ALL)],
            lambda c, s, p: c.generate_relin_key_seeded_host(s.K, T, p["sk"], SEED, p["b"]),
            lambda R, s, x: {"b": _key_ref(R, s, x["sk"])[0, :, 0]}),
        Row("dpfhe_galois_keygen_seeded", [sk(), dev("b", OUTPUT, lambda s: (s.n_rot - 1) * s.dnum, ALL)],
            lambda c, s, p: c.generate_galois_keys_seeded(s.K, T, p["sk"], items(s)[1:], SEED, p["b"]),
            lambda R, s, x: {"b": _key_ref(R, s, x["sk"])[1:, :, 0]}),
        Row("dpfhe_galois_keygen_seeded_host", [hsk(), hst("b", OUTPUT, lambda s: (s.n_rot - 1) * s.dnum, ALL)],
            lambda c, s, p: c.generate_galois_keys_seeded_host(s.K, T, p["sk"], items(s)[1:], SEED, p["b"]),
            lambda R, s, x: {"b": _key_ref(R, s, x["sk"])[1:, :, 0]}),
        Row("dpfhe_expand_switch_keys", [dev("b", OPERAND, DIG, ALL), dev("keys", OUTPUT, KEYS, ALL)],
            lambda c, s, p: c.expand_switch_keys(s.K, A_SEED, items(s), p["b"], p["keys"]), kexp_ref),
        Row("dpfhe_upload_seeded_switch_keys", [hst("b", OPERAND, DIG, ALL), hst("keys", OUTPUT, KEYS, ALL)],
            lambda c, s, p: _via_device(c, p, "keys", (s.n_rot, s.dnum, 2, s.L, s.N),
                                        lambda o: c.upload_seeded_switch_keys(s.K, A_SEED, items(s), p["b"], o)),
            kexp_ref, note="device output through a tensor of its own"),
        Row("dpfhe_expand_switch_keys_host", [hst("b", OPERAND, DIG, ALL), hst("keys", OUTPUT, KEYS, ALL)],
            lambda c, s, p: c.expand_switch_keys_host(s.K, A_SEED, items(s), p["b"], p["keys"]), kexp_ref),
    ]
    return {r.fn: r for r in rows}


def runs_at(fn, s):
    """the top-level ciphertext rows take ciphertexts of every limb (K = 0, no level); the level rows run at s.lv; the key rows at any
    shape with a Galois key (n_rot >= 2: the first item is the relinearisation key)"""
    if "keygen" in fn or "switch_keys" in fn:
        return s.n_rot >= 2
    return fn.endswith(("_level", "_level_host")) or (s.K == 0 and s.level is None)

