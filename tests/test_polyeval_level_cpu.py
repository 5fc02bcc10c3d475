"""BGV polynomial evaluation from a start level l below the top (DESIGN.md section 2.22) without a GPU: the restatement of the schedule
(tests/polyeval_ref.py) run on the chain over {q_0 .. q_{l-1}, p_0 .. p_{K-1}} with restrict_key(key, Lq, K, l) of the top-level key,
decrypting under the oracle to p(slots) mod t from every start level, at degree 1 and at the deepest degree the level allows.  This is
what the device's level evaluators are compared against."""
import numpy as np
import pytest

import polyeval_ref as pr
from test_polyeval_cpu import T, _decrypt_slots, _encrypt_slots


@pytest.mark.parametrize("K,Lq", [(1, 3), (2, 5), (3, 5)])
def test_restatement_from_every_start_level(oracle_mod, K, Lq):
    logn, B = 10, 2
    top = oracle_mod.Oracle(logn, Lq + K)
    s = top.keygen_secret(11)
    key = top.keygen_relin_grouped(K, 12, T, s)
    rng = np.random.default_rng(10 * K + Lq)
    for l in range(K, Lq + 1):
        ch = pr.Chain(oracle_mod, logn, list(top.moduli)[:l] + list(top.moduli)[Lq:], K)
        kl = pr.restrict_key(key, Lq, K, l)
        D = min(l - 1, l - K + 1)
        for d in sorted({1, 1 << D}):
            coeffs = [int(c) for c in rng.integers(-1000, 1000, d + 1)]
            z = rng.integers(0, T, (B, 2, top.N // 2), dtype=np.int64)
            ct = _encrypt_slots(ch.ct(l), np.ascontiguousarray(s[:l]), z, T, 20)
            out = pr.polyeval(ch, T, coeffs, ct, kl)
            Lf = l - pr.ceil_log2(d)
            assert out.shape == (B, 2, Lf, top.N), (l, d)
            assert np.array_equal(_decrypt_slots(ch.ct(Lf), np.ascontiguousarray(s[:Lf]), out, T), pr.poly_mod_t(coeffs, z, T)), (l, d)
