"""The device build of the scalar arithmetic and of the register-level transform pieces on the H100, bit for bit against the host
build that tests/test_devarith_cpu.py pins to exact integers and to the emulator.

On sm_90a much of modarith.cuh is different code from the host's: csub's borrow select, the PTX carry chains of mad_lo64,
shoup_tail (one per arithmetic variant), mul128 and sub128, Barrett's funnel shifts (by 0 for the smallest modulus), __umul64hi
and __umulhi.  Inside whole kernels these paths only ever see canonical or uniform data, so a slip that needs one particular
carry or borrow would show up as an occasional wrong ciphertext.  Here every op runs on every modulus of every configuration
(tests/arith_cases.py) over its structured cases and 2^20 uniform ones (2^16 for the 16-point pieces, 32 butterflies each), and
every output word, lazy values included, must equal the host's.  The structured cases' device outputs also go through the
exact-integer checks directly, so that a failure names the input and the expected value."""
import numpy as np
import pytest

import arith_cases as ac
from test_devarith_cpu import CONFIGS, IDS, _fail_msg, harness, host_cases

pytestmark = pytest.mark.gpu


def _first_diff(cid, op, idx, x, want, got):
    k = int(np.flatnonzero(np.any(want != got, axis=1))[0])
    n = int(np.count_nonzero(np.any(want != got, axis=1)))
    return "%s %s [%d]: device differs from host on %d cases; first input %s: host %s, device %s" % (
        cid, op, idx, n, [hex(int(v)) for v in x[k]], [hex(int(v)) for v in want[k]], [hex(int(v)) for v in got[k]])


@pytest.mark.parametrize("cid", IDS)
def test_device_equals_host(cid):
    _, variant, mods, ts = CONFIGS[IDS.index(cid)]
    da = harness.DevArith(variant, mods, ts)
    jobs = [(l, q, da.limb_params(l), op) for l, q in enumerate(mods) for op in ac.ops_for(da.limb_params(l), False)]
    jobs += [(k, t, None, op) for k, t in enumerate(ts) for op in ac.U32_OPS]
    for idx, q, lp, op in jobs:
        s, r, hs, hr = host_cases(da, cid, idx, q, lp, op, seed=ac.seed_of(cid, q, op))
        x, want = np.concatenate([s, r]), np.concatenate([hs, hr])
        got = da.device(op, idx, x)
        bad = ac.check(op, q, lp, s, got[:len(s)])
        assert not bad, _fail_msg(cid, op, idx, bad)
        assert np.array_equal(got, want), _first_diff(cid, op, idx, x, want, got)
