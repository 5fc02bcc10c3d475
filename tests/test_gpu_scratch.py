"""The context's device-memory accounting (dpfhe_context_device_bytes) through one sequence of calls on one context: every step's
increase against the scratch and tables its shapes need, a repeated call of the same size that leaves the count unchanged,
dpfhe_context_trim and a call after it that brings its buffer back, and the launch count of every step."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

LOGN, L, K = 12, 4, 2                 # four limbs, the last two special primes for the grouped calls (Lq = 2, one digit)
N = 1 << LOGN
P = L * N                             # words of a polynomial over every limb
LQ = L - K
PIPE_DEPTH = 3                        # host-buffer pipeline slots: each has an input and an output staging buffer
CKKS_POW2_E = 1024                    # exponents of the CKKS table 2^e mod q


def empty(*shape):
    return torch.empty(shape, dtype=torch.int64, device="cuda")


def pick_chunk(item_bytes, n_items, num_sms):
    """items per chunk of the host-buffer pipeline: ~64 MiB per staged operand, at least one wave of the SMs"""
    c = max(1, (64 << 20) // item_bytes)
    if c < num_sms <= n_items:
        c = num_sms
    return min(c, n_items)


def test_device_bytes_through_a_call_sequence(monkeypatch):
    import deeppowers_b200 as dp
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = dp.Context(LOGN, L)
    seed = [100]

    def uniform(n_polys):   # valid residues on every limb, [n_polys][L][N]
        x = empty(n_polys, L, N)
        ctx.fill_uniform(seed[0], x, n_polys)
        seed[0] += 1
        return x

    # every input first, so that the steps below launch only what they measure
    ct = uniform(2 * 5).view(5, 2, L, N)
    ctq = uniform(2 * 5)[:, :LQ].contiguous().view(5, 2, LQ, N)
    gks = [uniform(2 * L).view(L, 2, L, N) for _ in range(2)]
    gks_grouped = [uniform(2).view(1, 2, L, N) for _ in range(2)]
    slots = torch.zeros((3, N // 2), dtype=torch.complex128, device="cuda")
    bgv_slots = torch.zeros((3, 2, N // 2), dtype=torch.int64, device="cuda")
    pt = empty(3, L, N)
    low = empty(8, L, N)
    torch.cuda.synchronize()

    state = {"bytes": ctx.device_bytes(), "launches": ctx.launch_count()}
    assert state["bytes"] > 0                             # 1. creation: transform tables, key-switch slots and flags

    def step(call, grows, launches):
        """runs one call; grows: its increase of device_bytes (None: not known from the shapes); returns the increase"""
        call()
        ctx.synchronize()
        b, n = ctx.device_bytes(), ctx.launch_count()
        increase = b - state["bytes"]
        assert grows is None or increase == grows
        assert n - state["launches"] == launches
        state["bytes"], state["launches"] = b, n
        return increase

    # 2. the modulus switches share one scratch of tau rows, [n_polys][K][N]: it grows to the larger need and is reused
    step(lambda: ctx.mod_switch_down(ct, low, 3), 3 * N * 8, 2)
    step(lambda: ctx.mod_switch_down(ct, low, 3), 0, 2)
    step(lambda: ctx.mod_down_special(K, ct, low, 4), 4 * K * N * 8 - 3 * N * 8, 2)
    step(lambda: ctx.mod_down_special(K, ct, low, 4), 0, 2)
    step(lambda: ctx.mod_switch_down(ct, low, 2), 0, 2)

    # 3. hoisted rotations under a 1 MiB cap: shared transforms [chunk][L][L][N] and zero flags [chunk] for chunks of two of the
    # five ciphertexts, and, once, the per-rotation constants M [L][N], kprime [2][L][N] and delta [L][L]
    monkeypatch.setenv("DPFHE_HOIST_CAP_MB", "1")
    chunk = (1 << 20) // (L * L * N * 8)
    assert chunk == 2
    galois = [ctx.galois_elt(1), ctx.galois_elt(-1)]
    rot = empty(2, 5, 2, L, N)
    per_chunk = 1 + 2 * (4 + 1 + 1)                       # hoist; per rotation: prepare (4), apply, recompute
    consts = 3 * P * 8 + L * L * 8
    step(lambda: ctx.rotate_hoisted(ct, galois, gks, rot, 5), chunk * (L * L * N * 8 + 4) + consts, 3 * per_chunk)
    step(lambda: ctx.rotate_hoisted(ct, galois, gks, rot, 5), 0, 3 * per_chunk)
    # the special-prime rows of the grouped key switches are allocated by the first grouped call and kept
    d = ctq[:, 1].contiguous()
    outq = empty(5, 2, LQ, N)
    assert step(lambda: ctx.keyswitch_grouped(K, d, gks_grouped[0], outq, 1), None, 2) > 0
    step(lambda: ctx.keyswitch_grouped(K, d, gks_grouped[0], outq, 1), 0, 2)
    # grouped hoisted rotations: lifted digits [1][L][N], accumulators [2][L][N] and tau' rows [2][K][N] per ciphertext of a chunk
    per_ct = (L * N + 2 * L * N + 2 * K * N) * 8
    chunk_g = (1 << 20) // per_ct
    assert chunk_g == 2
    rotq = empty(2, 5, 2, LQ, N)
    step(lambda: ctx.rotate_hoisted_grouped(K, ctq, galois, gks_grouped, rotq, 5), chunk_g * per_ct, 3 * (1 + 2 * 4))
    step(lambda: ctx.rotate_hoisted_grouped(K, ctq, galois, gks_grouped, rotq, 5), 0, 3 * (1 + 2 * 4))
    monkeypatch.delenv("DPFHE_HOIST_CAP_MB")

    # 4. CKKS encoding: twiddles [N] (complex), slot permutation [N/2] (u32) and 2^e mod q [L][1024], and coefficient rows [n_vec][N]
    ckks_tables = N * 16 + (N // 2) * 4 + L * CKKS_POW2_E * 8
    step(lambda: ctx.ckks_encode(slots, pt, 3, 2.0**40), ckks_tables + 3 * N * 8, 2)
    step(lambda: ctx.ckks_encode(slots, pt, 3, 2.0**40), 0, 2)

    # 5. BGV encoding: the tables of one plaintext modulus, twiddles and slot positions [5][N] (u32), replaced when t changes; the
    # encoders' scratch ([n_vec][N] u32) already holds the rows
    step(lambda: ctx.bgv_encode(bgv_slots, pt, 3, 65537), 5 * N * 4, 2)
    step(lambda: ctx.bgv_encode(bgv_slots, pt, 3, 167772161), 0, 2)
    step(lambda: ctx.bgv_encode(bgv_slots, pt, 3, 65537), 0, 2)

    # 6. a host-buffer call: PIPE_DEPTH input and output staging buffers of one chunk, and the shared plaintext
    h_ct = ct[:3].cpu().numpy().view(np.uint64)
    h_pt = pt[0].cpu().numpy().view(np.uint64)
    h_out = np.empty_like(h_ct)
    c = pick_chunk(2 * P * 8, 3, num_sms)
    staging = PIPE_DEPTH * 2 * (c * 2 * P * 8) + P * 8
    step(lambda: ctx.ct_mul_plain_host(h_ct, h_pt, h_out), staging, 1)
    step(lambda: ctx.ct_mul_plain_host(h_ct, h_pt, h_out), 0, 1)

    # 7. trim releases every scratch buffer and the encoding tables, and keeps the hoisting constants and the special-prime rows
    kept = ctx.device_bytes()
    ctx._chk(ctx._l.dpfhe_context_trim(ctx._h))
    released = 4 * N * K * 8 + chunk * (L * L * N * 8 + 4) + chunk_g * per_ct + ckks_tables + 3 * N * 8 + 5 * N * 4 + staging
    assert kept - ctx.device_bytes() == released
    assert ctx.launch_count() == state["launches"]
    state["bytes"] = ctx.device_bytes()

    # 8. after the trim the scratch comes back on demand
    step(lambda: ctx.mod_switch_down(ct, low, 3), 3 * N * 8, 2)
    step(lambda: ctx.ct_mul_plain_host(h_ct, h_pt, h_out), staging, 1)
    ctx.close()
