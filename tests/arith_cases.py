"""Cases and exact-integer checks for the scalar arithmetic and the register-level transform pieces (tests/devarith/devarith.cu),
shared by tests/test_devarith_cpu.py (host build) and tests/test_gpu_devarith.py (device build == host build, bit for bit).

Every op runs only on moduli its arithmetic build accepts and only on inputs inside its documented domain (modarith.cuh's table,
ntt_core.cuh's butterfly comments).  `check` recomputes each result with Python integers and returns the cases whose output is not
congruent, leaves its documented range, or (umulhi64, mul128, sub128, the canonical forms) is not exact.  `corners` names the
lazy-range corners an output reaches, so that the tests can assert that the cases really get there.
"""
import zlib

import numpy as np

import bases
from bgv_ref import T_VALUES

M64 = 1 << 64
M32 = 1 << 32
SB = 4                      # types.hpp: the Shoup and Barrett quotient estimates may be up to two short
LOG_N = 12                  # the harness derives limb constants for N = 4096
TWO_N = 2 << LOG_N
HALVES = (0, 0x80000000, 0xFFFFFFFF)
N_RANDOM = 1 << 20          # uniform cases per op and modulus (scalar ops)
N_RANDOM_16 = 1 << 16       # uniform cases of the 16-point pieces: 32 butterflies each


# ---- moduli ---------------------------------------------------------------------------------------------------------------
def is_prime(n):
    """Miller-Rabin with the first twelve prime bases: exact below 2^64"""
    if n < 2:
        return False
    small = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    for p in small:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in small:
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


class _Primality:
    dpo_is_prime = staticmethod(is_prime)


def default_basis(L=2):
    """the L largest primes below 2^60 of the form k * 2^32 + 1 (host_params.cpp, DESIGN.md §2.1)"""
    out, c = [], (1 << 60) + 1
    while len(out) < L:
        c -= 1 << 32
        if is_prime(c):
            out.append(c)
    return out


def near60_threshold_primes():
    """the NTT primes on either side of 2^64 / 17: canon_near60 applies above (floor(2^64/q) == 16), not below"""
    thr = M64 // 17
    above = thr - thr % TWO_N + TWO_N + 1
    while not is_prime(above):
        above += TWO_N
    below = thr - thr % TWO_N + 1
    while not is_prime(below):
        below -= TWO_N
    assert M64 // above == 16 and M64 // below == 17
    return [above, below]


def largest_plain_modulus():
    """the largest valid BGV plaintext modulus at N = 4096: prime, t < 2^31, t = 1 mod 2N"""
    t = (1 << 31) - (1 << 31) % TWO_N + 1
    while t >= 1 << 31 or not is_prime(t):
        t -= TWO_N
    return t


def configs():
    """[(id, arithmetic build, limb moduli, plaintext moduli)]: every build only on moduli it accepts.  The 32-bit ops (plaintext
    moduli) do not depend on the build; they run in both, once each."""
    ts = list(T_VALUES) + [largest_plain_modulus()]
    fast_mixed = [bases._fast_prime(_Primality, b) for b in (37, 40, 45, 48, 50, 55)]
    return [
        ("gen-default", "gen", default_basis(), ts),          # what DPFHE_FORCE_GENERIC runs on the default basis
        ("fast-default", "fast", default_basis(), ts),
        ("gen-smallest", "gen", [bases.SMALLEST_GENERIC], []),  # bar_shift = 32: the device's funnel shifts shift by 0
        ("gen-largest", "gen", [bases.LARGEST_GENERIC], []),
        ("gen-near60", "gen", near60_threshold_primes(), []),
        ("fast-mixed", "fast", fast_mixed, []),
    ]


U32_OPS = ("mulhi32", "shoup32", "add32", "sub32", "reduce64_32")


def seed_of(*parts):
    """a seed that names the cases (configuration, modulus, op), the same in every process"""
    return zlib.crc32(repr(parts).encode())


# ---- the forward transform's bound schedule (ntt_core.cuh) ---------------------------------------------------------------
def fwd_bound_after(bin_, stages):
    b = bin_
    for _ in range(stages):
        b = (8 if b + SB > 16 else b) + SB
    return b


def fwd16_entry_bounds():
    """B0, B1, B2 of fwd_passes_blk for every BIN the bodies pass (1 canonical, 3 word-reduced, 4) and K = LOGN - 12 in {0, 1, 2}"""
    return sorted({fwd_bound_after(b, k + s) for b in (1, 3, 4) for k in (0, 1, 2) for s in (0, 4, 8)})


FWD16 = ["fwd16_%d" % b for b in fwd16_entry_bounds()]
TRANSFORM16 = FWD16 + ["inv16"]


def ops_for(lp, u32):
    """the ops one limb (or, with u32, one plaintext modulus) runs"""
    if u32:
        return list(U32_OPS)
    ops = ["umulhi64", "mulhi_approx", "csub", "mad_lo64", "sub_mul_q", "shoup_exact", "shoup_lazy", "mul128", "sub128",
           "barrett_lazy", "barrett_lazy_long", "mulmod_lazy", "mulmod", "word_reduce", "canon", "canon4", "canon_store", "pti_fold",
           "bgv_lift", "ct_bfly", "gs_bfly", "inv_final_product"] + TRANSFORM16
    if lp["mu32"] == 16:
        ops.append("canon_near60")   # only defined where floor(2^64 / q) == 16
    return ops


# ---- helpers ------------------------------------------------------------------------------------------------------------
def shoup(w, q, bits=64):
    return (w << bits) // q


def mulhi_err(x, y):
    """hi64(x*y) minus the three-product estimate of mulhi_approx (DESIGN.md §4.1): the carry of the dropped low words, 0..2"""
    xl, xh, yl, yh = x & (M32 - 1), x >> 32, y & (M32 - 1), y >> 32
    return ((xh * yl & (M32 - 1)) + (xl * yh & (M32 - 1)) + (xl * yl >> 32)) >> 32


def singles(q):
    """0, 1, q-1, q, q+1, k q - 1, k q, k q + 1 for k <= 16, 2^63, 2^64 - 2, 2^64 - 1, words whose halves are 0, 2^31, 2^32 - 1"""
    s = {0, 1, q - 1, q, q + 1, 1 << 63, M64 - 2, M64 - 1}
    for k in range(2, 17):
        s |= {k * q - 1, k * q, k * q + 1}
    s |= {h << 32 | l for h in HALVES for l in HALVES}
    return sorted(v for v in s if 0 <= v < M64)


def below(vals, top):
    return sorted({v for v in vals if v < top} | {top - 1})


def twiddles(q):
    return sorted({0, 1, q - 1, q // 2, (q - 1) & ~(M32 - 1), M32 - 1})


def short_by_two(ws, rng, want=4):
    """multiplicands x for which the estimate of hi64(x * ws) is exactly two short (none when ws's words make it impossible)"""
    n, m = 1 << 13, np.uint64(M32 - 1)
    # half uniform low words, half low words just below 2^32 by offsets of every size
    shift = np.maximum(rng.integers(32, 61, n), rng.integers(0, 2, n) * 32).astype(np.uint64)
    shift[: n // 2] = 32
    lo = m - (_u64(rng, n) >> shift)
    x = _u64(rng, n, M32) << np.uint64(32) | lo
    xl, xh, yl, yh = lo, x >> np.uint64(32), np.uint64(ws & (M32 - 1)), np.uint64(ws >> 32)
    err = ((xh * yl & m) + (xl * yh & m) + (xl * yl >> np.uint64(32))) >> np.uint64(32)   # mulhi_err, vectorised
    out = [int(v) for v in x[err == 2][:want]]
    assert all(mulhi_err(v, ws) == 2 for v in out)
    return out


def _np(rows):
    return np.array(rows, dtype=object).astype(np.uint64) if rows else np.zeros((0, 1), dtype=np.uint64)


def _u64(rng, n, top=M64):
    if top == M64:
        return rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True)
    return rng.integers(0, top, n, dtype=np.uint64)


def _mul_wide(a, b):
    """exact 64 x 64 -> 128-bit products of uint64 arrays, (hi, lo), from 32-bit halves"""
    m = np.uint64(M32 - 1)
    s = np.uint64(32)
    al, ah, bl, bh = a & m, a >> s, b & m, b >> s
    ll, lh, hl, hh = al * bl, al * bh, ah * bl, ah * bh
    mid = (ll >> s) + (lh & m) + (hl & m)
    lo = (ll & m) | (mid << s)
    hi = hh + (lh >> s) + (hl >> s) + (mid >> s)
    return hi, lo


def _tw_pool(q, rng, n=1 << 12):
    w = [int(v) for v in _u64(rng, n, q)]
    return np.array(w, dtype=np.uint64), np.array([shoup(v, q) for v in w], dtype=np.uint64)


# ---- cases ----------------------------------------------------------------------------------------------------------------
def structured(op, q, lp, rng):
    """[n][nin] rows of structured inputs for op on modulus q (a plaintext modulus t for the 32-bit ops)"""
    S = singles(q)
    rows = []
    if op in ("umulhi64", "mulhi_approx", "mul128", "mad_lo64", "sub_mul_q"):
        rows = [(a, b) for a in S for b in S]
        for w in twiddles(q):                      # operand pairs on which the estimate is exactly two short
            ws = shoup(w, q)
            rows += [(x, ws) for x in short_by_two(ws, rng)]
        if op == "mad_lo64":
            rows = [(a, b, c) for (a, b), c in zip(rows, S * (len(rows) // len(S) + 1))]
    elif op == "csub":
        for m in (q, 2 * q, 8 * q, SB * q, 1 << 63):
            xs = set(S) | {m - 1, m, m + 1, 2 * m - 1, 2 * m, M64 - 1}
            ml, mh = m & (M32 - 1), m >> 32
            for d in (0, 1, 2, 7):                 # x >= m with x's low word below m's: the borrow of the low-word subtraction
                for e in (1, 2, ml):
                    if 0 < e <= ml and mh + 1 + d < M32:
                        xs.add((mh + 1 + d) << 32 | (ml - e))
            rows += [(x, m) for x in xs if x < M64]
    elif op in ("shoup_exact", "shoup_lazy", "inv_final_product"):
        for w in twiddles(q):
            ws = shoup(w, q)
            rows += [(x, w, ws) for x in S + short_by_two(ws, rng)]
    elif op == "sub128":
        words = [0, 1, M32 - 1, M32, 1 << 63, M64 - 2, M64 - 1, q, q - 1]
        vals = sorted({h << 64 | l for h in words for l in words})
        rows = [(a >> 64, a & (M64 - 1), b >> 64, b & (M64 - 1)) for a in vals for b in vals if a >= b]
    elif op in ("barrett_lazy", "mulmod_lazy"):
        fac = {1: below([0, 1, q // 2, q - 2, q - 1, M32 - 1, M32], q), 2: below([q, q + 1, 2 * q - 2], 2 * q),
               4: below([2 * q, 3 * q - 1, 3 * q, 4 * q - 2], 4 * q)}
        prods = [(a, b) for ba, bb in ((1, 1), (1, 2), (2, 1), (2, 2), (1, 4), (4, 1)) for a in fac[ba] for b in fac[bb]]
        if op == "mulmod_lazy":
            rows = prods
        else:
            zs = {a * b for a, b in prods} | {4 * q * q - 1, (q - 1) ** 2, q * q, q * q - 1, q * q + 1, 3 * q * q, 2 * q * q + q}
            zs |= {k * q * q + d for k in range(1, 4) for d in (-1, 0, 1)} | {M64 - 1, M64, M64 + 1, 0, 1}
            rows = [(z >> 64, z & (M64 - 1)) for z in zs if 0 <= z < 4 * q * q]
    elif op == "barrett_lazy_long":
        b = q.bit_length()
        top = 1 << (2 * b + 4)
        zs = {0, 1, q, top - 1, top - 2, 16 * (q - 1) ** 2, (q - 1) ** 2, 15 * q * q, M64 - 1, M64, top >> 1, (top >> 1) - 1}
        zs |= {k * q * q + d for k in range(1, 17) for d in (-1, 0, 1)}
        rows = [(z >> 64, z & (M64 - 1)) for z in zs if 0 <= z < top]
    elif op == "mulmod":
        c = below([0, 1, 2, q // 2, q - 2, M32 - 1, M32, (q - 1) & ~(M32 - 1)], q)
        rows = [(a, b) for a in c for b in c]
    elif op in ("word_reduce", "canon_near60"):
        rows = [(x,) for x in S]
    elif op in ("canon", "canon4", "canon_store"):
        top = 4 * q if op == "canon4" else (M64 if op == "canon_store" and lp["mu32"] == 16 else 16 * q)
        rows = [(x,) for x in below(S, top)]
    elif op == "pti_fold":
        rows = [pti_terms([(q - 1, q - 1)] * n) for n in (1, 2, 15, 16)]
        rows += [pti_terms([(0, 0)]), pti_terms([(q - 1, 1)]), pti_terms([(M32 - 1, q - 1)] * 16), pti_terms([((1 << 30) - 1, (1 << 30) - 1)] * 16)]
        rows += [pti_terms([(q - 1 - k, q - 1 - 2 * k)] * 16) for k in range(1, 5)]
    elif op == "bgv_lift":
        for t in T_VALUES + (largest_plain_modulus(),):
            rows += [(c, t) for c in {0, 1, t // 2 - 1, t // 2, t // 2 + 1, t - 2, t - 1}]
    elif op == "ct_bfly":
        xs = below([0, 1, q - 1, q, 4 * q - 1, 8 * q - 1, 8 * q, 11 * q], 12 * q)
        for w in twiddles(q):
            ws = shoup(w, q)
            ys = S + short_by_two(ws, rng, 2)
            rows += [(x, y, w, ws) for x in xs for y in ys]
    elif op == "gs_bfly":
        xs = below([0, 1, q - 1, q, 2 * q, 3 * q + 1, 4 * q - 2], SB * q)
        for w in twiddles(q):
            ws = shoup(w, q)
            rows += [(x, y, w, ws) for x in xs for y in xs]
    elif op in TRANSFORM16:
        B = SB if op == "inv16" else int(op.split("_")[1])
        tws = twiddles(q)
        for k, top in enumerate([0, 1, B * q - 1, q - 1, None, None]):
            for m, w in enumerate(tws):
                if top is None:   # every input at the top of the bound or alternating with 0, one twiddle everywhere
                    x = [(B * q - 1) if (i + k) % 2 else 0 for i in range(16)]
                else:
                    x = [top] * 16
                rows.append(x + [w] * 15 + [shoup(w, q)] * 15)
        x = [B * q - 1 - i for i in range(16)]
        ws_all = [int(v) for v in _u64(rng, 15, q)]
        rows.append(x + ws_all + [shoup(w, q) for w in ws_all])
    elif op == "mulhi32":
        v = [0, 1, 2, 0x7FFFFFFF, 0x80000000, M32 - 2, M32 - 1, q - 1, q]
        rows = [(a, b) for a in v for b in v]
    elif op == "shoup32":
        t = q
        for w in sorted({0, 1, 2, t // 2, t - 1, ((1 << 32) % t)}):
            ws = shoup(w, t, 32)
            rows += [(x, w, ws) for x in (0, 1, t - 1, t, t + 1, 2 * t - 1, 2 * t, 0x7FFFFFFF, 0x80000000, M32 - 2, M32 - 1)]
    elif op in ("add32", "sub32"):
        c = [0, 1, q // 2, q // 2 + 1, q - 2, q - 1]
        rows = [(a, b) for a in c for b in c]
    elif op == "reduce64_32":
        t = q
        xs = set(S) | {k * t + d for k in (1, 2, M32 // t, M32 // t + 1) for d in (-1, 0, 1)} | {M32 - 1, M32, M32 + 1, (M64 - 1) // t * t}
        rows = [(x,) for x in xs if 0 <= x < M64]
    else:
        raise KeyError(op)
    return _np(rows)


def pti_terms(pairs):
    """the four split-operand sums of pt_inner_tile for a list of (x, y) canonical factor pairs"""
    m30 = (1 << 30) - 1
    return (sum((x & m30) * (y & m30) for x, y in pairs), sum((x & m30) * (y >> 30) for x, y in pairs),
            sum((x >> 30) * (y & m30) for x, y in pairs), sum((x >> 30) * (y >> 30) for x, y in pairs))


def uniform(op, q, lp, rng, n):
    """[n][nin] uniform inputs inside op's domain"""
    u = lambda top=M64: _u64(rng, n, top)   # noqa: E731
    if op in ("umulhi64", "mulhi_approx", "mul128", "sub_mul_q"):
        return np.stack([u(), u()], 1)
    if op == "mad_lo64":
        return np.stack([u(), u(), u()], 1)
    if op == "csub":
        m = np.array([q, 2 * q, 8 * q, SB * q, 1 << 63], dtype=np.uint64)[rng.integers(0, 5, n)]
        x = u()
        half = rng.integers(0, 2, n).astype(bool) & (m != np.uint64(1 << 63))   # below 2m, where both outcomes are common
        x[half] = x[half] % (m[half] * np.uint64(2))
        return np.stack([x, m], 1)
    if op in ("shoup_exact", "shoup_lazy", "inv_final_product"):
        w, ws = _tw_pool(q, rng)
        k = rng.integers(0, len(w), n)
        return np.stack([u(), w[k], ws[k]], 1)
    if op == "sub128":
        a, b = np.stack([u(), u()], 1), np.stack([u(), u()], 1)
        swap = (a[:, 0] < b[:, 0]) | ((a[:, 0] == b[:, 0]) & (a[:, 1] < b[:, 1]))
        a[swap], b[swap] = b[swap].copy(), a[swap].copy()
        return np.concatenate([a, b], 1)
    if op in ("barrett_lazy", "mulmod_lazy"):
        # factor bounds (1, 1), (1, 4), (4, 1), (2, 2): canonical products, and the lazy ones the documented domain allows
        kind = rng.integers(0, 4, n)
        ta = np.array([q, q, 4 * q, 2 * q], dtype=np.uint64)[kind]
        tb = np.array([q, 4 * q, q, 2 * q], dtype=np.uint64)[kind]
        a, b = u() % ta, u() % tb
        if op == "mulmod_lazy":
            return np.stack([a, b], 1)
        hi, lo = _mul_wide(a, b)
        return np.stack([hi, lo], 1)
    if op == "barrett_lazy_long":
        top_hi = 1 << (2 * q.bit_length() + 4 - 64)
        return np.stack([u(top_hi), u()], 1)
    if op == "mulmod":
        return np.stack([u(q), u(q)], 1)
    if op in ("word_reduce", "canon_near60"):
        return u()[:, None]
    if op in ("canon", "canon4", "canon_store"):
        top = 4 * q if op == "canon4" else (M64 if op == "canon_store" and lp["mu32"] == 16 else 16 * q)
        return u(top)[:, None]
    if op == "pti_fold":
        m30 = np.uint64((1 << 30) - 1)
        s30 = np.uint64(30)
        # sums of up to 16 products of canonical factors: k1 copies of one product and k2 of another, k1 + k2 <= 16
        k1 = rng.integers(1, 17, n)
        k = np.stack([k1, rng.integers(0, 17 - k1)]).astype(np.uint64)
        x, y = _u64(rng, (2, n), q), _u64(rng, (2, n), q)
        xl, xh, yl, yh = x & m30, x >> s30, y & m30, y >> s30
        return np.stack([(k * xl * yl).sum(0), (k * xl * yh).sum(0), (k * xh * yl).sum(0), (k * xh * yh).sum(0)], 1)
    if op == "bgv_lift":
        ts = np.array(list(T_VALUES) + [largest_plain_modulus()], dtype=np.uint64)[rng.integers(0, len(T_VALUES) + 1, n)]
        return np.stack([u() % ts, ts], 1)
    if op in ("ct_bfly", "gs_bfly"):
        w, ws = _tw_pool(q, rng)
        k = rng.integers(0, len(w), n)
        x = u(12 * q if op == "ct_bfly" else SB * q)
        y = u() if op == "ct_bfly" else u(SB * q)
        return np.stack([x, y, w[k], ws[k]], 1)
    if op in TRANSFORM16:
        B = SB if op == "inv16" else int(op.split("_")[1])
        w, ws = _tw_pool(q, rng)
        k = rng.integers(0, len(w), (n, 15))
        return np.concatenate([_u64(rng, (n, 16), B * q), w[k], ws[k]], 1)
    t = q
    if op == "mulhi32":
        return np.stack([u(M32), u(M32)], 1)
    if op == "shoup32":
        w = u(t)
        ws = (w << np.uint64(32)) // np.uint64(t)
        return np.stack([u(M32), w, ws], 1)
    if op in ("add32", "sub32"):
        return np.stack([u(t), u(t)], 1)
    if op == "reduce64_32":
        return u()[:, None]
    raise KeyError(op)


# ---- exact checks ---------------------------------------------------------------------------------------------------------
def fwd16_exact(x, tw, q):
    x = list(x)
    for u in range(4):
        half = 8 >> u
        for j in range(1 << u):
            w = tw[(1 << u) - 1 + j]
            for i in range(half):
                a, b = x[j * 2 * half + i], x[j * 2 * half + half + i]
                x[j * 2 * half + i], x[j * 2 * half + half + i] = (a + w * b) % q, (a - w * b) % q
    return x


def inv16_exact(x, tw, q):
    x = list(x)
    for u in range(3, -1, -1):
        half = 8 >> u
        for j in range(1 << u):
            w = tw[(1 << u) - 1 + j]
            for i in range(half):
                a, b = x[j * 2 * half + i], x[j * 2 * half + half + i]
                x[j * 2 * half + i], x[j * 2 * half + half + i] = (a + b) % q, (a - b) * w % q
    return x


def check_one(op, q, lp, i, o):
    """None if output o (tuple of ints) of op on input i is right, else what is wrong"""
    def lazy(r, v, bound, what="range"):
        if r % q != v % q:
            return "not congruent: %d != %d mod q" % (r, v % q)
        if not r < bound * q:
            return "%s: %d >= %s q" % (what, r, bound)
        return None

    if op == "umulhi64":
        return None if o[0] == i[0] * i[1] >> 64 else "want %d" % (i[0] * i[1] >> 64)
    if op == "mulhi_approx":
        d = (i[0] * i[1] >> 64) - o[0]
        return None if 0 <= d <= 2 else "hi64 - estimate = %d" % d
    if op == "csub":
        want = i[0] - i[1] if i[0] >= i[1] else i[0]
        return None if o[0] == want else "want %d" % want
    if op == "mad_lo64":
        want = (i[2] + i[0] * i[1]) % M64
        return None if o[0] == want else "want %d" % want
    if op == "sub_mul_q":
        want = (i[0] - i[1] * q) % M64
        return None if o[0] == want else "want %d" % want
    if op == "shoup_exact":
        return lazy(o[0], i[0] * i[1], 2)
    if op == "shoup_lazy":
        return lazy(o[0], i[0] * i[1], SB)
    if op == "inv_final_product":
        want = i[0] * i[1] % q
        return None if o[0] == want else "want %d" % want
    if op == "mul128":
        return None if (o[0] << 64 | o[1]) == i[0] * i[1] else "want %d" % (i[0] * i[1])
    if op == "sub128":
        want = (i[0] << 64 | i[1]) - (i[2] << 64 | i[3])
        return None if (o[0] << 64 | o[1]) == want else "want %d" % want
    if op == "barrett_lazy":
        z = i[0] << 64 | i[1]
        return lazy(o[0], z, SB if z <= (q - 1) ** 2 else SB + 1)
    if op == "mulmod_lazy":
        return lazy(o[0], i[0] * i[1], SB if max(i) < q else SB + 1)
    if op == "barrett_lazy_long":
        return lazy(o[0], i[0] << 64 | i[1], 15)
    if op == "pti_fold":
        return lazy(o[0], i[0] + ((i[1] + i[2]) << 30) + (i[3] << 60), 3)
    if op == "word_reduce":
        return lazy(o[0], i[0], 3)
    if op in ("mulmod", "canon", "canon4", "canon_near60", "canon_store"):
        want = (i[0] * i[1] if op == "mulmod" else i[0]) % q
        return None if o[0] == want else "want %d" % want
    if op == "bgv_lift":
        c, t = i
        want = c if c <= t // 2 else q - (t - c)
        return None if o[0] == want else "want %d" % want
    if op == "ct_bfly":
        x, y, w, _ = i
        t = o[0] - x
        if not 0 <= t < SB * q or o[0] + o[1] != 2 * x + SB * q:
            return "x' - x = %d outside [0, SB q) or x' + y' != 2x + SB q" % t
        return lazy(o[0], x + w * y, 16) or lazy(o[1], x - w * y, 16)
    if op == "gs_bfly":
        x, y, w, _ = i
        return lazy(o[0], x + y, SB) or lazy(o[1], (x - y) * w, SB)
    if op in TRANSFORM16:
        tw = i[16:31]
        exact = (fwd16_exact if op != "inv16" else inv16_exact)(i[:16], tw, q)
        bound = SB if op == "inv16" else fwd_bound_after(int(op.split("_")[1]), 4)
        for k in range(16):
            e = lazy(o[k], exact[k], bound)
            if e:
                return "element %d: %s" % (k, e)
        return None
    t = q
    if op == "mulhi32":
        return None if o[0] == i[0] * i[1] >> 32 else "want %d" % (i[0] * i[1] >> 32)
    want = {"shoup32": lambda: i[0] * i[1] % t, "add32": lambda: (i[0] + i[1]) % t, "sub32": lambda: (i[0] - i[1]) % t,
            "reduce64_32": lambda: i[0] % t}[op]()
    return None if o[0] == want else "want %d" % want


def check(op, q, lp, inp, out, limit=5):
    """[(input, output, what is wrong)] for the first `limit` wrong cases"""
    bad = []
    for i, o in zip(inp.tolist(), out.tolist()):
        e = check_one(op, q, lp, i, o)
        if e:
            bad.append((i, o, e))
            if len(bad) >= limit:
                break
    return bad


def corners(op, q, inp, out):
    """the lazy-range corners the outputs reach (python ints, vectorised where it is cheap)"""
    got = set()
    if op == "mulhi_approx":
        d = {(a * b >> 64) - r for (a, b), (r,) in zip(inp.tolist(), out.tolist())}
        got |= {"short_by_%d" % k for k in d}
    elif op == "csub":
        x, m = inp[:, 0], inp[:, 1]
        lo = np.uint64(M32 - 1)
        if np.any((x >= m) & ((x & lo) < (m & lo))):
            got.add("low_word_borrow")
        if np.any(x < m):
            got.add("kept")
    elif op == "reduce64_32":
        if np.any(inp[:, 0] == np.uint64(M64 - 1)):
            got.add("x=2^64-1")
    else:
        r = out if op in TRANSFORM16 or op in ("ct_bfly", "gs_bfly") else out[:, :1]
        if op == "ct_bfly":   # the Shoup product inside: x' - x
            r = (out[:, 0] - inp[:, 0])[:, None]
        band = r // np.uint64(q)
        got |= {"band_%d" % int(b) for b in np.unique(band) if int(b) < 64}
    return got
