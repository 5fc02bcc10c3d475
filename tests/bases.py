"""Catalogue of moduli bases beyond the default one, shared by the CPU (emulator) and GPU tests.

The default basis (DESIGN.md §2.1) takes three shortcuts: every modulus is k * 2^32 + 1 (the dpfhe::fast kernels run),
qmax < 2 qmin (a digit is not word-reduced when it moves to another limb) and floor(2^64 / q) == 16 (the forward transform's
store canonicalises with one conditional subtraction, canon_near60).  Each basis here turns a different set of them off, and
`check_paths` asserts the set, so that a later edit of a basis cannot silently stop covering a path.

Every prime is 1 mod 2^15, so one basis is valid at every supported N; six limbs, so that two special primes (K = 2) leave a
ragged last digit as well as foreign digits.  The primes are derived, not listed, with the oracle's primality test.
"""

TWO_N_MAX = 1 << 15          # 2N at N = 16384
FAST_STEP = 1 << 32
N_LIMBS = 6


def is_fast(q):
    return q & 0xFFFFFFFF == 1


def _scan(lib, start, step, want_fast, count=1):
    """`count` primes c = start, start + step, ... (step may be negative) with c = 1 mod 2^15 and is_fast(c) == want_fast"""
    assert start % TWO_N_MAX == 1 and step % TWO_N_MAX == 0
    out, c = [], start
    while len(out) < count:
        if is_fast(c) == want_fast and lib.dpo_is_prime(c):
            out.append(c)
        c += step
    return out


def _generic_prime(lib, bits):
    """the largest generic (not k * 2^32 + 1) NTT prime below 2^bits"""
    return _scan(lib, (1 << bits) - TWO_N_MAX + 1, -TWO_N_MAX, False)[0]


def _fast_prime(lib, bits):
    """the smallest k * 2^32 + 1 prime above 2^(bits-1)"""
    return _scan(lib, (1 << (bits - 1)) + 1, FAST_STEP, True)[0]


def _smallest_generic(lib):
    """the smallest generic NTT prime the context accepts (q > 2^33): bar_shift = 32, the device Barrett shifts by zero"""
    return _scan(lib, (1 << 33) + 1, TWO_N_MAX, False)[0]


def derive(lib):
    """{basis id: list of six moduli}; the last K of a basis are the special primes of the K-special-prime families"""
    mixed = [_generic_prime(lib, 59), _generic_prime(lib, 50), _generic_prime(lib, 40), _smallest_generic(lib),
             _generic_prime(lib, 55), _generic_prime(lib, 45)]
    return {
        # special primes (55 and 45 bits) between the ciphertext moduli's sizes
        "gen_mixed": mixed,
        # the same set ascending: the special primes are the largest
        "gen_ascending": sorted(mixed),
        # generic, but canon_near60 applies to every limb and no lift reduction: the generic kernels' own shortcuts
        "gen_near60": _scan(lib, (1 << 60) - TWO_N_MAX + 1, -TWO_N_MAX, False, N_LIMBS),
        # fast arithmetic without the store shortcut, with the lift reduction
        "fast_mixed": [_fast_prime(lib, b) for b in (37, 40, 45, 48, 50, 55)],
        # fast arithmetic without the store shortcut and without the lift reduction
        "fast_narrow": _scan(lib, (1 << 48) - FAST_STEP + 1, -FAST_STEP, True, N_LIMBS),
    }


# the paths each basis is meant to select: (fast kernels, lift reduction, limbs taking canon_near60)
PATHS = {
    "gen_mixed": (False, True, "none"),
    "gen_ascending": (False, True, "none"),
    "gen_near60": (False, False, "all"),
    "fast_mixed": (True, True, "none"),
    "fast_narrow": (True, False, "none"),
}

SMALLEST_GENERIC = 8590163969            # 2^33 + 7 * 2^15 + 1
SMALLEST_FAST_37 = 77309411329           # 18 * 2^32 + 1
LARGEST_GENERIC = 1152921504606748673    # 2^60 - 3 * 2^15 + 1


def selects(moduli):
    """what the library derives from a basis (abi.cu dpfhe_context_create, modarith.cuh canon_near60_applies)"""
    fast = all(is_fast(q) for q in moduli)
    lift_reduce = not max(moduli) < 2 * min(moduli)
    near60 = [2**64 // q == 16 for q in moduli]
    return fast, lift_reduce, "all" if all(near60) else ("none" if not any(near60) else "some")


def check_paths(bases):
    for name, mods in bases.items():
        assert len(mods) == N_LIMBS and len(set(mods)) == N_LIMBS, name
        assert all(2**33 < q < 2**60 and q % TWO_N_MAX == 1 for q in mods), name
        assert selects(mods) == PATHS[name], (name, selects(mods))
    assert SMALLEST_GENERIC in bases["gen_mixed"] and SMALLEST_GENERIC.bit_length() == 34
    assert bases["gen_near60"][0] == LARGEST_GENERIC
    assert min(bases["fast_mixed"]) == SMALLEST_FAST_37


_cache = {}


def catalogue(oracle_mod):
    """the checked catalogue (derived once per process)"""
    if not _cache:
        bases = derive(oracle_mod.lib())
        check_paths(bases)
        _cache.update(bases)
    return dict(_cache)


NAMES = list(PATHS)
