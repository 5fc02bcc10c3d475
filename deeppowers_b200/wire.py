"""Python mirror of include/dpfhe_wire.hpp (flat DPFHEv1 files: 160-byte header + raw u64 payload)."""
import struct

import numpy as np

MAGIC = b"DPFHEv1\x00"
CIPHERTEXTS, SWITCH_KEY, PLAINTEXTS, HYBRID_SWITCH_KEY, GROUPED_SWITCH_KEY = 1, 2, 3, 4, 5   # hybrid / grouped: n_limbs includes the special primes;
# a grouped key's `count` is the number of special primes K, its payload [ceil((n_limbs-K)/K)][2][n_limbs][N]
PUBLIC_KEY = 6   # (b, a): payload [2][n_limbs][N], count = 1
# seeded objects (DESIGN.md section 2.23): a 5-word prefix (the public seed as four LE words, then first_index / the key's item number)
# and c0 [count][n_limbs][N] (SEEDED_CIPHERTEXTS) or the b rows [digits][n_limbs][N] (SEEDED_SWITCH_KEY, count = K special primes, 0 .. 4)
SEEDED_CIPHERTEXTS, SEEDED_SWITCH_KEY = 7, 8
SEEDED_PREFIX_WORDS = 5
# compact ciphertexts (DESIGN.md section 2.24): a 2-word prefix (bits, t_plain) and [count][2][N bits / 64] packed words; n_limbs = 1,
# moduli[0] = q0, form = 0 (coefficient)
COMPACT_CIPHERTEXTS = 10
COMPACT_PREFIX_WORDS = 2
_HDR = struct.Struct("<8sIIIIQ16Q")


def check_compact_prefix(log_n, n_limbs, form, q0, bits, t_plain):
    """the prefix (bits, t_plain) of compact ciphertexts against their header"""
    if n_limbs != 1 or form != 0:
        raise ValueError("compact ciphertexts are one limb in coefficient form")
    if not (2 <= bits and bits + log_n < 64 and (1 << (bits + log_n)) < q0):
        raise ValueError("bits of compact ciphertexts out of range for q0")
    if t_plain and (not t_plain & 1 or not 3 <= t_plain < 1 << (bits - 1)):
        raise ValueError("plaintext modulus of compact ciphertexts must be 0 or odd with 3 <= t < 2^(bits-1)")


def payload_words(log_n, n_limbs, kind, count, compact=None):
    """compact: (form, q0, bits, t_plain) of compact ciphertexts, whose payload is sized by its prefix"""
    if not (1 <= log_n <= 17 and 1 <= n_limbs <= 16):
        raise ValueError("bad parameters")
    if kind not in (CIPHERTEXTS, SWITCH_KEY, PLAINTEXTS, HYBRID_SWITCH_KEY, GROUPED_SWITCH_KEY, PUBLIC_KEY, SEEDED_CIPHERTEXTS, SEEDED_SWITCH_KEY,
                    COMPACT_CIPHERTEXTS):
        raise ValueError("unknown kind")
    poly = (1 << log_n) * n_limbs
    if kind == COMPACT_CIPHERTEXTS:
        if compact is None:
            raise ValueError("compact ciphertexts are sized by their prefix")
        form, q0, bits, t_plain = compact
        check_compact_prefix(log_n, n_limbs, form, q0, bits, t_plain)
        if count < 1:
            raise ValueError("no compact ciphertexts")
        return COMPACT_PREFIX_WORDS + count * 2 * (1 << log_n) // 64 * bits
    if kind == SEEDED_CIPHERTEXTS:
        if count < 1:
            raise ValueError("no seeded ciphertexts")
        return SEEDED_PREFIX_WORDS + count * poly
    if kind == SEEDED_SWITCH_KEY:
        if not (0 <= count <= 4 and 2 * count <= n_limbs):
            raise ValueError("bad number of special primes")
        return SEEDED_PREFIX_WORDS + (-(-(n_limbs - count) // count) if count else n_limbs) * poly
    if kind == GROUPED_SWITCH_KEY:
        if not (1 <= count <= 4 and 2 * count <= n_limbs):
            raise ValueError("bad number of special primes")
        return 2 * (-(-(n_limbs - count) // count)) * poly
    return {CIPHERTEXTS: count * 2 * poly, SWITCH_KEY: 2 * n_limbs * poly, PLAINTEXTS: count * poly,
            HYBRID_SWITCH_KEY: 2 * (n_limbs - 1) * poly, PUBLIC_KEY: 2 * poly}[kind]


def seeded_prefix(a_seed, number):
    """the 5-word prefix of a seeded kind: the 32-byte public seed as four little-endian words, then first_index or the item number"""
    if len(a_seed) != 32:
        raise ValueError("a public seed is 32 bytes")
    return np.concatenate([np.frombuffer(bytes(a_seed), dtype="<u8"), np.array([number], dtype="<u8")]).astype(np.uint64)


def split_seeded(payload):
    """(public seed bytes, first_index or item number, the rows) of a seeded kind's payload"""
    return payload[:4].astype("<u8").tobytes(), int(payload[4]), payload[SEEDED_PREFIX_WORDS:]


def _check_prefix(log_n, kind, count, payload):
    if kind == SEEDED_CIPHERTEXTS and int(payload[4]) + count - 1 >= 1 << 64:
        raise ValueError("item numbers of seeded ciphertexts wrap")
    if kind == SEEDED_SWITCH_KEY:
        item = int(payload[4])
        if item and (not item & 1 or item >= 2 << log_n):
            raise ValueError("item number of a seeded key is neither 0 nor a Galois element")


def compact_prefix(bits, t_plain):
    """the 2-word prefix of compact ciphertexts"""
    return np.array([bits, t_plain], dtype=np.uint64)


def write(path, log_n, n_limbs, kind, count, moduli, payload, form=1):
    payload = np.ascontiguousarray(payload, dtype="<u8").reshape(-1)
    compact = (form, int(moduli[0]), int(payload[0]), int(payload[1])) if kind == COMPACT_CIPHERTEXTS and payload.size >= 2 else None
    if payload.size != payload_words(log_n, n_limbs, kind, count, compact):
        raise ValueError("payload size does not match the header")
    _check_prefix(log_n, kind, count, payload)
    mods = list(int(m) for m in moduli) + [0] * (16 - len(moduli))
    with open(path, "wb") as f:
        f.write(_HDR.pack(MAGIC, log_n, n_limbs, kind, form, count, *mods))
        f.write(payload.tobytes())


def read(path):
    with open(path, "rb") as f:
        raw = f.read(_HDR.size)
        if len(raw) != _HDR.size:
            raise ValueError("truncated header")
        magic, log_n, n_limbs, kind, form, count, *mods = _HDR.unpack(raw)
        if magic != MAGIC:
            raise ValueError("not a DPFHEv1 file")
        compact = None
        if kind == COMPACT_CIPHERTEXTS:
            prefix = np.frombuffer(f.read(8 * COMPACT_PREFIX_WORDS), dtype="<u8")
            if prefix.size != COMPACT_PREFIX_WORDS:
                raise ValueError("truncated payload")
            compact = (form, mods[0], int(prefix[0]), int(prefix[1]))
        words = payload_words(log_n, n_limbs, kind, count, compact)
        f.seek(0, 2)
        if f.tell() != _HDR.size + 8 * words:      # the header is untrusted: it must describe exactly this file
            raise ValueError("file size does not match the header")
        f.seek(_HDR.size)
        data = np.frombuffer(f.read(words * 8), dtype="<u8")
        if data.size != words:
            raise ValueError("truncated payload")
        _check_prefix(log_n, kind, count, data)
    return {"log_n": log_n, "n_limbs": n_limbs, "kind": kind, "form": form, "count": count, "moduli": mods[:n_limbs]}, data.astype(np.uint64)
