"""Generates tests/golden/chacha20_kat.json: ChaCha20 blocks (RFC 8439 §2.3) computed by an independent implementation, the
`cryptography` package's OpenSSL ChaCha20, so that tests/keys_ref.c is pinned where that package is missing.

Each case is one 64-byte block for (key, counter, nonce): the keystream of `cryptography`'s ChaCha20 with the 16-byte
initial value counter (4 bytes, little-endian) || nonce (12 bytes), i.e. the encryption of 64 zero bytes.

    python tests/golden/make_chacha20_kat.py
"""
import json
import os
import random
import struct

from cryptography.hazmat.primitives.ciphers import Cipher, algorithms


def block(key, counter, nonce_words):
    iv = struct.pack("<I", counter) + struct.pack("<3I", *nonce_words)
    enc = Cipher(algorithms.ChaCha20(key, iv), mode=None).encryptor()
    return list(struct.unpack("<16I", enc.update(bytes(64))))


def main():
    rng = random.Random(0xC4AC4A20)
    cases = [
        # RFC 8439 §2.3.2: key 00 01 .. 1f, counter 1, nonce 00 00 00 09 00 00 00 4a 00 00 00 00
        (bytes(range(32)), 1, (0x09000000, 0x4A000000, 0)),
        (bytes(32), 0, (0, 0, 0)),
        (bytes([0xFF]) * 32, 0xFFFFFFFF, (0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)),
    ]
    for _ in range(13):
        cases.append((bytes(rng.getrandbits(8) for _ in range(32)), rng.getrandbits(32), tuple(rng.getrandbits(32) for _ in range(3))))
    out = [{"key": k.hex(), "counter": c, "nonce": list(n), "block": block(k, c, n)} for k, c, n in cases]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "chacha20_kat.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote", path, len(out), "cases")


if __name__ == "__main__":
    main()
