/* keys_ref.c — DESIGN.md §2.14 restated in C11 (TEST INFRASTRUCTURE ONLY; shares no code with deeppowers_b200/csrc).
 *
 * ChaCha20 written from RFC 8439 §2.3, the three samplers of the specification (the uniform reduction by unsigned __int128 %),
 * and the nonce table.  tests/keys_ref.py composes these rows with the oracle's transforms and pointwise operations. */
#include <stddef.h>
#include <stdint.h>

static uint32_t rol(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }

static void quarter(uint32_t *s, int a, int b, int c, int d) {
    s[a] += s[b]; s[d] ^= s[a]; s[d] = rol(s[d], 16);
    s[c] += s[d]; s[b] ^= s[c]; s[b] = rol(s[b], 12);
    s[a] += s[b]; s[d] ^= s[a]; s[d] = rol(s[d], 8);
    s[c] += s[d]; s[b] ^= s[c]; s[b] = rol(s[b], 7);
}

/* RFC 8439 §2.3: 16 output words of the block function for a 32-byte key, a 32-bit counter and a 96-bit nonce (three words) */
void kr_chacha20_block(const uint8_t key[32], uint32_t counter, const uint32_t nonce[3], uint32_t out[16]) {
    uint32_t init[16], s[16];
    init[0] = 0x61707865; init[1] = 0x3320646e; init[2] = 0x79622d32; init[3] = 0x6b206574;
    for (int i = 0; i < 8; i++)
        init[4 + i] = (uint32_t)key[4 * i] | (uint32_t)key[4 * i + 1] << 8 | (uint32_t)key[4 * i + 2] << 16 | (uint32_t)key[4 * i + 3] << 24;
    init[12] = counter;
    init[13] = nonce[0]; init[14] = nonce[1]; init[15] = nonce[2];
    for (int i = 0; i < 16; i++) s[i] = init[i];
    for (int r = 0; r < 10; r++) {
        quarter(s, 0, 4, 8, 12); quarter(s, 1, 5, 9, 13); quarter(s, 2, 6, 10, 14); quarter(s, 3, 7, 11, 15);
        quarter(s, 0, 5, 10, 15); quarter(s, 1, 6, 11, 12); quarter(s, 2, 7, 8, 13); quarter(s, 3, 4, 9, 14);
    }
    for (int i = 0; i < 16; i++) out[i] = s[i] + init[i];
}

/* the nonce word n0 of a row: domain | K << 8 | digit << 16 | limb << 24; domains 1 secret, 2 key a, 3 key e, 4 enc a, 5 enc e */
uint32_t kr_nonce0(uint32_t domain, uint32_t K, uint32_t digit, uint32_t limb) { return domain | K << 8 | digit << 16 | limb << 24; }

static void row_nonce(uint32_t n0, uint64_t item, uint32_t nonce[3]) {
    nonce[0] = n0;
    nonce[1] = (uint32_t)item;
    nonce[2] = (uint32_t)(item >> 32);
}

/* n ternary coefficients: 16 per block, s_k = floor(3 w / 2^32) - 1 */
void kr_ternary(const uint8_t seed[32], uint32_t n0, uint64_t item, size_t n, int64_t *out) {
    uint32_t nonce[3], w[16];
    row_nonce(n0, item, nonce);
    for (size_t k = 0; k < n; k++) {
        if (k % 16 == 0) kr_chacha20_block(seed, (uint32_t)(k / 16), nonce, w);
        out[k] = (int64_t)((3 * (uint64_t)w[k % 16]) >> 32) - 1;
    }
}

/* n centred binomial coefficients (eta = 21): 8 per block, r = w_2i | w_2i+1 << 32 */
void kr_cbd(const uint8_t seed[32], uint32_t n0, uint64_t item, size_t n, int64_t *out) {
    uint32_t nonce[3], w[16];
    row_nonce(n0, item, nonce);
    for (size_t k = 0; k < n; k++) {
        if (k % 8 == 0) kr_chacha20_block(seed, (uint32_t)(k / 8), nonce, w);
        const uint64_t r = (uint64_t)w[2 * (k % 8)] | (uint64_t)w[2 * (k % 8) + 1] << 32;
        out[k] = (int64_t)__builtin_popcountll(r & 0x1FFFFF) - (int64_t)__builtin_popcountll((r >> 21) & 0x1FFFFF);
    }
}

/* n uniform residues mod q: 4 per block, the 128-bit little-endian integer of words 4j .. 4j+3 reduced exactly */
void kr_uniform(const uint8_t seed[32], uint32_t n0, uint64_t item, uint64_t q, size_t n, uint64_t *out) {
    uint32_t nonce[3], w[16];
    row_nonce(n0, item, nonce);
    for (size_t k = 0; k < n; k++) {
        if (k % 4 == 0) kr_chacha20_block(seed, (uint32_t)(k / 4), nonce, w);
        const uint32_t *v = w + 4 * (k % 4);
        const unsigned __int128 x = (unsigned __int128)v[0] | (unsigned __int128)v[1] << 32 | (unsigned __int128)v[2] << 64 |
                                    (unsigned __int128)v[3] << 96;
        out[k] = (uint64_t)(x % q);
    }
}

/* the uniform reduction of one 128-bit value hi:lo (for tests of the extremes) */
uint64_t kr_reduce128(uint64_t lo, uint64_t hi, uint64_t q) {
    return (uint64_t)((((unsigned __int128)hi << 64) | lo) % q);
}
