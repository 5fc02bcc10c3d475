// host_params.hpp — host-side derivation of the parameter set (DESIGN.md §2.1):
// NTT-friendly primes, smallest primitive 2N-th roots, twiddle tables in the device layout.
// Independent of oracle/ (the product never links the oracle); tests compare the two.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "types.hpp"

namespace dpfhe {

struct HostLimb {
    LimbParams lp;
    uint64_t psi;
    std::vector<uint64_t> root_powers;      // psi^bitrev(i), natural table order
    std::vector<uint64_t> inv_root_powers;  // psi^-bitrev(i)
    std::vector<U64x2> tw;                  // device layout (tw_pos), with Shoup companions
    std::vector<U64x2> itw;
};

struct HostParams {
    unsigned log_n = 0, L = 0;
    std::vector<HostLimb> limbs;
};

// returns "" on success, else an error message
std::string build_host_params(unsigned log_n, unsigned L, const uint64_t *moduli, HostParams &out);

// constants for dropping the last limb of `hp` (t_plain = 0: plain rounding); requires hp.L >= 2 and t_plain < q_last
void build_ms_consts(const HostParams &hp, uint64_t t_plain, MsConsts &K);

// constants of grouped hybrid key switching with the last K limbs of `hp` as special primes (types.hpp: GroupConsts); Km
// receives the constants of the division by P.  Requires 1 <= K <= KS_MAX_SPECIAL, K < hp.L, t_plain < every special prime.
void build_group_consts(const HostParams &hp, unsigned K, uint64_t t_plain, GroupConsts &G, MsConsts &Km);
// multiply-and-rescale (DESIGN.md §2.19): the constants of the division by P' = P * qbar, qbar = q_{L-K-1} the last ciphertext modulus:
// G and Km as build_group_consts would build them for P', and R the dropped limb's row (its pointers stay null: the launcher sets
// them).  Requires what build_group_consts does, L - K >= 2 and t_plain < qbar.
void build_rescale_consts(const HostParams &hp, unsigned K, uint64_t t_plain, GroupConsts &G, MsConsts &Km, RescaleConsts &R);

// CKKS slot encoding (DESIGN.md §2.12): the twiddles (cos, sin)(pi k / N), k < N, each correctly rounded; the slot
// permutation t_j, j < N/2; and 2^e mod q_l, [L][CKKS_POW2_E]
void build_ckks_tables(const HostParams &hp, std::vector<Cplx> &tw, std::vector<uint32_t> &tj, std::vector<uint64_t> &pow2);
// decoding constants (Garner inverses, the digits of (Q-1)/2, the moduli as doubles) with the divisor `scale`
void build_ckks_consts(const HostParams &hp, double scale, CkksConsts &K);

// BGV slot encoding (DESIGN.md §2.13).  A valid plaintext modulus is a prime t < 2^31 with t = 1 (mod 2N).
bool bgv_plain_modulus_valid(unsigned log_n, uint64_t t);
// the constants of the 32-bit arithmetic modulo a prime t < 2^31 (modarith.cuh: shoup32, reduce64_32)
Mod32 make_mod32(uint64_t t);
// zeta = g^((t-1)/2N), g the least quadratic non-residue mod t (requires a valid t)
uint64_t bgv_zeta(unsigned log_n, uint64_t t);
// tab receives [5][N] words: the four twiddle rows of BgvTables::tw, then the slot positions; T the constants of t (its
// pointers stay null: the caller places tab).  Returns false, building nothing, for an invalid t.
bool build_bgv_tables(const HostParams &hp, uint64_t t, std::vector<uint32_t> &tab, BgvTables &T);
// decoding constants: CKKS's Garner inverses and digits of (Q-1)/2, q_i mod t and Q mod t (requires a valid t)
void build_bgv_consts(const HostParams &hp, uint64_t t, BgvConsts &K);

// Compact ciphertexts (DESIGN.md §2.24): the constants of the switch between q0 and 2^bits at N = 2^log_n, for arguments the caller has
// checked (2 <= bits, N 2^bits < q0, t_plain = 0 or odd with 3 <= t_plain < 2^(bits-1))
void build_compact_args(uint64_t q0, unsigned log_n, unsigned bits, uint64_t t_plain, CompactArgs &A);

// key generation and encryption (DESIGN.md §2.14): the constants of one launch of the key / encryption kernels for the 32-byte seed,
// K special primes (0: per-limb digits) and the noise factor t (t = 0: unscaled); the pointers and item numbers stay unset
KeyArgs build_key_args(const HostParams &hp, const uint8_t seed[32], unsigned K, uint64_t t_plain);

uint64_t host_mulmod(uint64_t a, uint64_t b, uint64_t q);
uint64_t host_powmod(uint64_t a, uint64_t e, uint64_t q);
bool host_is_prime(uint64_t n);

}  // namespace dpfhe
