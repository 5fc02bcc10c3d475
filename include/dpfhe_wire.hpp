// dpfhe_wire.hpp — flat wire / disk format for ciphertexts, plaintexts and switch keys (SURVEY.md §8 row f-3).
//
// The reference has no ciphertext format of its own: its demo exchanges opaque Concrete blobs through temp
// files (demo/fhe_server.py:126-130) and its only binary format is the rank/dims/raw-bytes weight file of
// GPTWeights (src/core/execution/models/gpt_weights.cpp:40-55).  This format follows the latter's spirit:
// a fixed little-endian header, then the raw u64 payload exactly as the C ABI consumes it.
//
//   offset  size  field
//   0       8     magic "DPFHEv1\0"
//   8       4     log_n
//   12      4     n_limbs (L)
//   16      4     kind: 1 = ciphertext batch [count][2][L][N], 2 = switch key [L][2][L][N] (count = 1),
//                       3 = plaintext [count][L][N]
//                       4 = hybrid switch key [L-1][2][L][N] (the last modulus is the special prime; count = 1),
//                       5 = grouped hybrid switch key [ceil((L-K)/K)][2][L][N] with count = K special primes (1 <= K <= 4, 2K <= L)
//                       6 = public key [2][L][N] (b, a) (count = 1)
//                       7 = seeded ciphertexts (DESIGN.md §2.23): a 5-word prefix (the public seed as four LE words, then first_index)
//                           and c0 [count][L][N]
//                       8 = seeded switch key: a 5-word prefix (the public seed as four LE words, then the item number: 0 for the
//                           relinearisation key, else the Galois element) and the b rows [digits][L][N], count = K special primes
//                           (0 <= K <= 4, 2K <= L; digits = L for K = 0, else ceil((L-K)/K))
//                      10 = compact ciphertexts (DESIGN.md §2.24): a 2-word prefix (bits, t_plain) and [count][2][N bits / 64] packed
//                           words; n_limbs = 1, moduli[0] = q0, form = 0 (coefficient).  2 <= bits with N 2^bits < q0; t_plain = 0
//                           (CKKS) or odd with 3 <= t_plain < 2^(bits-1)
//   20      4     form: 1 = evaluation (NTT, bit-reversed order), 0 = coefficient
//   24      8     count
//   32      128   moduli[16] (unused entries 0)
//   160     ...   payload, u64 little-endian
#pragma once

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace deeppowers {
namespace api {
namespace fhe {

// HybridSwitchKey: n_limbs counts the special prime (the last modulus); payload [n_limbs-1][2][n_limbs][N]
// GroupedSwitchKey: n_limbs counts the K = count special primes at the end of the basis; payload [ceil((n_limbs-K)/K)][2][n_limbs][N]
enum class WireKind : std::uint32_t {
    Ciphertexts = 1, SwitchKey = 2, Plaintexts = 3, HybridSwitchKey = 4, GroupedSwitchKey = 5, PublicKey = 6, SeededCiphertexts = 7,
    SeededSwitchKey = 8, CompactCiphertexts = 10
};
constexpr std::size_t kSeededPrefixWords = 5;   // the public seed (4 words) and first_index / the item number
constexpr std::size_t kCompactPrefixWords = 2;  // bits, t_plain

struct WireHeader {
    char magic[8];
    std::uint32_t log_n, n_limbs, kind, form;
    std::uint64_t count;
    std::uint64_t moduli[16];
};
static_assert(sizeof(WireHeader) == 160, "wire header must be 160 bytes");

// the prefix (bits, t_plain) of compact ciphertexts against their header, which it completes: one limb, coefficient form,
// 2 <= bits with N 2^bits < moduli[0], t_plain 0 or odd with 3 <= t_plain < 2^(bits-1)
inline void check_compact_prefix(const WireHeader &h, const std::uint64_t *prefix) {
    if (h.n_limbs != 1 || h.form != 0) throw std::runtime_error("dpfhe wire: compact ciphertexts are one limb in coefficient form");
    const std::uint64_t bits = prefix[0], t = prefix[1];
    // compared without a sum (log_n <= 17 is checked first), so that no `bits` wraps past the range check
    if (bits < 2 || bits >= 64 - std::uint64_t(h.log_n) || (std::uint64_t(1) << (bits + h.log_n)) >= h.moduli[0])
        throw std::runtime_error("dpfhe wire: bits of compact ciphertexts out of range for q0");
    if (t && (!(t & 1) || t < 3 || t >= (std::uint64_t(1) << (bits - 1))))
        throw std::runtime_error("dpfhe wire: plaintext modulus of compact ciphertexts must be 0 or odd with 3 <= t < 2^(bits-1)");
}

// words of payload a header announces; throws on an unknown kind, bad parameters or a count whose byte size does not fit
// size_t (a header is untrusted input: the count of a file must never be able to wrap the size computation).  Compact ciphertexts
// are sized by their prefix, the payload's first two words, which `prefix` points at (checked here).
inline std::size_t wire_payload_words(const WireHeader &h, const std::uint64_t *prefix = nullptr) {
    if (h.log_n < 1 || h.log_n > 17 || h.n_limbs < 1 || h.n_limbs > 16) throw std::runtime_error("dpfhe wire: bad parameters");
    const std::size_t poly = (std::size_t(1) << h.log_n) * h.n_limbs;   // <= 2^21 words
    const std::size_t max_words = static_cast<std::size_t>(-1) / 8;
    auto checked = [&](std::uint64_t count, std::size_t per_item) -> std::size_t {
        if (count > max_words / per_item) throw std::runtime_error("dpfhe wire: count does not fit in memory");
        return static_cast<std::size_t>(count) * per_item;
    };
    switch (static_cast<WireKind>(h.kind)) {
        case WireKind::Ciphertexts: return checked(h.count, 2 * poly);
        case WireKind::SwitchKey: return std::size_t(2) * h.n_limbs * poly;
        case WireKind::Plaintexts: return checked(h.count, poly);
        case WireKind::HybridSwitchKey: return std::size_t(2) * (h.n_limbs - 1) * poly;
        case WireKind::PublicKey: return std::size_t(2) * poly;
        case WireKind::GroupedSwitchKey: {
            if (h.count < 1 || h.count > 4 || 2 * h.count > h.n_limbs) throw std::runtime_error("dpfhe wire: bad number of special primes");
            const std::size_t k = static_cast<std::size_t>(h.count), digits = (h.n_limbs - k + k - 1) / k;
            return std::size_t(2) * digits * poly;
        }
        case WireKind::SeededCiphertexts:
            if (h.count < 1) throw std::runtime_error("dpfhe wire: no seeded ciphertexts");
            return kSeededPrefixWords + checked(h.count, poly);
        case WireKind::SeededSwitchKey: {
            if (h.count > 4 || 2 * h.count > h.n_limbs) throw std::runtime_error("dpfhe wire: bad number of special primes");
            const std::size_t k = static_cast<std::size_t>(h.count), digits = k ? (h.n_limbs - k + k - 1) / k : h.n_limbs;
            return kSeededPrefixWords + digits * poly;
        }
        case WireKind::CompactCiphertexts:
            if (!prefix) throw std::runtime_error("dpfhe wire: compact ciphertexts are sized by their prefix");
            check_compact_prefix(h, prefix);
            if (h.count < 1) throw std::runtime_error("dpfhe wire: no compact ciphertexts");
            return kCompactPrefixWords + checked(h.count, 2 * ((std::size_t(1) << h.log_n) / 64) * static_cast<std::size_t>(prefix[0]));
    }
    throw std::runtime_error("dpfhe wire: unknown kind");
}

// the prefix of a seeded kind, which the header does not describe: the item numbers first_index .. first_index + count - 1 of seeded
// ciphertexts must not wrap, and a seeded key's item number is 0 or a Galois element (odd, < 2N)
inline void check_wire_prefix(const WireHeader &h, const std::uint64_t *payload) {
    if (h.kind == static_cast<std::uint32_t>(WireKind::SeededCiphertexts) && payload[4] > ~std::uint64_t(0) - (h.count - 1))
        throw std::runtime_error("dpfhe wire: item numbers of seeded ciphertexts wrap");
    if (h.kind == static_cast<std::uint32_t>(WireKind::SeededSwitchKey) && payload[4] != 0 &&
        (!(payload[4] & 1) || payload[4] >= (std::uint64_t(2) << h.log_n)))
        throw std::runtime_error("dpfhe wire: item number of a seeded key is neither 0 nor a Galois element");
}

inline WireHeader make_wire_header(unsigned log_n, unsigned n_limbs, WireKind kind, std::uint64_t count, const std::uint64_t *moduli) {
    WireHeader h;
    std::memset(&h, 0, sizeof(h));
    std::memcpy(h.magic, "DPFHEv1", 8);
    h.log_n = log_n;
    h.n_limbs = n_limbs;
    h.kind = static_cast<std::uint32_t>(kind);
    h.form = 1;
    h.count = count;
    for (unsigned l = 0; l < n_limbs && l < 16; ++l) h.moduli[l] = moduli[l];
    return h;
}

inline void write_wire_file(const std::string &path, const WireHeader &h, const std::uint64_t *payload) {
    std::FILE *f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("dpfhe wire: cannot open " + path + " for writing");
    const std::size_t words = wire_payload_words(h, payload);
    check_wire_prefix(h, payload);
    const bool ok = std::fwrite(&h, sizeof(h), 1, f) == 1 && std::fwrite(payload, 8, words, f) == words;
    std::fclose(f);
    if (!ok) throw std::runtime_error("dpfhe wire: short write to " + path);
}

// Reads a whole file.  The header is validated before anything is sized from it: the payload the header announces must be
// exactly what the file holds (so a forged count can neither wrap the size computation nor make the caller trust more
// items than were read), and the file is closed on every path.
inline WireHeader read_wire_file(const std::string &path, std::vector<std::uint64_t> &payload) {
    struct Closer {
        std::FILE *f;
        ~Closer() { if (f) std::fclose(f); }
    } file{std::fopen(path.c_str(), "rb")};
    if (!file.f) throw std::runtime_error("dpfhe wire: cannot open " + path);
    WireHeader h;
    if (std::fread(&h, sizeof(h), 1, file.f) != 1 || std::memcmp(h.magic, "DPFHEv1", 8) != 0)
        throw std::runtime_error("dpfhe wire: " + path + " is not a DPFHEv1 file");
    std::uint64_t prefix[kCompactPrefixWords] = {0, 0};
    if (h.kind == static_cast<std::uint32_t>(WireKind::CompactCiphertexts) && std::fread(prefix, 8, kCompactPrefixWords, file.f) != kCompactPrefixWords)
        throw std::runtime_error("dpfhe wire: truncated payload in " + path);
    std::size_t words = 0;
    try {
        words = wire_payload_words(h, prefix);
    } catch (const std::runtime_error &e) {
        throw std::runtime_error(std::string(e.what()) + " in " + path);
    }
    if (std::fseek(file.f, 0, SEEK_END) != 0) throw std::runtime_error("dpfhe wire: cannot seek in " + path);
    const long end = std::ftell(file.f);
    if (end < 0 || static_cast<unsigned long long>(end) != sizeof(h) + 8ull * words)
        throw std::runtime_error("dpfhe wire: size of " + path + " does not match its header");
    if (std::fseek(file.f, static_cast<long>(sizeof(h)), SEEK_SET) != 0) throw std::runtime_error("dpfhe wire: cannot seek in " + path);
    payload.resize(words);
    if (std::fread(payload.data(), 8, words, file.f) != words) throw std::runtime_error("dpfhe wire: truncated payload in " + path);
    try {
        check_wire_prefix(h, payload.data());
    } catch (const std::runtime_error &e) {
        throw std::runtime_error(std::string(e.what()) + " in " + path);
    }
    return h;
}

}  // namespace fhe
}  // namespace api
}  // namespace deeppowers
