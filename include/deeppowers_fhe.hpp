// deeppowers_fhe.hpp — C++ host API of the encrypted hot path, in the reference's house style.
//
// The reference's public header (src/api/cpp/include/deeppowers.hpp:41-87) exposes
// deeppowers::api::{Model, GenerationConfig, load_model, ...} and has no Ciphertext/Evaluator types
// (SURVEY.md §0); this header adds them next to it, as namespace deeppowers::api::fhe, following
// the same conventions:
//   - errors are C++ exceptions (std::runtime_error), as CUDA_CHECK does in
//     src/core/hal/cuda/cuda_device.cpp:9-16 — every non-zero status of the C ABI is re-thrown
//     with dpfhe_last_error() as the message;
//   - resource-owning classes are non-copyable RAII handles (compare Model's pimpl,
//     deeppowers.hpp:73-75, and CUDADevice's dtor, cuda_device.cpp:26-41);
//   - one Evaluator is bound to one device (compare hal::CUDADevice(0), src/api/cpp/src/deeppowers.cpp:15).
// Header-only over the extern "C" library (include/dpfhe.h, libdpfhe.so); no CUDA headers needed.
#pragma once

#include <array>
#include <complex>
#include <cstddef>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "dpfhe.h"

namespace deeppowers {
namespace api {
namespace fhe {

// Parameters of the ring Z_q[X]/(X^N+1) in RNS form.
struct EncryptionParameters {
    unsigned log_n = 13;                   // N = 8192
    unsigned n_limbs = 4;                  // L
    std::vector<std::uint64_t> moduli;     // empty: the L largest primes k*2^32+1 below 2^60 (the default basis)
};

// Non-owning view of `count` ciphertexts [count][2][L][N] (evaluation form) in host or device memory.
struct CiphertextBatch {
    std::uint64_t *data = nullptr;
    std::size_t count = 0;
};
struct ConstCiphertextBatch {
    const std::uint64_t *data = nullptr;
    std::size_t count = 0;
    ConstCiphertextBatch() = default;
    ConstCiphertextBatch(const std::uint64_t *d, std::size_t c) : data(d), count(c) {}
    ConstCiphertextBatch(const CiphertextBatch &b) : data(b.data), count(b.count) {}
};

namespace detail {
// the part the library objects built on an Evaluator share (below)
template <class H, void (*Destroy)(H *), int (*Apply)(H *, const std::uint64_t *, std::uint64_t *, std::size_t, void *),
          int (*ApplyHost)(H *, const std::uint64_t *, std::uint64_t *, std::size_t)>
class ContextObject;
}  // namespace detail

class Evaluator {
public:
    explicit Evaluator(const EncryptionParameters &parms, int device_id = 0) : log_n_(parms.log_n), limbs_(parms.n_limbs) {
        dpfhe_params p;
        p.log_n = parms.log_n;
        p.n_limbs = parms.n_limbs;
        p.moduli = parms.moduli.empty() ? nullptr : parms.moduli.data();
        if (!parms.moduli.empty() && parms.moduli.size() != parms.n_limbs)
            throw std::runtime_error("EncryptionParameters: moduli.size() must equal n_limbs");
        check(dpfhe_context_create(&p, device_id, &ctx_));
    }
    ~Evaluator() { dpfhe_context_destroy(ctx_); }
    Evaluator(const Evaluator &) = delete;
    Evaluator &operator=(const Evaluator &) = delete;

    std::size_t poly_degree() const { return std::size_t(1) << log_n_; }
    unsigned limbs() const { return limbs_; }
    std::size_t poly_words() const { return poly_degree() * limbs_; }           // [L][N]
    std::size_t ciphertext_words() const { return 2 * poly_words(); }           // [2][L][N]
    std::size_t switch_key_words() const { return 2 * limbs_ * poly_words(); }  // [L][2][L][N]
    std::uint64_t modulus(unsigned limb) const {
        std::uint64_t q = 0;
        check(dpfhe_get_modulus(ctx_, limb, &q));
        return q;
    }
    // Galois element of a rotation by `steps` slots: 5^steps mod 2N
    std::uint64_t galois_element(long steps) const {
        const std::uint64_t two_n = std::uint64_t(2) << log_n_, half = poly_degree() / 2;
        std::uint64_t e = ((steps % (long)half) + (long)half) % (long)half, g = 1, b = 5;
        for (; e; e >>= 1, b = b * b % two_n)
            if (e & 1) g = g * b % two_n;
        return g;
    }

    // ---- CKKS slot encoding (DESIGN.md §2.12): `count` vectors of slot_count() slots <-> `count` plaintexts of poly_words()
    //      words in evaluation form; synchronous host-buffer calls ----
    std::size_t slot_count() const { return poly_degree() / 2; }
    void encode_ckks(const std::complex<double> *slots, std::size_t count, double scale, std::uint64_t *plain_eval) {
        check(dpfhe_ckks_encode_host(ctx_, reinterpret_cast<const double *>(slots), plain_eval, count, scale));
    }
    void decode_ckks(const std::uint64_t *plain_eval, std::size_t count, double scale, std::complex<double> *slots) {
        check(dpfhe_ckks_decode_host(ctx_, plain_eval, reinterpret_cast<double *>(slots), count, scale));
    }

    // ---- BGV slot encoding (DESIGN.md §2.13): `count` vectors of poly_degree() slots ([2][N/2], int64 in, values in
    //      [0, plain_modulus) out) <-> `count` plaintexts of poly_words() words in evaluation form; synchronous host-buffer calls ----
    void encode_bgv(const std::int64_t *slots, std::size_t count, std::uint64_t plain_modulus, std::uint64_t *plain_eval) {
        check(dpfhe_bgv_encode_host(ctx_, slots, plain_eval, count, plain_modulus));
    }
    void decode_bgv(const std::uint64_t *plain_eval, std::size_t count, std::uint64_t plain_modulus, std::uint64_t *slots) {
        check(dpfhe_bgv_decode_host(ctx_, plain_eval, slots, count, plain_modulus));
    }

    // ---- keys, encryption, decryption (DESIGN.md §2.14), drawn from the ChaCha20 stream of a 32-byte seed.  The seed is the
    //      storage form of the secret.  special = 0: per-limb-digit keys (switch_key_words()), else grouped keys of
    //      grouped_digits(special) digits; plain_modulus = 0 leaves the noise unscaled (CKKS).  Host forms are synchronous. ----
    typedef std::array<std::uint8_t, 32> Seed;
    static Seed random_seed() {
        Seed s;
        check(dpfhe_random_seed(s.data()));
        return s;
    }
    std::size_t key_words(unsigned special) const { return (special ? grouped_digits(special) : limbs_) * 2 * poly_words(); }
    void generate_secret(const Seed &seed, std::uint64_t *secret) { check(dpfhe_secret_keygen_host(ctx_, seed.data(), secret)); }
    void generate_relin_key(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t *key) {
        check(dpfhe_relin_keygen_host(ctx_, special, plain_modulus, secret, seed.data(), key));
    }
    // keys [steps.size()][key_words(special)] for rotations by steps[i] slots
    void generate_galois_keys(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const std::vector<long> &steps,
                              const Seed &seed, std::uint64_t *keys) {
        generate_galois_keys_for_elements(special, plain_modulus, secret, galois_elements(steps), seed, keys);
    }
    // the same for Galois elements (odd, < 2N), e.g. the conjugation 2N - 1
    void generate_galois_keys_for_elements(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret,
                                           const std::vector<std::uint64_t> &elements, const Seed &seed, std::uint64_t *keys) {
        check(dpfhe_galois_keygen_host(ctx_, special, plain_modulus, secret, elements.size(), elements.data(), seed.data(), keys));
    }
    void encrypt(std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t first_index,
                 const std::uint64_t *plain_eval, CiphertextBatch out) {
        check(dpfhe_encrypt_host(ctx_, plain_modulus, secret, seed.data(), first_index, plain_eval, out.data, out.count));
    }
    // ct holds ct.count ciphertexts of n_comp (2 or 3: before relinearisation) polynomials each
    void decrypt(const std::uint64_t *secret, ConstCiphertextBatch ct, std::uint64_t *plain_eval, unsigned n_comp = 2) {
        check(dpfhe_decrypt_host(ctx_, secret, ct.data, n_comp, plain_eval, ct.count));
    }
    void generate_secret_device(const Seed &seed, std::uint64_t *secret, void *stream = nullptr) {
        check(dpfhe_secret_keygen(ctx_, seed.data(), secret, stream));
    }
    void generate_relin_key_device(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed,
                                   std::uint64_t *key, void *stream = nullptr) {
        check(dpfhe_relin_keygen(ctx_, special, plain_modulus, secret, seed.data(), key, stream));
    }
    void generate_galois_keys_device(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const std::vector<long> &steps,
                                     const Seed &seed, std::uint64_t *keys, void *stream = nullptr) {
        generate_galois_keys_for_elements_device(special, plain_modulus, secret, galois_elements(steps), seed, keys, stream);
    }
    void generate_galois_keys_for_elements_device(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret,
                                                  const std::vector<std::uint64_t> &elements, const Seed &seed, std::uint64_t *keys,
                                                  void *stream = nullptr) {
        check(dpfhe_galois_keygen(ctx_, special, plain_modulus, secret, elements.size(), elements.data(), seed.data(), keys, stream));
    }
    void encrypt_device(std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t first_index,
                        const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        check(dpfhe_encrypt(ctx_, plain_modulus, secret, seed.data(), first_index, plain_eval, out.data, out.count, stream));
    }
    void decrypt_device(const std::uint64_t *secret, ConstCiphertextBatch ct, std::uint64_t *plain_eval, unsigned n_comp = 2,
                        void *stream = nullptr) {
        check(dpfhe_decrypt(ctx_, secret, ct.data, n_comp, plain_eval, ct.count, stream));
    }
    // ---- public keys: public_key [2 * poly_words()] made by the key owner (secret and seed); anyone holding it encrypts with a
    //      seed of their own, which must stay as secret as the plaintexts.  Use a public key with the plain_modulus it was made with.
    std::size_t public_key_words() const { return 2 * poly_words(); }
    void generate_public_key(std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t *public_key) {
        check(dpfhe_public_keygen_host(ctx_, plain_modulus, secret, seed.data(), public_key));
    }
    void generate_public_key_device(std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t *public_key,
                                    void *stream = nullptr) {
        check(dpfhe_public_keygen(ctx_, plain_modulus, secret, seed.data(), public_key, stream));
    }
    void encrypt_public(std::uint64_t plain_modulus, const std::uint64_t *public_key, const Seed &seed, std::uint64_t first_index,
                        const std::uint64_t *plain_eval, CiphertextBatch out) {
        check(dpfhe_encrypt_public_host(ctx_, plain_modulus, public_key, seed.data(), first_index, plain_eval, out.data, out.count));
    }
    void encrypt_public_device(std::uint64_t plain_modulus, const std::uint64_t *public_key, const Seed &seed, std::uint64_t first_index,
                               const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        check(dpfhe_encrypt_public(ctx_, plain_modulus, public_key, seed.data(), first_index, plain_eval, out.data, out.count, stream));
    }
    // ---- the keyless calls at level `level` of the chain (DESIGN.md §2.22): bit for bit the call of the same name on an evaluator over
    //      the first `level` limbs; plaintexts carry level * poly_degree() words, ciphertexts twice that.  The secret and the public key
    //      are this evaluator's top-level ones.  1 <= level <= limbs().  Under special primes these encode, encrypt, decrypt and decode
    //      the ciphertexts of every level on this one evaluator. ----
    void encode_ckks(unsigned level, const std::complex<double> *slots, std::size_t count, double scale, std::uint64_t *plain_eval) {
        check(dpfhe_ckks_encode_level_host(ctx_, level, reinterpret_cast<const double *>(slots), plain_eval, count, scale));
    }
    void decode_ckks(unsigned level, const std::uint64_t *plain_eval, std::size_t count, double scale, std::complex<double> *slots) {
        check(dpfhe_ckks_decode_level_host(ctx_, level, plain_eval, reinterpret_cast<double *>(slots), count, scale));
    }
    void encode_bgv(unsigned level, const std::int64_t *slots, std::size_t count, std::uint64_t plain_modulus, std::uint64_t *plain_eval) {
        check(dpfhe_bgv_encode_level_host(ctx_, level, slots, plain_eval, count, plain_modulus));
    }
    void decode_bgv(unsigned level, const std::uint64_t *plain_eval, std::size_t count, std::uint64_t plain_modulus, std::uint64_t *slots) {
        check(dpfhe_bgv_decode_level_host(ctx_, level, plain_eval, slots, count, plain_modulus));
    }
    void encrypt(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t first_index,
                 const std::uint64_t *plain_eval, CiphertextBatch out) {
        check(dpfhe_encrypt_level_host(ctx_, level, plain_modulus, secret, seed.data(), first_index, plain_eval, out.data, out.count));
    }
    void decrypt(unsigned level, const std::uint64_t *secret, ConstCiphertextBatch ct, std::uint64_t *plain_eval, unsigned n_comp = 2) {
        check(dpfhe_decrypt_level_host(ctx_, level, secret, ct.data, n_comp, plain_eval, ct.count));
    }
    void encrypt_device(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t first_index,
                        const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        check(dpfhe_encrypt_level(ctx_, level, plain_modulus, secret, seed.data(), first_index, plain_eval, out.data, out.count, stream));
    }
    void decrypt_device(unsigned level, const std::uint64_t *secret, ConstCiphertextBatch ct, std::uint64_t *plain_eval, unsigned n_comp = 2,
                        void *stream = nullptr) {
        check(dpfhe_decrypt_level(ctx_, level, secret, ct.data, n_comp, plain_eval, ct.count, stream));
    }
    void encrypt_public(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *public_key, const Seed &seed, std::uint64_t first_index,
                        const std::uint64_t *plain_eval, CiphertextBatch out) {
        check(dpfhe_encrypt_public_level_host(ctx_, level, plain_modulus, public_key, seed.data(), first_index, plain_eval, out.data, out.count));
    }
    void encrypt_public_device(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *public_key, const Seed &seed,
                               std::uint64_t first_index, const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        check(dpfhe_encrypt_public_level(ctx_, level, plain_modulus, public_key, seed.data(), first_index, plain_eval, out.data, out.count,
                                         stream));
    }
    std::vector<std::uint64_t> galois_elements(const std::vector<long> &steps) const {
        std::vector<std::uint64_t> elts;
        for (long k : steps) elts.push_back(galois_element(k));
        return elts;
    }

    // ---- seeded ciphertexts and switch keys (DESIGN.md §2.23): only c0 [count][level][N] / the b rows [n][digits][L][N] are made;
    //      the `a` rows come from the public seed of the key owner's seed (public_seed), and the expand / upload calls give the full
    //      ciphertexts [count][2][level][N] and keys [n][digits][2][L][N].  Key items: 0 (relinearisation key) or a Galois element. ----
    static Seed public_seed(const Seed &seed) {
        Seed a;
        check(dpfhe_seeded_public_seed(seed.data(), a.data()));
        return a;
    }
    std::size_t seeded_key_words(unsigned special) const { return key_words(special) / 2; }
    void encrypt_seeded(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t first_index,
                        const std::uint64_t *plain_eval, std::size_t count, std::uint64_t *c0) {
        check(dpfhe_encrypt_seeded_level_host(ctx_, level, plain_modulus, secret, seed.data(), first_index, plain_eval, c0, count));
    }
    void encrypt_seeded_device(unsigned level, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed,
                               std::uint64_t first_index, const std::uint64_t *plain_eval, std::size_t count, std::uint64_t *c0,
                               void *stream = nullptr) {
        check(dpfhe_encrypt_seeded_level(ctx_, level, plain_modulus, secret, seed.data(), first_index, plain_eval, c0, count, stream));
    }
    void generate_relin_key_seeded(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const Seed &seed, std::uint64_t *b) {
        check(dpfhe_relin_keygen_seeded_host(ctx_, special, plain_modulus, secret, seed.data(), b));
    }
    void generate_galois_keys_seeded(unsigned special, std::uint64_t plain_modulus, const std::uint64_t *secret, const std::vector<long> &steps,
                                     const Seed &seed, std::uint64_t *b) {
        const std::vector<std::uint64_t> elts = galois_elements(steps);
        check(dpfhe_galois_keygen_seeded_host(ctx_, special, plain_modulus, secret, elts.size(), elts.data(), seed.data(), b));
    }
    // device c0 -> device ciphertexts; host c0 -> device ciphertexts (half the bytes over the bus, synchronous)
    void expand_ciphertexts_device(unsigned level, const Seed &a_seed, std::uint64_t first_index, const std::uint64_t *c0, CiphertextBatch out,
                                   void *stream = nullptr) {
        check(dpfhe_expand_ciphertexts_level(ctx_, level, a_seed.data(), first_index, c0, out.data, out.count, stream));
    }
    void upload_seeded_ciphertexts(unsigned level, const Seed &a_seed, std::uint64_t first_index, const std::uint64_t *host_c0, CiphertextBatch out) {
        check(dpfhe_upload_seeded_ciphertexts_level(ctx_, level, a_seed.data(), first_index, host_c0, out.data, out.count));
    }
    void expand_switch_keys_device(unsigned special, const Seed &a_seed, const std::vector<std::uint64_t> &items, const std::uint64_t *b,
                                   std::uint64_t *keys, void *stream = nullptr) {
        check(dpfhe_expand_switch_keys(ctx_, special, a_seed.data(), items.size(), items.data(), b, keys, stream));
    }
    void upload_seeded_switch_keys(unsigned special, const Seed &a_seed, const std::vector<std::uint64_t> &items, const std::uint64_t *host_b,
                                   std::uint64_t *keys) {
        check(dpfhe_upload_seeded_switch_keys(ctx_, special, a_seed.data(), items.size(), items.data(), host_b, keys));
    }
    void expand_switch_keys(unsigned special, const Seed &a_seed, const std::vector<std::uint64_t> &items, const std::uint64_t *host_b,
                            std::uint64_t *host_keys) {
        check(dpfhe_expand_switch_keys_host(ctx_, special, a_seed.data(), items.size(), items.data(), host_b, host_keys));
    }

    // ---- compact ciphertexts (DESIGN.md §2.24): level-1 ciphertexts switched to 2^bits and bit-packed, [count][2][N bits / 64] words;
    //      plain_modulus = 0 for CKKS.  Decryption gives level-1 plaintexts [count][1][N] for the level-1 decoders. ----
    std::size_t compact_words(unsigned bits) const { return poly_degree() * bits / 32; }
    void compact_ciphertexts_device(unsigned level, unsigned bits, std::uint64_t plain_modulus, ConstCiphertextBatch ct, std::uint64_t *out,
                                    void *stream = nullptr) {
        check(dpfhe_compact_ciphertexts(ctx_, level, bits, plain_modulus, ct.data, out, ct.count, stream));
    }
    // device ciphertexts -> host compact words (synchronous)
    void download_compact_ciphertexts(unsigned level, unsigned bits, std::uint64_t plain_modulus, ConstCiphertextBatch ct, std::uint64_t *host_out) {
        check(dpfhe_download_compact_ciphertexts(ctx_, level, bits, plain_modulus, ct.data, host_out, ct.count));
    }
    void decrypt_compact(unsigned bits, std::uint64_t plain_modulus, const std::uint64_t *secret, const std::uint64_t *compact, std::size_t count,
                         std::uint64_t *plain_eval) {
        check(dpfhe_decrypt_compact_host(ctx_, bits, plain_modulus, secret, compact, plain_eval, count));
    }
    void decrypt_compact_device(unsigned bits, std::uint64_t plain_modulus, const std::uint64_t *secret, const std::uint64_t *compact,
                                std::size_t count, std::uint64_t *plain_eval, void *stream = nullptr) {
        check(dpfhe_decrypt_compact(ctx_, bits, plain_modulus, secret, compact, plain_eval, count, stream));
    }

    // ---- host-buffer calls: synchronous; H2D / compute / D2H are pipelined inside the library ----
    void multiply_relin(ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key, CiphertextBatch out) {
        same(a.count, b.count, out.count);
        check(dpfhe_ct_mul_relin_host(ctx_, a.data, b.data, relin_key, out.data, a.count));
    }
    void multiply_plain(ConstCiphertextBatch ct, const std::uint64_t *plain_eval, CiphertextBatch out) {
        same(ct.count, ct.count, out.count);
        check(dpfhe_ct_mul_plain_host(ctx_, ct.data, plain_eval, out.data, ct.count));
    }
    void rotate(ConstCiphertextBatch ct, long steps, const std::uint64_t *galois_key, CiphertextBatch out) {
        same(ct.count, ct.count, out.count);
        check(dpfhe_rotate_host(ctx_, ct.data, galois_element(steps), galois_key, out.data, ct.count));
    }
    // special-prime (hybrid) forms: this evaluator's last limb is the special prime; batches hold limbs()-1 limbs
    void multiply_relin_hybrid(ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key, CiphertextBatch out,
                               std::uint64_t plain_modulus = 0) {
        same(a.count, b.count, out.count);
        check(dpfhe_ct_mul_relin_hybrid_host(ctx_, a.data, b.data, relin_key, out.data, a.count, plain_modulus));
    }
    void rotate_hybrid(ConstCiphertextBatch ct, long steps, const std::uint64_t *galois_key, CiphertextBatch out,
                       std::uint64_t plain_modulus = 0) {
        same(ct.count, ct.count, out.count);
        check(dpfhe_rotate_hybrid_host(ctx_, ct.data, galois_element(steps), galois_key, out.data, ct.count, plain_modulus));
    }
    // grouped hybrid forms (digits of `special` limbs, `special` special primes at the end of the basis; dpfhe.h): batches hold
    // limbs()-special limbs, keys grouped_digits(special) digits
    unsigned grouped_digits(unsigned special) const {
        unsigned d = 0;
        check(dpfhe_grouped_digits(ctx_, special, &d));
        return d;
    }
    void multiply_relin_grouped(unsigned special, ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key, CiphertextBatch out,
                                std::uint64_t plain_modulus = 0) {
        same(a.count, b.count, out.count);
        check(dpfhe_ct_mul_relin_grouped_host(ctx_, special, a.data, b.data, relin_key, out.data, a.count, plain_modulus));
    }
    void rotate_grouped(unsigned special, ConstCiphertextBatch ct, long steps, const std::uint64_t *galois_key, CiphertextBatch out,
                        std::uint64_t plain_modulus = 0) {
        same(ct.count, ct.count, out.count);
        check(dpfhe_rotate_grouped_host(ctx_, special, ct.data, galois_element(steps), galois_key, out.data, ct.count, plain_modulus));
    }
    void multiply_relin_grouped_device(unsigned special, const std::uint64_t *a, const std::uint64_t *b, const std::uint64_t *relin_key,
                                       std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_ct_mul_relin_grouped(ctx_, special, a, b, relin_key, out, count, plain_modulus, stream));
    }
    void rotate_grouped_device(unsigned special, const std::uint64_t *ct, long steps, const std::uint64_t *galois_key, std::uint64_t *out,
                               std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_rotate_grouped(ctx_, special, ct, galois_element(steps), galois_key, out, count, plain_modulus, stream));
    }
    // out[r] = ct rotated by steps[r] with galois_keys[r], the rotations sharing the basis conversion of ct (same plaintexts as
    // rotate_grouped_device, not the same bits); out holds n_rot * count ciphertexts
    void rotate_hoisted_grouped_device(unsigned special, const std::uint64_t *ct, const std::vector<long> &steps,
                                       const std::vector<const std::uint64_t *> &galois_keys, std::uint64_t *out, std::size_t count,
                                       std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (steps.size() != galois_keys.size()) throw std::invalid_argument("one Galois key per rotation");
        std::vector<std::uint64_t> elts(steps.size());
        for (std::size_t r = 0; r < steps.size(); ++r) elts[r] = galois_element(steps[r]);
        check(dpfhe_rotate_hoisted_grouped(ctx_, special, ct, steps.size(), elts.data(), galois_keys.data(), out, count, plain_modulus, stream));
    }
    // out = ct + the sum of ct rotated by every steps[r] (1 .. 15 rotations), with one division by P for all of them (DESIGN.md §2.17);
    // out must not overlap ct
    void rotate_sum_grouped_device(unsigned special, const std::uint64_t *ct, const std::vector<long> &steps,
                                   const std::vector<const std::uint64_t *> &galois_keys, std::uint64_t *out, std::size_t count,
                                   std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (steps.size() != galois_keys.size()) throw std::invalid_argument("one Galois key per rotation");
        std::vector<std::uint64_t> elts(steps.size());
        for (std::size_t r = 0; r < steps.size(); ++r) elts[r] = galois_element(steps[r]);
        check(dpfhe_rotate_sum_grouped(ctx_, special, ct, steps.size(), elts.data(), galois_keys.data(), out, count, plain_modulus, stream));
    }
    // out = the relinearised sum of the products a[i] x b[i] (1 .. 64 pairs, DESIGN.md §2.18): the tensor products are summed
    // before ONE key switch and one division by P.  a[i] and b[i] may be the same batch, a batch may appear in several pairs; out
    // must not overlap any of them.  One pair is multiply_relin_grouped, bit for bit.  Host buffers (pipelined) need the pairs back
    // to back, so the host form takes the two operand arrays [n_terms][count] directly; the device form takes one batch per term.
    void dot_relin_grouped(unsigned special, std::size_t n_terms, const std::uint64_t *a, const std::uint64_t *b, const std::uint64_t *relin_key,
                           CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        check(dpfhe_ct_dot_grouped_host(ctx_, special, n_terms, a, b, relin_key, out.data, out.count, plain_modulus));
    }
    void dot_relin_grouped_device(unsigned special, const std::vector<const std::uint64_t *> &a, const std::vector<const std::uint64_t *> &b,
                                  const std::uint64_t *relin_key, std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0,
                                  void *stream = nullptr) {
        if (a.size() != b.size()) throw std::invalid_argument("one right operand per left operand");
        check(dpfhe_ct_dot_grouped(ctx_, special, a.size(), a.data(), b.data(), relin_key, out, count, plain_modulus, stream));
    }
    // multiply-and-rescale (DESIGN.md §2.19): multiply_relin_grouped / dot_relin_grouped followed by the rescale (BGV: modulus switch)
    // that drops the last ciphertext limb, in one division.  The inputs hold limbs()-special limbs, out limbs()-special-1.
    void multiply_relin_rescale_grouped(unsigned special, ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key,
                                        CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        same(a.count, b.count, out.count);
        check(dpfhe_ct_mul_relin_rescale_grouped_host(ctx_, special, a.data, b.data, relin_key, out.data, a.count, plain_modulus));
    }
    void multiply_relin_rescale_grouped_device(unsigned special, const std::uint64_t *a, const std::uint64_t *b, const std::uint64_t *relin_key,
                                               std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_ct_mul_relin_rescale_grouped(ctx_, special, a, b, relin_key, out, count, plain_modulus, stream));
    }
    void dot_relin_rescale_grouped(unsigned special, std::size_t n_terms, const std::uint64_t *a, const std::uint64_t *b,
                                   const std::uint64_t *relin_key, CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        check(dpfhe_ct_dot_rescale_grouped_host(ctx_, special, n_terms, a, b, relin_key, out.data, out.count, plain_modulus));
    }
    void dot_relin_rescale_grouped_device(unsigned special, const std::vector<const std::uint64_t *> &a,
                                          const std::vector<const std::uint64_t *> &b, const std::uint64_t *relin_key, std::uint64_t *out,
                                          std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (a.size() != b.size()) throw std::invalid_argument("one right operand per left operand");
        check(dpfhe_ct_dot_rescale_grouped(ctx_, special, a.size(), a.data(), b.data(), relin_key, out, count, plain_modulus, stream));
    }
    // the calls above at level `level` on this evaluator (DESIGN.md §2.20): batches hold `level` limbs (the rescale forms' out
    // level-1), the keys are this evaluator's top-level grouped keys, read in place; special <= level <= limbs()-special.  Bit for
    // bit the same call on an evaluator over the first `level` limbs and the special primes, with the key restricted to it.
    void multiply_relin_grouped_device(unsigned special, unsigned level, const std::uint64_t *a, const std::uint64_t *b,
                                       const std::uint64_t *relin_key, std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0,
                                       void *stream = nullptr) {
        check(dpfhe_ct_mul_relin_grouped_level(ctx_, special, level, a, b, relin_key, out, count, plain_modulus, stream));
    }
    void multiply_relin_rescale_grouped(unsigned special, unsigned level, ConstCiphertextBatch a, ConstCiphertextBatch b,
                                        const std::uint64_t *relin_key, CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        same(a.count, b.count, out.count);
        check(dpfhe_ct_mul_relin_rescale_grouped_level_host(ctx_, special, level, a.data, b.data, relin_key, out.data, a.count, plain_modulus));
    }
    void multiply_relin_rescale_grouped_device(unsigned special, unsigned level, const std::uint64_t *a, const std::uint64_t *b,
                                               const std::uint64_t *relin_key, std::uint64_t *out, std::size_t count,
                                               std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_ct_mul_relin_rescale_grouped_level(ctx_, special, level, a, b, relin_key, out, count, plain_modulus, stream));
    }
    void dot_relin_grouped_device(unsigned special, unsigned level, const std::vector<const std::uint64_t *> &a,
                                  const std::vector<const std::uint64_t *> &b, const std::uint64_t *relin_key, std::uint64_t *out,
                                  std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (a.size() != b.size()) throw std::invalid_argument("one right operand per left operand");
        check(dpfhe_ct_dot_grouped_level(ctx_, special, level, a.size(), a.data(), b.data(), relin_key, out, count, plain_modulus, stream));
    }
    void dot_relin_rescale_grouped(unsigned special, unsigned level, std::size_t n_terms, const std::uint64_t *a, const std::uint64_t *b,
                                   const std::uint64_t *relin_key, CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        check(dpfhe_ct_dot_rescale_grouped_level_host(ctx_, special, level, n_terms, a, b, relin_key, out.data, out.count, plain_modulus));
    }
    void dot_relin_rescale_grouped_device(unsigned special, unsigned level, const std::vector<const std::uint64_t *> &a,
                                          const std::vector<const std::uint64_t *> &b, const std::uint64_t *relin_key, std::uint64_t *out,
                                          std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (a.size() != b.size()) throw std::invalid_argument("one right operand per left operand");
        check(dpfhe_ct_dot_rescale_grouped_level(ctx_, special, level, a.size(), a.data(), b.data(), relin_key, out, count, plain_modulus, stream));
    }
    void rotate_grouped_device(unsigned special, unsigned level, const std::uint64_t *ct, long steps, const std::uint64_t *galois_key,
                               std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_rotate_grouped_level(ctx_, special, level, ct, galois_element(steps), galois_key, out, count, plain_modulus, stream));
    }
    void rotate_sum_grouped_device(unsigned special, unsigned level, const std::uint64_t *ct, const std::vector<long> &steps,
                                   const std::vector<const std::uint64_t *> &galois_keys, std::uint64_t *out, std::size_t count,
                                   std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (steps.size() != galois_keys.size()) throw std::invalid_argument("one Galois key per rotation");
        std::vector<std::uint64_t> elts(steps.size());
        for (std::size_t r = 0; r < steps.size(); ++r) elts[r] = galois_element(steps[r]);
        check(dpfhe_rotate_sum_grouped_level(ctx_, special, level, ct, steps.size(), elts.data(), galois_keys.data(), out, count, plain_modulus,
                                             stream));
    }
    // the hoisted rotations at level `level` (DESIGN.md §2.21): ct holds `level` limbs, out n_rot * count such ciphertexts
    void rotate_hoisted_grouped_device(unsigned special, unsigned level, const std::uint64_t *ct, const std::vector<long> &steps,
                                       const std::vector<const std::uint64_t *> &galois_keys, std::uint64_t *out, std::size_t count,
                                       std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        if (steps.size() != galois_keys.size()) throw std::invalid_argument("one Galois key per rotation");
        std::vector<std::uint64_t> elts(steps.size());
        for (std::size_t r = 0; r < steps.size(); ++r) elts[r] = galois_element(steps[r]);
        check(dpfhe_rotate_hoisted_grouped_level(ctx_, special, level, ct, steps.size(), elts.data(), galois_keys.data(), out, count, plain_modulus,
                                                 stream));
    }
    // divide by the product of the last `special` limbs: in holds limbs() limbs per polynomial, out limbs()-special
    void mod_down_special_device(unsigned special, const std::uint64_t *ct, std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0,
                                 void *stream = nullptr) {
        check(dpfhe_mod_down_special(ctx_, special, ct, out, 2 * count, plain_modulus, stream));
    }
    // drop the last limb: in holds limbs() limbs per polynomial, out limbs()-1
    void mod_switch_to_next(ConstCiphertextBatch in, CiphertextBatch out, std::uint64_t plain_modulus = 0) {
        same(in.count, in.count, out.count);
        check(dpfhe_mod_switch_down_host(ctx_, in.data, out.data, 2 * in.count, plain_modulus));
    }
    void transform_to_ntt(std::uint64_t *polys, std::size_t n_polys) { check(dpfhe_ntt_fwd_host(ctx_, polys, n_polys)); }
    void transform_from_ntt(std::uint64_t *polys, std::size_t n_polys) { check(dpfhe_ntt_inv_host(ctx_, polys, n_polys)); }

    // ---- device-pointer calls: asynchronous on `stream` (a cudaStream_t; nullptr = the evaluator's own) ----
    void multiply_relin_device(const std::uint64_t *a, const std::uint64_t *b, const std::uint64_t *relin_key, std::uint64_t *out,
                               std::size_t count, void *stream = nullptr) {
        check(dpfhe_ct_mul_relin(ctx_, a, b, relin_key, out, count, stream));
    }
    void multiply_plain_device(const std::uint64_t *ct, const std::uint64_t *plain_eval, std::uint64_t *out, std::size_t count,
                               void *stream = nullptr) {
        check(dpfhe_ct_mul_plain(ctx_, ct, plain_eval, out, count, stream));
    }
    void rotate_device(const std::uint64_t *ct, long steps, const std::uint64_t *galois_key, std::uint64_t *out, std::size_t count,
                       void *stream = nullptr) {
        check(dpfhe_rotate(ctx_, ct, galois_element(steps), galois_key, out, count, stream));
    }
    // several rotations of the same batch, sharing the digit decomposition; out is [steps.size()][count] ciphertexts and
    // galois_keys[r] the device pointer of the key for steps[r].  Same bits as rotate_device called steps.size() times.
    void rotate_many_device(const std::uint64_t *ct, const std::vector<long> &steps, const std::vector<const std::uint64_t *> &galois_keys,
                            std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        if (steps.size() != galois_keys.size()) throw std::runtime_error("one Galois key per rotation step");
        std::vector<std::uint64_t> elts;
        for (long k : steps) elts.push_back(galois_element(k));
        check(dpfhe_rotate_hoisted(ctx_, ct, steps.size(), elts.data(), galois_keys.data(), out, count, stream));
    }
    void add_device(const std::uint64_t *a, const std::uint64_t *b, std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        check(dpfhe_poly_add(ctx_, a, b, out, 2 * count, stream));   // a ciphertext is two polynomials
    }
    // out = (c0 + plain_eval, c1) over all limbs, plain_eval [L][N] shared by the batch: host buffers (pipelined) and device buffers
    void add_plain(ConstCiphertextBatch ct, const std::uint64_t *plain_eval, CiphertextBatch out) {
        if (ct.count != out.count) throw std::runtime_error("ciphertext batches must have the same count");
        check(dpfhe_ct_add_plain_host(ctx_, ct.data, plain_eval, out.data, ct.count));
    }
    void add_plain_device(const std::uint64_t *ct, const std::uint64_t *plain_eval, std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        check(dpfhe_ct_add_plain(ctx_, ct, plain_eval, out, count, stream));
    }
    // out = sum_i coeffs[i] cts[i] + constant (on c0), 1 .. 64 device batches of `count` ciphertexts; out may be one of them
    void lincomb_device(const std::vector<const std::uint64_t *> &cts, const std::vector<std::int64_t> &coeffs, std::int64_t constant,
                        std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        if (cts.size() != coeffs.size()) throw std::runtime_error("one coefficient per ciphertext batch");
        check(dpfhe_ct_lincomb(ctx_, cts.size(), cts.data(), coeffs.data(), constant, out, count, stream));
    }
    // the three calls above and mod_switch_to_next_device at level `level` (DESIGN.md §2.22): ciphertexts and plaintexts carry `level`
    // limbs (mod_switch_to_next_device: out level-1); 1 <= level <= limbs()
    void add_plain_device(unsigned level, const std::uint64_t *ct, const std::uint64_t *plain_eval, std::uint64_t *out, std::size_t count,
                          void *stream = nullptr) {
        check(dpfhe_ct_add_plain_level(ctx_, level, ct, plain_eval, out, count, stream));
    }
    void multiply_plain_device(unsigned level, const std::uint64_t *ct, const std::uint64_t *plain_eval, std::uint64_t *out, std::size_t count,
                               void *stream = nullptr) {
        check(dpfhe_ct_mul_plain_level(ctx_, level, ct, plain_eval, out, count, stream));
    }
    void lincomb_device(unsigned level, const std::vector<const std::uint64_t *> &cts, const std::vector<std::int64_t> &coeffs,
                        std::int64_t constant, std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        if (cts.size() != coeffs.size()) throw std::runtime_error("one coefficient per ciphertext batch");
        check(dpfhe_ct_lincomb_level(ctx_, level, cts.size(), cts.data(), coeffs.data(), constant, out, count, stream));
    }
    void mod_switch_to_next_device(unsigned level, const std::uint64_t *ct, std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0,
                                   void *stream = nullptr) {
        check(dpfhe_mod_switch_down_level(ctx_, level, ct, out, 2 * count, plain_modulus, stream));
    }
    void multiply_plain_accumulate_device(const std::uint64_t *ct, const std::uint64_t *plain_eval, std::uint64_t *acc, std::size_t count,
                                          void *stream = nullptr) {
        check(dpfhe_ct_mul_plain_acc(ctx_, ct, plain_eval, acc, count, stream));
    }
    // out[g][k] = sum_b steps[b][k] o plain[g][b]: the fused inner loop of a baby-step/giant-step matrix-vector product
    // (steps [n_steps][count] ciphertexts, plain [n_groups][n_steps] plaintexts in evaluation form, out [n_groups][count])
    void multiply_plain_inner_device(const std::uint64_t *steps, std::size_t n_steps, const std::uint64_t *plain, std::size_t n_groups,
                                     std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        check(dpfhe_ct_mul_plain_inner(ctx_, steps, n_steps, plain, n_groups, out, count, stream));
    }
    // drop the last limb of `count` ciphertexts (2*count polynomials); the result belongs to the first L-1 moduli
    void mod_switch_to_next_device(const std::uint64_t *ct, std::uint64_t *out, std::size_t count, std::uint64_t plain_modulus = 0,
                                   void *stream = nullptr) {
        check(dpfhe_mod_switch_down(ctx_, ct, out, 2 * count, plain_modulus, stream));
    }
    // hybrid (special-prime) key switching: this evaluator's last limb is the special prime, ciphertexts carry
    // limbs()-1 limbs and keys are [limbs()-1][2][limbs()][N]
    void multiply_relin_hybrid_device(const std::uint64_t *a, const std::uint64_t *b, const std::uint64_t *relin_key, std::uint64_t *out,
                                      std::size_t count, std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_ct_mul_relin_hybrid(ctx_, a, b, relin_key, out, count, plain_modulus, stream));
    }
    void rotate_hybrid_device(const std::uint64_t *ct, long steps, const std::uint64_t *galois_key, std::uint64_t *out, std::size_t count,
                              std::uint64_t plain_modulus = 0, void *stream = nullptr) {
        check(dpfhe_rotate_hybrid(ctx_, ct, galois_element(steps), galois_key, out, count, plain_modulus, stream));
    }
    void keyswitch_device(const std::uint64_t *digits, const std::uint64_t *key, std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        check(dpfhe_keyswitch(ctx_, digits, key, out, count, stream));
    }
    void transform_to_ntt_device(std::uint64_t *polys, std::size_t n_polys, void *stream = nullptr) {
        check(dpfhe_ntt_fwd(ctx_, polys, n_polys, stream));
    }
    void transform_from_ntt_device(std::uint64_t *polys, std::size_t n_polys, void *stream = nullptr) {
        check(dpfhe_ntt_inv(ctx_, polys, n_polys, stream));
    }

    // waits for every call issued through this evaluator, whatever stream it ran on
    void synchronize() { check(dpfhe_synchronize(ctx_)); }

    dpfhe_ctx *native_handle() { return ctx_; }

private:
    template <class H, void (*)(H *), int (*)(H *, const std::uint64_t *, std::uint64_t *, std::size_t, void *),
              int (*)(H *, const std::uint64_t *, std::uint64_t *, std::size_t)>
    friend class detail::ContextObject;
    static void check(int status) {
        if (status != DPFHE_OK) throw std::runtime_error(dpfhe_last_error());
    }
    static void same(std::size_t a, std::size_t b, std::size_t c) {
        if (a != b || a != c) throw std::runtime_error("ciphertext batches must have the same count");
    }
    dpfhe_ctx *ctx_ = nullptr;
    unsigned log_n_, limbs_;
};

// Encrypts under one secret with one seed, numbering the ciphertexts itself: every call continues where the previous one stopped,
// so no (seed, index) pair repeats within one Encryptor.  The secret is in host memory (Memory::host: encrypt takes host buffers) or
// in device memory (Memory::device: encrypt takes device buffers, asynchronous on `stream`).
class Encryptor {
public:
    enum class Memory { host, device };
    Encryptor(Evaluator &ev, Memory where, const std::uint64_t *secret, const Evaluator::Seed &seed, std::uint64_t plain_modulus,
              std::uint64_t first_index = 0)
        : ev_(ev), where_(where), secret_(secret), seed_(seed), t_(plain_modulus), next_(first_index) {}
    void encrypt(const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        if (where_ == Memory::host) ev_.encrypt(t_, secret_, seed_, next_, plain_eval, out);
        else ev_.encrypt_device(t_, secret_, seed_, next_, plain_eval, out, stream);
        next_ += out.count;
    }
    std::uint64_t next_index() const { return next_; }

private:
    Evaluator &ev_;
    Memory where_;
    const std::uint64_t *secret_;
    Evaluator::Seed seed_;
    std::uint64_t t_, next_;
};

// Seeded symmetric encryption at a level (DESIGN.md §2.23), numbering the ciphertexts itself as Encryptor does: it writes c0 only and
// holds the public seed (public_seed()) that a receiver needs, with next_index(), to expand them.  Host or device memory as Encryptor.
class SeededEncryptor {
public:
    using Memory = Encryptor::Memory;
    SeededEncryptor(Evaluator &ev, Memory where, unsigned level, const std::uint64_t *secret, const Evaluator::Seed &seed,
                    std::uint64_t plain_modulus, std::uint64_t first_index = 0)
        : ev_(ev), where_(where), level_(level), secret_(secret), seed_(seed), a_seed_(Evaluator::public_seed(seed)), t_(plain_modulus),
          next_(first_index) {}
    // c0 [count][level][N] of the next `count` item numbers
    void encrypt(const std::uint64_t *plain_eval, std::size_t count, std::uint64_t *c0, void *stream = nullptr) {
        if (where_ == Memory::host) ev_.encrypt_seeded(level_, t_, secret_, seed_, next_, plain_eval, count, c0);
        else ev_.encrypt_seeded_device(level_, t_, secret_, seed_, next_, plain_eval, count, c0, stream);
        next_ += count;
    }
    const Evaluator::Seed &public_seed() const { return a_seed_; }
    std::uint64_t next_index() const { return next_; }

private:
    Evaluator &ev_;
    Memory where_;
    unsigned level_;
    const std::uint64_t *secret_;
    Evaluator::Seed seed_, a_seed_;
    std::uint64_t t_, next_;
};

// Encrypts under a public key with the encrypting party's own seed, numbering the ciphertexts itself as Encryptor does.  It takes
// no secret: whoever holds the public key can encrypt, and only the key owner can decrypt.  The seed must be kept as secret as the
// plaintexts (Evaluator::random_seed() draws one).  The public key is in host memory (Memory::host) or device memory (Memory::device).
class PublicEncryptor {
public:
    using Memory = Encryptor::Memory;
    PublicEncryptor(Evaluator &ev, Memory where, const std::uint64_t *public_key, const Evaluator::Seed &seed, std::uint64_t plain_modulus,
                    std::uint64_t first_index = 0)
        : ev_(ev), where_(where), pk_(public_key), seed_(seed), t_(plain_modulus), next_(first_index) {}
    void encrypt(const std::uint64_t *plain_eval, CiphertextBatch out, void *stream = nullptr) {
        if (where_ == Memory::host) ev_.encrypt_public(t_, pk_, seed_, next_, plain_eval, out);
        else ev_.encrypt_public_device(t_, pk_, seed_, next_, plain_eval, out, stream);
        next_ += out.count;
    }
    std::uint64_t next_index() const { return next_; }

private:
    Evaluator &ev_;
    Memory where_;
    const std::uint64_t *pk_;
    Evaluator::Seed seed_;
    std::uint64_t t_, next_;
};

namespace detail {

// A non-copyable owner of the C handle H with the host-buffer and device-buffer applications.  The public classes derive from it and
// add their constructors (which fill h_) and accessors.
template <class H, void (*Destroy)(H *), int (*Apply)(H *, const std::uint64_t *, std::uint64_t *, std::size_t, void *),
          int (*ApplyHost)(H *, const std::uint64_t *, std::uint64_t *, std::size_t)>
class ContextObject {
public:
    ContextObject(const ContextObject &) = delete;
    ContextObject &operator=(const ContextObject &) = delete;
    void apply(ConstCiphertextBatch in, CiphertextBatch out) {   // host buffers, pipelined
        if (in.count != out.count) throw std::runtime_error("ciphertext batches must have the same count");
        check(ApplyHost(h_, in.data, out.data, in.count));
    }
    void apply_device(const std::uint64_t *in, std::uint64_t *out, std::size_t count, void *stream = nullptr) {
        check(Apply(h_, in, out, count, stream));
    }

protected:
    ContextObject() = default;
    ~ContextObject() { Destroy(h_); }
    static void check(int status) { Evaluator::check(status); }
    H *h_ = nullptr;
};
using LinearObject = ContextObject<dpfhe_linear, dpfhe_linear_destroy, dpfhe_linear_apply, dpfhe_linear_apply_host>;
using PolyEvalObject = ContextObject<dpfhe_polyeval, dpfhe_polyeval_destroy, dpfhe_polyeval_apply, dpfhe_polyeval_apply_host>;
using SlotSumObject = ContextObject<dpfhe_slotsum, dpfhe_slotsum_destroy, dpfhe_slotsum_apply, dpfhe_slotsum_apply_host>;

}  // namespace detail

// An encrypted linear layer y = W x (baby-step/giant-step diagonals) whose weights and Galois keys live on the device.
// diagonals: [n][L][N] plaintexts in evaluation form (diagonal g*baby + b pre-rotated by -g*baby), n a multiple of baby;
// baby_keys: [baby-1][L][2][L][N] keys of the rotations by 1 .. baby-1 slots; giant_key: [L][2][L][N], rotation by `baby`.
class LinearLayer : public detail::LinearObject {
public:
    LinearLayer(Evaluator &ev, const std::uint64_t *diagonals, std::size_t n_diagonals, std::size_t baby, const std::uint64_t *baby_keys,
                const std::uint64_t *giant_key) {
        check(dpfhe_linear_create(ev.native_handle(), diagonals, n_diagonals, baby, baby_keys, giant_key, &h_));
    }
    // with grouped special-prime keys: the evaluator's last `special` limbs are special primes, ciphertexts and diagonals carry
    // limbs()-special limbs, keys are [dnum][2][limbs()][N] (dpfhe_linear_create_grouped)
    LinearLayer(Evaluator &ev, unsigned special, const std::uint64_t *diagonals, std::size_t n_diagonals, std::size_t baby,
                const std::uint64_t *baby_keys, const std::uint64_t *giant_key, std::uint64_t plain_modulus) {
        check(dpfhe_linear_create_grouped(ev.native_handle(), special, diagonals, n_diagonals, baby, baby_keys, giant_key, plain_modulus,
                                                     &h_));
    }
    // the same layer at level `level` of the chain (DESIGN.md §2.21): ciphertexts and diagonals carry `level` limbs (a diagonal is the
    // first `level` rows of its top-level encoding), the keys are the top-level ones (dpfhe_linear_create_grouped_level)
    LinearLayer(Evaluator &ev, unsigned special, unsigned level, const std::uint64_t *diagonals, std::size_t n_diagonals, std::size_t baby,
                const std::uint64_t *baby_keys, const std::uint64_t *giant_key, std::uint64_t plain_modulus) {
        check(dpfhe_linear_create_grouped_level(ev.native_handle(), special, level, diagonals, n_diagonals, baby, baby_keys, giant_key,
                                                plain_modulus, &h_));
    }
};

// BGV polynomial evaluation on encrypted slots down the modulus chain (dpfhe_polyeval_*): p(x) = sum_k coeffs[k] x^k mod
// plain_modulus, slot by slot.  The evaluator's last `special` limbs are special primes; relin_key is the grouped relinearisation key
// [dnum][2][limbs()][N] of the top level (host memory).  Inputs carry limbs()-special limbs, results result_limbs().
class PolyEval : public detail::PolyEvalObject {
public:
    PolyEval(Evaluator &ev, unsigned special, std::uint64_t plain_modulus, const std::vector<std::int64_t> &coeffs, const std::uint64_t *relin_key) {
        if (coeffs.size() < 2) throw std::runtime_error("a polynomial of degree at least 1");
        check(dpfhe_polyeval_create_grouped(ev.native_handle(), special, plain_modulus, coeffs.data(), coeffs.size() - 1, relin_key, &h_));
    }
    // the evaluator at level `level` of the chain (DESIGN.md §2.22): inputs carry `level` limbs, the key is the top-level one
    PolyEval(Evaluator &ev, unsigned special, unsigned level, std::uint64_t plain_modulus, const std::vector<std::int64_t> &coeffs,
             const std::uint64_t *relin_key) {
        if (coeffs.size() < 2) throw std::runtime_error("a polynomial of degree at least 1");
        check(dpfhe_polyeval_create_grouped_level(ev.native_handle(), special, level, plain_modulus, coeffs.data(), coeffs.size() - 1, relin_key,
                                                  &h_));
    }
    unsigned result_limbs() const { return dpfhe_polyeval_result_limbs(h_); }
};

// Slot sums (dpfhe_slotsum_*, DESIGN.md §2.17): slot i of the result is sum_{j < prod(radices)} x[(i + j * stride) mod N/2] in every
// row.  galois_keys: the grouped Galois keys of the rotations by SlotSum::steps(stride, radices), in that order, back to back in host
// memory (what Evaluator::generate_galois_keys writes); plain_modulus 0 for CKKS.
class SlotSum : public detail::SlotSumObject {
public:
    SlotSum(Evaluator &ev, unsigned special, std::size_t stride, const std::vector<unsigned> &radices, const std::uint64_t *galois_keys,
            std::uint64_t plain_modulus = 0) {
        check(dpfhe_slotsum_create_grouped(ev.native_handle(), special, stride, radices.data(), radices.size(), galois_keys, plain_modulus,
                                                      &h_));
    }
    // the slot sum at level `level` of the chain (DESIGN.md §2.21): ciphertexts carry `level` limbs, the keys are the top-level ones
    SlotSum(Evaluator &ev, unsigned special, unsigned level, std::size_t stride, const std::vector<unsigned> &radices,
            const std::uint64_t *galois_keys, std::uint64_t plain_modulus = 0) {
        check(dpfhe_slotsum_create_grouped_level(ev.native_handle(), special, level, stride, radices.data(), radices.size(), galois_keys,
                                                 plain_modulus, &h_));
    }
    // the rotation steps, stage by stage and ascending within a stage: the order of the keys
    static std::vector<long> steps(std::size_t stride, const std::vector<unsigned> &radices) {
        std::size_t n = 0;
        check(dpfhe_slotsum_steps(stride, radices.data(), radices.size(), nullptr, &n));
        std::vector<int> s(n);
        check(dpfhe_slotsum_steps(stride, radices.data(), radices.size(), s.data(), &n));
        return std::vector<long>(s.begin(), s.end());
    }
};

// CKKS polynomial evaluation on encrypted slots down the rescaling chain (dpfhe_polyeval_create_ckks, DESIGN.md §2.16): p(z) = sum_k
// coeffs[k] z^k with real coefficients, slot by slot.  Inputs at scale scale_in carry limbs()-special limbs; results carry
// result_limbs() limbs at result_scale() (scale_out, or scale_in when scale_out is 0).  relin_key: the grouped relinearisation key
// of the top level generated with plain modulus 0 (host memory).
class CkksPolyEval : public detail::PolyEvalObject {
public:
    CkksPolyEval(Evaluator &ev, unsigned special, const std::vector<double> &coeffs, double scale_in, const std::uint64_t *relin_key,
                 double scale_out = 0) {
        if (coeffs.size() < 2) throw std::runtime_error("a polynomial of degree at least 1");
        check(dpfhe_polyeval_create_ckks(ev.native_handle(), special, coeffs.data(), coeffs.size() - 1, scale_in,
                                                    scale_out == 0 ? scale_in : scale_out, relin_key, &h_));
    }
    // the evaluator at level `level` of the chain (DESIGN.md §2.22): inputs carry `level` limbs, the key is the top-level one
    CkksPolyEval(Evaluator &ev, unsigned special, unsigned level, const std::vector<double> &coeffs, double scale_in, const std::uint64_t *relin_key,
                 double scale_out = 0) {
        if (coeffs.size() < 2) throw std::runtime_error("a polynomial of degree at least 1");
        check(dpfhe_polyeval_create_ckks_level(ev.native_handle(), special, level, coeffs.data(), coeffs.size() - 1, scale_in,
                                               scale_out == 0 ? scale_in : scale_out, relin_key, &h_));
    }
    unsigned result_limbs() const { return dpfhe_polyeval_result_limbs(h_); }
    double result_scale() const { return dpfhe_polyeval_result_scale(h_); }
};

// Several GPUs behind one object (dpfhe_multi_*): contiguous shards of every batch, one context and host thread per device, no
// collective.  The reference's distributed layer is one MPI rank per GPU (src/core/distributed/distributed_context.cpp:242-250).
class MultiEvaluator {
public:
    // devices empty = every visible GPU
    explicit MultiEvaluator(const EncryptionParameters &parms, const std::vector<int> &devices = {}) : log_n_(parms.log_n), limbs_(parms.n_limbs) {
        dpfhe_params p;
        p.log_n = parms.log_n;
        p.n_limbs = parms.n_limbs;
        p.moduli = parms.moduli.empty() ? nullptr : parms.moduli.data();
        check(dpfhe_multi_create(&p, devices.empty() ? nullptr : devices.data(), (int)devices.size(), &m_));
    }
    ~MultiEvaluator() { dpfhe_multi_destroy(m_); }
    MultiEvaluator(const MultiEvaluator &) = delete;
    MultiEvaluator &operator=(const MultiEvaluator &) = delete;
    int device_count() const { return dpfhe_multi_device_count(m_); }
    std::size_t poly_degree() const { return std::size_t(1) << log_n_; }
    unsigned limbs() const { return limbs_; }
    std::uint64_t modulus(unsigned limb) const {
        std::uint64_t q = 0;
        check(dpfhe_get_modulus(dpfhe_multi_context(m_, 0), limb, &q));
        return q;
    }
    // host buffers: every device pipelines its own shard; the result needs no gather
    void multiply_relin(ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key, CiphertextBatch out) {
        if (a.count != b.count || a.count != out.count) throw std::runtime_error("ciphertext batches must have the same count");
        check(dpfhe_multi_ct_mul_relin_host(m_, a.data, b.data, relin_key, out.data, a.count));
    }
    // the same with a special-prime relinearisation key (digits of `special` limbs, `special` special primes; batches hold
    // limbs() - special limbs)
    void multiply_relin_grouped(unsigned special, ConstCiphertextBatch a, ConstCiphertextBatch b, const std::uint64_t *relin_key, CiphertextBatch out,
                                std::uint64_t plain_modulus = 0) {
        if (a.count != b.count || a.count != out.count) throw std::runtime_error("ciphertext batches must have the same count");
        check(dpfhe_multi_ct_mul_relin_grouped_host(m_, special, a.data, b.data, relin_key, out.data, a.count, plain_modulus));
    }
    // device buffers: a[r], b[r], relin_key[r] on device r (shard r of the batch); the whole result on device `root`
    void multiply_relin_gather_device(const std::vector<const std::uint64_t *> &a, const std::vector<const std::uint64_t *> &b,
                                      const std::vector<const std::uint64_t *> &relin_key, std::uint64_t *out_on_root, int root, std::size_t count) {
        if ((int)a.size() != device_count() || a.size() != b.size() || a.size() != relin_key.size())
            throw std::runtime_error("one operand pointer per device");
        check(dpfhe_multi_ct_mul_relin_gather(m_, a.data(), b.data(), relin_key.data(), out_on_root, root, count));
    }
    dpfhe_multi *native_handle() { return m_; }

private:
    static void check(int status) {
        if (status != DPFHE_OK) throw std::runtime_error(dpfhe_last_error());
    }
    dpfhe_multi *m_ = nullptr;
    unsigned log_n_, limbs_;
};

}  // namespace fhe
}  // namespace api
}  // namespace deeppowers
