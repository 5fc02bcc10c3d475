// encrypted_public.cpp — public-key encryption with nothing but libdpfhe.so.  A key owner makes the secret, the public key and a
// relinearisation key; a data owner, with a seed of its own and no access to the secret, encrypts BGV slots under the public key;
// the product of the two ciphertexts is computed; the key owner decrypts it and checks the slot-wise products mod t.
#include <deeppowers_fhe.hpp>

#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

namespace {

// the data owner: holds the public key and its own seed, never the secret
std::vector<std::uint64_t> encrypt_as_data_owner(Evaluator &ev, const std::vector<std::uint64_t> &public_key, std::uint64_t t,
                                                 const std::vector<std::int64_t> &slots, std::size_t count) {
    std::vector<std::uint64_t> plain(count * ev.poly_words()), ct(count * ev.ciphertext_words());
    ev.encode_bgv(slots.data(), count, t, plain.data());
    PublicEncryptor enc(ev, PublicEncryptor::Memory::host, public_key.data(), Evaluator::random_seed(), t);
    enc.encrypt(plain.data(), CiphertextBatch{ct.data(), count});
    return ct;
}

}  // namespace

int main() {
    try {
        EncryptionParameters parms;   // N = 8192, the four largest default moduli
        Evaluator ev(parms);
        const std::uint64_t t = 65537;   // prime, 1 mod 2N
        const std::size_t n = ev.poly_degree(), P = ev.poly_words();

        // the key owner
        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(P), public_key(ev.public_key_words()), relin(ev.key_words(0));
        ev.generate_secret(seed, secret.data());
        ev.generate_public_key(t, secret.data(), seed, public_key.data());
        ev.generate_relin_key(0, t, secret.data(), seed, relin.data());

        std::mt19937_64 rng(2);
        std::vector<std::int64_t> slots(2 * n);   // two vectors of N slots
        for (auto &v : slots) v = (std::int64_t)(rng() % t);
        const std::vector<std::uint64_t> ct = encrypt_as_data_owner(ev, public_key, t, slots, 2);

        std::vector<std::uint64_t> prod(ev.ciphertext_words()), phase(P), out(n);
        ev.multiply_relin(ConstCiphertextBatch(ct.data(), 1), ConstCiphertextBatch(ct.data() + ev.ciphertext_words(), 1), relin.data(),
                          CiphertextBatch{prod.data(), 1});
        ev.decrypt(secret.data(), ConstCiphertextBatch(prod.data(), 1), phase.data());
        ev.decode_bgv(phase.data(), 1, t, out.data());

        std::size_t wrong = 0;
        for (std::size_t i = 0; i < n; ++i)
            if (out[i] != (std::uint64_t)slots[i] * (std::uint64_t)slots[n + i] % t) ++wrong;
        std::cout << n << " slot products, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
