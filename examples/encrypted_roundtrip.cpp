// encrypted_roundtrip.cpp — one honest BGV round trip with nothing but libdpfhe.so: integer slots -> plaintexts -> ciphertexts
// under a secret generated on the device -> ct x ct with a device-generated relinearisation key -> decryption -> slots, checked
// against the slot-wise products mod t.
#include <deeppowers_fhe.hpp>

#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        EncryptionParameters parms;   // N = 8192, the four largest default moduli
        Evaluator ev(parms);
        const std::uint64_t t = 65537;   // prime, 1 mod 2N
        const std::size_t n = ev.poly_degree(), P = ev.poly_words();
        const Evaluator::Seed seed = Evaluator::random_seed();   // the storage form of the secret

        std::vector<std::uint64_t> secret(P), relin(ev.key_words(0));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(0, t, secret.data(), seed, relin.data());

        std::mt19937_64 rng(1);
        std::vector<std::int64_t> slots(2 * n);   // two vectors of N slots
        for (auto &v : slots) v = (std::int64_t)(rng() % t);
        std::vector<std::uint64_t> plain(2 * P), ct(2 * ev.ciphertext_words()), prod(ev.ciphertext_words()), phase(P), out(n);
        ev.encode_bgv(slots.data(), 2, t, plain.data());
        Encryptor enc(ev, Encryptor::Memory::host, secret.data(), seed, t);
        enc.encrypt(plain.data(), CiphertextBatch{ct.data(), 2});
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
