// encrypted_dot_product.cpp — attention scores in column packing with nothing but libdpfhe.so: 8192 query / key pairs of dimension 64,
// one ciphertext per component (ciphertext Q_d holds component d of every query in its 8192 slots, K_d that of every key), so the
// scores q . k = sum_d Q_d K_d are one inner product of 64 pairs of ciphertexts: dot_relin_grouped sums the 64 tensor products and
// relinearises once.  After decryption and decoding every slot holds its score exactly; the program returns 0 only then.
#include <deeppowers_fhe.hpp>

#include <cstdint>
#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        const unsigned Lq = 4, K = 2;        // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t D = 64;            // head dimension: 64 pairs of ciphertexts
        const std::uint64_t t = 167772161;   // prime, 1 mod 2N; 64 * 128 * 128 < t / 2
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);                 // key switching: ciphertext moduli + special primes
        const std::size_t n = ev.poly_degree();
        EncryptionParameters pq = parms;
        pq.n_limbs = Lq;
        for (unsigned i = 0; i < Lq; ++i) pq.moduli.push_back(ev.modulus(i));
        Evaluator evq(pq);                   // the ciphertext moduli: encoding, encryption, decryption

        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, t, secret.data(), seed, relin.data());

        std::mt19937_64 rng(64);
        std::vector<std::int64_t> slots(2 * D * n);   // Q_0 .. Q_63, then K_0 .. K_63: slot i of Q_d is component d of query i
        for (auto &v : slots) v = (std::int64_t)(rng() % 256) - 128;
        std::vector<std::uint64_t> pt(2 * D * evq.poly_words());
        evq.encode_bgv(slots.data(), 2 * D, t, pt.data());
        const std::size_t ctw = evq.ciphertext_words();
        std::vector<std::uint64_t> ct(2 * D * ctw), score(ctw);
        Encryptor enc(evq, Encryptor::Memory::host, secret.data(), seed, t);   // the secret's first Lq rows
        enc.encrypt(pt.data(), CiphertextBatch{ct.data(), 2 * D});

        // operands [n_terms][count = 1]: the 64 Q_d back to back, and the 64 K_d
        ev.dot_relin_grouped(K, D, ct.data(), ct.data() + D * ctw, relin.data(), CiphertextBatch{score.data(), 1}, t);

        std::vector<std::uint64_t> phase(evq.poly_words()), out(n);
        evq.decrypt(secret.data(), ConstCiphertextBatch(score.data(), 1), phase.data());
        evq.decode_bgv(phase.data(), 1, t, out.data());
        std::size_t wrong = 0;
        for (std::size_t i = 0; i < n; ++i) {
            std::int64_t want = 0;
            for (std::size_t d = 0; d < D; ++d) want += slots[d * n + i] * slots[(D + d) * n + i];
            std::int64_t got = (std::int64_t)out[i];
            if (got > (std::int64_t)(t / 2)) got -= (std::int64_t)t;
            if (got != want) ++wrong;
        }
        std::cout << n << " attention scores of dimension " << D << ", " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
