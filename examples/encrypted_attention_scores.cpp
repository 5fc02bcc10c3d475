// encrypted_attention_scores.cpp — attention scores q_h . k_h on encrypted data with nothing but libdpfhe.so: 64 query and 64 key
// vectors of int8, dimension 64, packed into one row of one ciphertext each (slot 64 h + d holds component d of vector h), multiplied
// slot by slot (multiply_relin_grouped) and summed over each head dimension with a SlotSum of stride 1 and radices {4, 4, 4}.  After
// decryption and decoding, slot 64 h holds q_h . k_h exactly; the program returns 0 only if every score is right.
#include <deeppowers_fhe.hpp>

#include <cstdint>
#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        const unsigned Lq = 4, K = 2;                    // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t H = 64, D = 64;                // 64 vectors of dimension 64: the N/2 = 4096 slots of one row
        const std::uint64_t t = 167772161;               // prime, 1 mod 2N
        const std::vector<unsigned> radices = {4, 4, 4}; // 64 slots in three summed-rotation stages
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);                             // key switching: ciphertext moduli + special primes
        const std::size_t n = ev.poly_degree();
        EncryptionParameters pq = parms;
        pq.n_limbs = Lq;
        for (unsigned i = 0; i < Lq; ++i) pq.moduli.push_back(ev.modulus(i));
        Evaluator evq(pq);                               // the ciphertext moduli: encoding, encryption, decryption

        const Evaluator::Seed seed = Evaluator::random_seed();
        const std::vector<long> steps = SlotSum::steps(1, radices);
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K)), galois(steps.size() * ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, t, secret.data(), seed, relin.data());
        ev.generate_galois_keys(K, t, secret.data(), steps, seed, galois.data());

        std::mt19937_64 rng(64);
        std::vector<std::int64_t> q(H * D), k(H * D);
        for (auto &v : q) v = (std::int64_t)(rng() % 256) - 128;
        for (auto &v : k) v = (std::int64_t)(rng() % 256) - 128;
        std::vector<std::int64_t> slots(2 * n, 0);       // two plaintexts: queries, keys (first row of each)
        for (std::size_t i = 0; i < H * D; ++i) {
            slots[i] = q[i];
            slots[n + i] = k[i];
        }
        std::vector<std::uint64_t> pt(2 * evq.poly_words());
        evq.encode_bgv(slots.data(), 2, t, pt.data());
        std::vector<std::uint64_t> ct(2 * evq.ciphertext_words()), prod(evq.ciphertext_words()), score(evq.ciphertext_words());
        Encryptor enc(evq, Encryptor::Memory::host, secret.data(), seed, t);   // the secret's first Lq rows
        enc.encrypt(pt.data(), CiphertextBatch{ct.data(), 2});

        ev.multiply_relin_grouped(K, ConstCiphertextBatch(ct.data(), 1), ConstCiphertextBatch(ct.data() + evq.ciphertext_words(), 1), relin.data(),
                                  CiphertextBatch{prod.data(), 1}, t);                                  // q_h[d] k_h[d] in slot 64 h + d
        SlotSum sum(ev, K, 1, radices, galois.data(), t);
        sum.apply(ConstCiphertextBatch(prod.data(), 1), CiphertextBatch{score.data(), 1});              // sum over d into slot 64 h

        std::vector<std::uint64_t> phase(evq.poly_words()), out(n);
        evq.decrypt(secret.data(), ConstCiphertextBatch(score.data(), 1), phase.data());
        evq.decode_bgv(phase.data(), 1, t, out.data());
        std::size_t wrong = 0;
        for (std::size_t h = 0; h < H; ++h) {
            std::int64_t want = 0;
            for (std::size_t d = 0; d < D; ++d) want += q[h * D + d] * k[h * D + d];
            std::int64_t got = (std::int64_t)out[h * D];
            if (got > (std::int64_t)(t / 2)) got -= (std::int64_t)t;
            if (got != want) ++wrong;
        }
        std::cout << H << " attention scores, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
