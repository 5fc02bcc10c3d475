// encrypted_mlp.cpp — one encrypted MLP block with nothing but libdpfhe.so: y = p(W x + b) slot by slot, where W x is the
// baby-step/giant-step linear layer with grouped special-prime keys, b an encoded bias added with add_plain, and p a BGV polynomial
// evaluated down the modulus chain (PolyEval); the result is decrypted, decoded and checked against the same computation mod t.
#include <deeppowers_fhe.hpp>

#include <cstdint>
#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        const unsigned Lq = 4, K = 2;                   // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t DIM = 64, BABY = 8, B = 4;    // a 64 x 64 layer, 8 baby steps, 4 input vectors
        const std::uint64_t t = 65537;                  // prime, 1 mod 2N
        const std::vector<std::int64_t> p = {3, -2, 1}; // the activation: 3 - 2x + x^2
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);                            // key switching: ciphertext moduli + special primes
        const std::size_t n = ev.poly_degree(), half = n / 2;
        EncryptionParameters pq = parms;
        pq.n_limbs = Lq;
        for (unsigned i = 0; i < Lq; ++i) pq.moduli.push_back(ev.modulus(i));
        Evaluator evq(pq);                              // the ciphertext moduli: encoding, encryption, the bias

        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K)), galois(BABY * ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, t, secret.data(), seed, relin.data());
        std::vector<long> steps;
        for (std::size_t b = 1; b <= BABY; ++b) steps.push_back((long)b);
        ev.generate_galois_keys(K, t, secret.data(), steps, seed, galois.data());

        std::mt19937_64 rng(7);
        auto small = [&](int r) { return (std::int64_t)(rng() % (2 * r + 1)) - r; };
        std::vector<std::int64_t> W(DIM * DIM), X(B * DIM), bias(DIM);
        for (auto &v : W) v = small(8);
        for (auto &v : X) v = small(8);
        for (auto &v : bias) v = small(50);

        // diagonal d = g * BABY + b holds W[i][(i + d) % DIM] in slots i of the first row, rotated right by g * BABY slots
        std::vector<std::int64_t> diag_slots(DIM * n, 0), x_slots(B * n, 0), b_slots(n, 0);
        for (std::size_t d = 0; d < DIM; ++d)
            for (std::size_t i = 0; i < DIM; ++i) diag_slots[d * n + (i + (d / BABY) * BABY) % half] = W[i * DIM + (i + d) % DIM];
        for (std::size_t k = 0; k < B; ++k)
            for (std::size_t i = 0; i < DIM; ++i) x_slots[k * n + i] = x_slots[k * n + DIM + i] = X[k * DIM + i];
        for (std::size_t i = 0; i < DIM; ++i) b_slots[i] = bias[i];
        std::vector<std::uint64_t> diags(DIM * evq.poly_words()), xpt(B * evq.poly_words()), bpt(evq.poly_words());
        evq.encode_bgv(diag_slots.data(), DIM, t, diags.data());
        evq.encode_bgv(x_slots.data(), B, t, xpt.data());
        evq.encode_bgv(b_slots.data(), 1, t, bpt.data());

        std::vector<std::uint64_t> ct(B * evq.ciphertext_words()), y(ct.size());
        Encryptor enc(evq, Encryptor::Memory::host, secret.data(), seed, t);   // the secret's first Lq rows
        enc.encrypt(xpt.data(), CiphertextBatch{ct.data(), B});

        LinearLayer layer(ev, K, diags.data(), DIM, BABY, galois.data(), galois.data() + (BABY - 1) * ev.key_words(K), t);
        layer.apply(ConstCiphertextBatch(ct.data(), B), CiphertextBatch{y.data(), B});                 // W x
        evq.add_plain(ConstCiphertextBatch(y.data(), B), bpt.data(), CiphertextBatch{y.data(), B});    // + b
        PolyEval act(ev, K, t, p, relin.data());
        const unsigned Lf = act.result_limbs();
        std::vector<std::uint64_t> z(B * 2 * Lf * n);
        act.apply(ConstCiphertextBatch(y.data(), B), CiphertextBatch{z.data(), B});                     // p(W x + b)

        EncryptionParameters pf = pq;
        pf.n_limbs = Lf;
        pf.moduli.resize(Lf);
        Evaluator evf(pf);                              // the result's moduli
        std::vector<std::uint64_t> phase(B * evf.poly_words()), out(B * n);
        evf.decrypt(secret.data(), ConstCiphertextBatch(z.data(), B), phase.data());
        evf.decode_bgv(phase.data(), B, t, out.data());

        std::size_t wrong = 0;
        for (std::size_t k = 0; k < B; ++k)
            for (std::size_t i = 0; i < DIM; ++i) {
                std::int64_t v = bias[i];
                for (std::size_t j = 0; j < DIM; ++j) v += W[i * DIM + j] * X[k * DIM + j];
                const std::int64_t x = ((v % (std::int64_t)t) + (std::int64_t)t) % (std::int64_t)t;
                std::int64_t r = 0;
                for (std::size_t c = p.size(); c-- > 0;) r = ((r * x + p[c]) % (std::int64_t)t + (std::int64_t)t) % (std::int64_t)t;
                if (out[k * n + i] != (std::uint64_t)r) ++wrong;
            }
        std::cout << B * DIM << " activations at " << Lf << " limbs, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
