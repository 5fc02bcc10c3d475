// encrypted_two_layer_mlp.cpp — two encrypted layers with nothing but libdpfhe.so, on ONE evaluator with ONE set of top-level keys:
// y = W2 p(W1 x + b1) slot by slot.  W1 runs at the top level, PolyEval takes the result down to Lf limbs, and W2 runs at level Lf
// on the same evaluator (LinearLayer's level constructor, DESIGN.md §2.21), reading the same top-level Galois keys: no second
// evaluator for the lower level and no restricted keys.  The result is decrypted, decoded and checked against the same computation
// mod t.
#include <deeppowers_fhe.hpp>

#include <algorithm>
#include <cstdint>
#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        const unsigned Lq = 4, K = 2;                   // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t DIM = 32, BABY = 8, B = 4;    // two 32 x 32 layers, 8 baby steps, 4 input vectors
        const std::uint64_t t = 65537;                  // prime, 1 mod 2N
        const std::vector<std::int64_t> p = {3, -2, 1}; // the activation: 3 - 2x + x^2
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);                            // every key switch, at every level
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
        ev.generate_galois_keys(K, t, secret.data(), steps, seed, galois.data());   // one set for both layers

        std::mt19937_64 rng(11);
        auto small = [&](int r) { return (std::int64_t)(rng() % (2 * r + 1)) - r; };
        std::vector<std::int64_t> W1(DIM * DIM), W2(DIM * DIM), X(B * DIM), bias(DIM);
        for (auto &v : W1) v = small(8);
        for (auto &v : W2) v = small(8);
        for (auto &v : X) v = small(8);
        for (auto &v : bias) v = small(50);

        // The diagonals of an M x M matrix: diagonal d holds W[i][(i + d) % M] in slots i of the first row, rotated right by
        // (d / BABY) * BABY slots; the input repeats its M slots at M .. 2M - 1.  Layer 1 is the 2 DIM x 2 DIM matrix [W1 0; W1 0]
        // on [x, 0], so that its result repeats W1 x at DIM .. 2 DIM - 1: the layout layer 2 reads.
        auto diagonals = [&](const std::vector<std::int64_t> &W, std::size_t M) {
            std::vector<std::int64_t> s(M * n, 0);
            for (std::size_t d = 0; d < M; ++d)
                for (std::size_t i = 0; i < M; ++i) s[d * n + (i + (d / BABY) * BABY) % half] = W[i * M + (i + d) % M];
            return s;
        };
        std::vector<std::int64_t> W1e(4 * DIM * DIM, 0);
        for (std::size_t i = 0; i < 2 * DIM; ++i)
            for (std::size_t j = 0; j < DIM; ++j) W1e[i * 2 * DIM + j] = W1[(i % DIM) * DIM + j];
        const std::vector<std::int64_t> d1 = diagonals(W1e, 2 * DIM), d2 = diagonals(W2, DIM);
        std::vector<std::int64_t> x_slots(B * n, 0), b_slots(n, 0);
        for (std::size_t k = 0; k < B; ++k)
            for (std::size_t i = 0; i < DIM; ++i) x_slots[k * n + i] = x_slots[k * n + 2 * DIM + i] = X[k * DIM + i];
        for (std::size_t i = 0; i < DIM; ++i) b_slots[i] = b_slots[DIM + i] = bias[i];
        std::vector<std::uint64_t> diags1(2 * DIM * evq.poly_words()), diags2(DIM * evq.poly_words()), xpt(B * evq.poly_words()), bpt(evq.poly_words());
        evq.encode_bgv(d1.data(), 2 * DIM, t, diags1.data());
        evq.encode_bgv(d2.data(), DIM, t, diags2.data());
        evq.encode_bgv(x_slots.data(), B, t, xpt.data());
        evq.encode_bgv(b_slots.data(), 1, t, bpt.data());

        std::vector<std::uint64_t> ct(B * evq.ciphertext_words()), y(ct.size());
        Encryptor enc(evq, Encryptor::Memory::host, secret.data(), seed, t);   // the secret's first Lq rows
        enc.encrypt(xpt.data(), CiphertextBatch{ct.data(), B});

        const std::uint64_t *giant_key = galois.data() + (BABY - 1) * ev.key_words(K);
        LinearLayer layer1(ev, K, diags1.data(), 2 * DIM, BABY, galois.data(), giant_key, t);
        layer1.apply(ConstCiphertextBatch(ct.data(), B), CiphertextBatch{y.data(), B});               // W1 x
        evq.add_plain(ConstCiphertextBatch(y.data(), B), bpt.data(), CiphertextBatch{y.data(), B});   // + b1
        PolyEval act(ev, K, t, p, relin.data());
        const unsigned Lf = act.result_limbs();
        std::vector<std::uint64_t> z(B * 2 * Lf * n), w(z.size());
        act.apply(ConstCiphertextBatch(y.data(), B), CiphertextBatch{z.data(), B});                    // p(W1 x + b1), Lf limbs

        // layer 2 at level Lf on the same evaluator and keys; a diagonal at Lf is the first Lf rows of its top-level encoding
        std::vector<std::uint64_t> diags2_lf(DIM * Lf * n);
        for (std::size_t d = 0; d < DIM; ++d)
            std::copy(diags2.begin() + d * Lq * n, diags2.begin() + (d * Lq + Lf) * n, diags2_lf.begin() + d * Lf * n);
        LinearLayer layer2(ev, K, Lf, diags2_lf.data(), DIM, BABY, galois.data(), giant_key, t);
        layer2.apply(ConstCiphertextBatch(z.data(), B), CiphertextBatch{w.data(), B});                 // W2 p(W1 x + b1)

        EncryptionParameters pf = pq;
        pf.n_limbs = Lf;
        pf.moduli.resize(Lf);
        Evaluator evf(pf);                              // the result's moduli: decryption and decoding only
        std::vector<std::uint64_t> phase(B * evf.poly_words()), out(B * n);
        evf.decrypt(secret.data(), ConstCiphertextBatch(w.data(), B), phase.data());
        evf.decode_bgv(phase.data(), B, t, out.data());

        const std::int64_t T = (std::int64_t)t;
        auto mod = [&](std::int64_t v) { return ((v % T) + T) % T; };
        std::size_t wrong = 0;
        for (std::size_t k = 0; k < B; ++k) {
            std::vector<std::int64_t> h(DIM);
            for (std::size_t i = 0; i < DIM; ++i) {
                std::int64_t v = bias[i];
                for (std::size_t j = 0; j < DIM; ++j) v += W1[i * DIM + j] * X[k * DIM + j];
                std::int64_t r = 0;
                for (std::size_t c = p.size(); c-- > 0;) r = mod(r * mod(v) + p[c]);
                h[i] = r;
            }
            for (std::size_t i = 0; i < DIM; ++i) {
                std::int64_t v = 0;
                for (std::size_t j = 0; j < DIM; ++j) v = mod(v + mod(W2[i * DIM + j] * h[j]));
                if (out[k * n + i] != (std::uint64_t)v) ++wrong;
            }
        }
        std::cout << B * DIM << " outputs of two layers at " << Lf << " limbs, one evaluator and one key set, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
