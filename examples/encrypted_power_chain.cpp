// encrypted_power_chain.cpp — x^8 on CKKS slots by three squarings down the modulus chain, on ONE evaluator with ONE relinearisation
// key: each multiply_relin_rescale_grouped call takes the level of its operands and reads the top-level key in place (DESIGN.md §2.20),
// so no evaluator and no restricted key is made per level.  Only the decryption uses an evaluator over the result's limbs.
#include <deeppowers_fhe.hpp>

#include <cmath>
#include <complex>
#include <cstdint>
#include <iostream>
#include <random>
#include <vector>

using namespace deeppowers::api::fhe;

int main() {
    try {
        const unsigned Lq = 5, K = 2;   // 5 ciphertext moduli + 2 special primes, N = 8192: three rescales leave q_0, q_1
        const std::size_t B = 4;        // ciphertexts
        EncryptionParameters parms;     // the default basis: primes k 2^32 + 1 just below 2^60
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);
        const std::size_t n = ev.poly_degree(), half = n / 2;
        auto prefix = [&](unsigned limbs) {   // an evaluator over the first `limbs` ciphertext moduli (encryption and decryption only)
            EncryptionParameters pp = parms;
            pp.n_limbs = limbs;
            for (unsigned i = 0; i < limbs; ++i) pp.moduli.push_back(ev.modulus(i));
            return pp;
        };
        Evaluator evq(prefix(Lq));
        // a scale near the primes keeps every square's scale near them: s' = s^2 / q_{l-1}
        double scale = (double)ev.modulus(1);

        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, 0, secret.data(), seed, relin.data());

        std::mt19937_64 rng(8);
        std::uniform_real_distribution<double> uni(-1.0, 1.0);
        std::vector<std::complex<double>> z(B * half);
        for (auto &v : z) v = uni(rng);
        std::vector<std::uint64_t> plain(B * evq.poly_words()), ct(B * evq.ciphertext_words());
        evq.encode_ckks(z.data(), B, scale, plain.data());
        evq.encrypt(0, secret.data(), seed, 0, plain.data(), CiphertextBatch{ct.data(), B});

        // x -> x^2 -> x^4 -> x^8 at levels Lq, Lq - 1, Lq - 2, every call with the same top-level key
        for (unsigned level = Lq; level > Lq - 3; --level) {
            std::vector<std::uint64_t> sq(B * 2 * (level - 1) * n);
            ev.multiply_relin_rescale_grouped(K, level, ConstCiphertextBatch(ct.data(), B), ConstCiphertextBatch(ct.data(), B), relin.data(),
                                              CiphertextBatch{sq.data(), B});
            ct.swap(sq);
            scale = scale * scale / (double)ev.modulus(level - 1);
        }

        const unsigned Lf = Lq - 3;
        Evaluator evf(prefix(Lf));
        std::vector<std::uint64_t> phase(B * evf.poly_words());
        evf.decrypt(secret.data(), ConstCiphertextBatch(ct.data(), B), phase.data());
        std::vector<std::complex<double>> y(B * half);
        evf.decode_ckks(phase.data(), B, scale, y.data());

        double worst = 0;
        for (std::size_t i = 0; i < B * half; ++i) worst = std::max(worst, std::abs(y[i] - std::pow(z[i], 8)));
        std::cout << B * half << " eighth powers at " << Lf << " limbs, one evaluator and one key, scale 2^" << std::log2(scale)
                  << ", largest error " << worst << std::endl;
        return worst < 1e-6 ? 0 : 2;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
