// encrypted_ckks_activation.cpp — a real-valued activation on CKKS slots with nothing but libdpfhe.so: keys from a seed (plain
// modulus 0), slots in [-1, 1] encoded and encrypted, a degree-7 least-squares fit of GELU on [-1, 1] evaluated down the rescaling
// chain (CkksPolyEval), then decryption, decoding at result_scale() and the largest error against the same polynomial in double.
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
        const unsigned Lq = 5, K = 2;   // 5 ciphertext moduli + 2 special primes, N = 8192: degree 7 needs 3 levels, the result keeps q_0
        const std::size_t B = 4;        // ciphertexts
        // GELU(x) = x Phi(x) fitted on 400 Chebyshev nodes of [-1, 1] (largest fitting error 7.5e-6)
        const std::vector<double> p = {7.478882192e-06, 0.5, 0.3986996239, 5.693399438e-16, -0.06524876431, 8.212237276e-16, 0.007893532612,
                                       4.90786802e-16};
        EncryptionParameters parms;     // the default basis: primes k 2^32 + 1 just below 2^60
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);
        const std::size_t n = ev.poly_degree(), half = n / 2;
        auto prefix = [&](unsigned limbs) {   // an evaluator over the first `limbs` ciphertext moduli
            EncryptionParameters pp = parms;
            pp.n_limbs = limbs;
            for (unsigned i = 0; i < limbs; ++i) pp.moduli.push_back(ev.modulus(i));
            return pp;
        };
        Evaluator evq(prefix(Lq));
        // inputs at a scale near the primes keep every power's scale near it; the result at 2^40 fits q_0 with room to spare
        const double scale_in = (double)ev.modulus(1), scale_out = std::ldexp(1.0, 40);

        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, 0, secret.data(), seed, relin.data());

        std::mt19937_64 rng(5);
        std::uniform_real_distribution<double> uni(-1.0, 1.0);
        std::vector<std::complex<double>> z(B * half);
        for (auto &v : z) v = uni(rng);
        std::vector<std::uint64_t> plain(B * evq.poly_words()), ct(B * evq.ciphertext_words());
        evq.encode_ckks(z.data(), B, scale_in, plain.data());
        evq.encrypt(0, secret.data(), seed, 0, plain.data(), CiphertextBatch{ct.data(), B});

        CkksPolyEval act(ev, K, p, scale_in, relin.data(), scale_out);
        const unsigned Lf = act.result_limbs();
        Evaluator evf(prefix(Lf));
        std::vector<std::uint64_t> out(B * evf.ciphertext_words()), phase(B * evf.poly_words());
        act.apply(ConstCiphertextBatch(ct.data(), B), CiphertextBatch{out.data(), B});
        evf.decrypt(secret.data(), ConstCiphertextBatch(out.data(), B), phase.data());
        std::vector<std::complex<double>> y(B * half);
        evf.decode_ckks(phase.data(), B, act.result_scale(), y.data());

        double worst = 0;
        for (std::size_t i = 0; i < B * half; ++i) {
            double want = 0;
            for (std::size_t k = p.size(); k-- > 0;) want = want * z[i].real() + p[k];
            worst = std::max(worst, std::abs(y[i] - want));
        }
        std::cout << B * half << " activations at " << Lf << " limb(s), scale 2^" << std::log2(act.result_scale()) << ", largest error "
                  << worst << std::endl;
        return worst < 1e-6 ? 0 : 2;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
