// encrypted_deep_mlp.cpp — a three-layer encrypted network y = W3 p(W2 p(W1 x + b1) + b2), slot by slot mod t, on ONE evaluator with
// ONE set of top-level keys.  The client encodes and encrypts at the ciphertext level Lq and decrypts and decodes at the result's level
// with the level calls of DESIGN.md §2.22; the server runs W1 at Lq, adds b1 at Lq, the activation p down to Lf1, W2 and b2 at Lf1, p
// again at Lf1 (PolyEval's level constructor) down to Lf2, and W3 at Lf2.  No evaluator over a prefix of the moduli and no restricted
// key.  The server's buffers are on the device (the CUDA runtime's cudaMalloc / cudaMemcpy move the data); the result is checked
// against the same computation mod t.
//
// Layout: every vector of DIM entries repeats with period DIM across the first slot row, and so does every diagonal, so each layer's
// output is already the periodic input of the next one.
#include <cuda_runtime.h>
#include <deeppowers_fhe.hpp>

#include <cstdint>
#include <iostream>
#include <random>
#include <stdexcept>
#include <vector>

using namespace deeppowers::api::fhe;

namespace {

void cuda_check(cudaError_t e) {
    if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
}

// a device copy of `words` 64-bit words
struct DeviceWords {
    std::uint64_t *p = nullptr;
    explicit DeviceWords(std::size_t words) { cuda_check(cudaMalloc(&p, words * 8)); }
    DeviceWords(const std::vector<std::uint64_t> &h) : DeviceWords(h.size()) { cuda_check(cudaMemcpy(p, h.data(), h.size() * 8, cudaMemcpyHostToDevice)); }
    ~DeviceWords() { cudaFree(p); }
    DeviceWords(const DeviceWords &) = delete;
    DeviceWords &operator=(const DeviceWords &) = delete;
};

}  // namespace

int main() {
    try {
        const unsigned Lq = 5, K = 2;                   // 5 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t DIM = 32, BABY = 8, B = 4;    // three 32 x 32 layers, 8 baby steps, 4 input vectors
        const std::uint64_t t = 65537;                  // prime, 1 mod 2N
        const std::vector<std::int64_t> p = {3, -2, 1}; // the activation: 3 - 2x + x^2
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);                            // the one evaluator: every call, at every level
        const std::size_t n = ev.poly_degree(), half = n / 2;

        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(ev.poly_words()), relin(ev.key_words(K)), galois(BABY * ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, t, secret.data(), seed, relin.data());
        std::vector<long> steps;
        for (std::size_t b = 1; b <= BABY; ++b) steps.push_back((long)b);
        ev.generate_galois_keys(K, t, secret.data(), steps, seed, galois.data());   // one set for the three layers
        const std::uint64_t *giant_key = galois.data() + (BABY - 1) * ev.key_words(K);

        std::mt19937_64 rng(13);
        auto small = [&](int r) { return (std::int64_t)(rng() % (2 * r + 1)) - r; };
        std::vector<std::vector<std::int64_t>> W(3, std::vector<std::int64_t>(DIM * DIM));
        for (auto &w : W)
            for (auto &v : w) v = small(8);
        std::vector<std::int64_t> X(B * DIM), b1(DIM), b2(DIM);
        for (auto &v : X) v = small(8);
        for (auto &v : b1) v = small(50);
        for (auto &v : b2) v = small(50);

        // diagonal d of a DIM x DIM matrix holds W[i % DIM][(i + d) % DIM] in slot i of the first row, rotated right by (d / BABY) * BABY
        auto encode_layer = [&](const std::vector<std::int64_t> &w, unsigned level) {
            std::vector<std::int64_t> s(DIM * n, 0);
            for (std::size_t d = 0; d < DIM; ++d)
                for (std::size_t i = 0; i < half; ++i) s[d * n + (i + (d / BABY) * BABY) % half] = w[(i % DIM) * DIM + (i + d) % DIM];
            std::vector<std::uint64_t> pt(DIM * level * n);
            ev.encode_bgv(level, s.data(), DIM, t, pt.data());
            return pt;
        };
        auto periodic = [&](const std::int64_t *v, std::size_t count) {
            std::vector<std::int64_t> s(count * n, 0);
            for (std::size_t k = 0; k < count; ++k)
                for (std::size_t i = 0; i < half; ++i) s[k * n + i] = v[k * DIM + i % DIM];
            return s;
        };

        // client: encode and encrypt at Lq
        const std::vector<std::int64_t> x_slots = periodic(X.data(), B);
        std::vector<std::uint64_t> xpt(B * Lq * n), ct(B * 2 * Lq * n);
        ev.encode_bgv(Lq, x_slots.data(), B, t, xpt.data());
        ev.encrypt(Lq, t, secret.data(), seed, 0, xpt.data(), CiphertextBatch{ct.data(), B});

        // server, on the device
        LinearLayer layer1(ev, K, encode_layer(W[0], Lq).data(), DIM, BABY, galois.data(), giant_key, t);
        PolyEval act1(ev, K, t, p, relin.data());
        const unsigned Lf1 = act1.result_limbs();
        LinearLayer layer2(ev, K, Lf1, encode_layer(W[1], Lf1).data(), DIM, BABY, galois.data(), giant_key, t);
        PolyEval act2(ev, K, Lf1, t, p, relin.data());
        const unsigned Lf2 = act2.result_limbs();
        LinearLayer layer3(ev, K, Lf2, encode_layer(W[2], Lf2).data(), DIM, BABY, galois.data(), giant_key, t);
        std::vector<std::uint64_t> b1pt(Lq * n), b2pt(Lf1 * n);
        ev.encode_bgv(Lq, periodic(b1.data(), 1).data(), 1, t, b1pt.data());
        ev.encode_bgv(Lf1, periodic(b2.data(), 1).data(), 1, t, b2pt.data());

        DeviceWords d_x(ct), d_b1(b1pt), d_b2(b2pt), d_y1(B * 2 * Lq * n), d_h1(B * 2 * Lf1 * n), d_y2(B * 2 * Lf1 * n),
            d_h2(B * 2 * Lf2 * n), d_y3(B * 2 * Lf2 * n);
        layer1.apply_device(d_x.p, d_y1.p, B);                 // W1 x
        ev.add_plain_device(Lq, d_y1.p, d_b1.p, d_y1.p, B);    // + b1
        act1.apply_device(d_y1.p, d_h1.p, B);                  // p(.), Lf1 limbs
        layer2.apply_device(d_h1.p, d_y2.p, B);                // W2 at Lf1
        ev.add_plain_device(Lf1, d_y2.p, d_b2.p, d_y2.p, B);   // + b2 at Lf1
        act2.apply_device(d_y2.p, d_h2.p, B);                  // p(.) at Lf1, Lf2 limbs
        layer3.apply_device(d_h2.p, d_y3.p, B);                // W3 at Lf2
        ev.synchronize();
        std::vector<std::uint64_t> y(B * 2 * Lf2 * n);
        cuda_check(cudaMemcpy(y.data(), d_y3.p, y.size() * 8, cudaMemcpyDeviceToHost));

        // client: decrypt and decode at the result's level
        std::vector<std::uint64_t> phase(B * Lf2 * n), out(B * n);
        ev.decrypt(Lf2, secret.data(), ConstCiphertextBatch(y.data(), B), phase.data());
        ev.decode_bgv(Lf2, phase.data(), B, t, out.data());

        const std::int64_t T = (std::int64_t)t;
        auto mod = [&](std::int64_t v) { return ((v % T) + T) % T; };
        auto layer = [&](const std::vector<std::int64_t> &w, const std::vector<std::int64_t> &v, const std::vector<std::int64_t> &bias) {
            std::vector<std::int64_t> r(DIM);
            for (std::size_t i = 0; i < DIM; ++i) {
                std::int64_t s = bias.empty() ? 0 : mod(bias[i]);
                for (std::size_t j = 0; j < DIM; ++j) s = mod(s + mod(w[i * DIM + j] * v[j]));
                r[i] = s;
            }
            return r;
        };
        auto act = [&](std::vector<std::int64_t> v) {
            for (auto &e : v) {
                std::int64_t r = 0;
                for (std::size_t c = p.size(); c-- > 0;) r = mod(r * e + p[c]);
                e = r;
            }
            return v;
        };
        std::size_t wrong = 0;
        for (std::size_t k = 0; k < B; ++k) {
            const std::vector<std::int64_t> xk(X.begin() + k * DIM, X.begin() + (k + 1) * DIM);
            const std::vector<std::int64_t> r = layer(W[2], act(layer(W[1], act(layer(W[0], xk, b1)), b2)), {});
            for (std::size_t i = 0; i < DIM; ++i)
                if (out[k * n + i] != (std::uint64_t)r[i]) ++wrong;
        }
        std::cout << B * DIM << " outputs of three layers at " << Lf2 << " limbs, one evaluator and one key set, " << wrong << " wrong"
                  << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
