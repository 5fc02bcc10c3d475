// encrypted_compact.cpp — compact result ciphertexts between a server and a client (DESIGN.md §2.24).  The client encrypts two
// batches of BGV slots at level Lq.  The server multiplies them with multiply_relin_rescale_grouped, which leaves the products one level
// down, and downloads them compacted: switched to q0, then to 2^bits, and bit-packed on the device, so that only N bits / 4 bytes per
// ciphertext cross the bus and the wire, against 16 (Lq - 1) N for the full products.  It writes them as wire kind 10.  The client reads
// the file, decrypts the compact ciphertexts to level-1 plaintexts, decodes them and checks every slot against the product of its
// inputs times the factors of the divisions (q_{Lq-1} q_{Lq-2} .. q_1)^-1 mod t.  The server's buffers are on the device (the CUDA
// runtime's cudaMalloc / cudaMemcpy move the data, as in encrypted_deep_mlp.cpp).
#include <cuda_runtime.h>
#include <deeppowers_fhe.hpp>
#include <dpfhe_wire.hpp>

#include <cstdint>
#include <cstring>
#include <iostream>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

using namespace deeppowers::api::fhe;

namespace {

void cuda_check(cudaError_t e) {
    if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
}

struct DeviceWords {
    std::uint64_t *p = nullptr;
    explicit DeviceWords(std::size_t words) { cuda_check(cudaMalloc(&p, words * 8)); }
    ~DeviceWords() { cudaFree(p); }
    DeviceWords(const DeviceWords &) = delete;
    DeviceWords &operator=(const DeviceWords &) = delete;
};

std::uint64_t inverse_mod(std::uint64_t a, std::uint64_t m) {   // m prime
    std::uint64_t r = 1, b = a % m;
    for (std::uint64_t e = m - 2; e; e >>= 1, b = b * b % m)
        if (e & 1) r = r * b % m;
    return r;
}

}  // namespace

int main(int argc, char **argv) {
    try {
        const unsigned Lq = 4, K = 2, bits = 36;         // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t B = 4;                         // products
        const std::uint64_t t = 65537;                   // prime, 1 mod 2N
        const std::string dir = argc > 1 ? argv[1] : ".";
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);
        const std::size_t n = ev.poly_degree(), Pq = Lq * n, P = ev.poly_words(), W = ev.compact_words(bits);
        std::vector<std::uint64_t> moduli;
        for (unsigned l = 0; l < Lq + K; ++l) moduli.push_back(ev.modulus(l));

        // ---- the client: secret, relinearisation key, ciphertexts of 2B slot vectors at level Lq
        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(P), key(ev.key_words(K));
        ev.generate_secret(seed, secret.data());
        ev.generate_relin_key(K, t, secret.data(), seed, key.data());
        std::mt19937_64 rng(5);
        std::vector<std::int64_t> slots(2 * B * n);
        for (auto &v : slots) v = static_cast<std::int64_t>(rng() % t);
        std::vector<std::uint64_t> plain(2 * B * Pq), ct(2 * B * 2 * Pq);
        ev.encode_bgv(Lq, slots.data(), 2 * B, t, plain.data());
        ev.encrypt(Lq, t, secret.data(), seed, 0, plain.data(), CiphertextBatch{ct.data(), 2 * B});

        // ---- the server: the products at level Lq - 1, downloaded compact and written as wire kind 10
        DeviceWords d_ct(ct.size()), d_key(key.size()), d_prod(B * 2 * (Lq - 1) * n);
        cuda_check(cudaMemcpy(d_ct.p, ct.data(), ct.size() * 8, cudaMemcpyHostToDevice));
        cuda_check(cudaMemcpy(d_key.p, key.data(), key.size() * 8, cudaMemcpyHostToDevice));
        ev.multiply_relin_rescale_grouped_device(K, d_ct.p, d_ct.p + B * 2 * Pq, d_key.p, d_prod.p, B, t);
        std::vector<std::uint64_t> payload(kCompactPrefixWords + B * W);
        payload[0] = bits;
        payload[1] = t;
        ev.download_compact_ciphertexts(Lq - 1, bits, t, ConstCiphertextBatch{d_prod.p, B}, payload.data() + kCompactPrefixWords);
        WireHeader h = make_wire_header(13, 1, WireKind::CompactCiphertexts, B, moduli.data());
        h.form = 0;
        const std::string f_out = dir + "/compact_results.dpfhe";
        write_wire_file(f_out, h, payload.data());

        // ---- the client: reads the results, decrypts them to level-1 plaintexts, decodes them
        std::vector<std::uint64_t> file;
        const WireHeader hr = read_wire_file(f_out, file);
        if (hr.kind != 10 || hr.count != B || file[0] != bits || file[1] != t) throw std::runtime_error("unexpected wire file");
        std::vector<std::uint64_t> pt(B * n), out(B * n);
        ev.decrypt_compact(bits, t, secret.data(), file.data() + kCompactPrefixWords, B, pt.data());
        ev.decode_bgv(1, pt.data(), B, t, out.data());
        std::uint64_t f = 1;   // the rescale divides by q_{Lq-1}, the compaction by q_{Lq-2} .. q_1
        for (unsigned l = 1; l < Lq; ++l) f = f * inverse_mod(moduli[l] % t, t) % t;
        std::size_t wrong = 0;
        for (std::size_t i = 0; i < B * n; ++i) {
            const std::uint64_t want = static_cast<std::uint64_t>(slots[i]) * static_cast<std::uint64_t>(slots[B * n + i]) % t * f % t;
            if (out[i] != want) ++wrong;
        }
        std::cout << "compact: " << B * W * 8 << " bytes for " << B * 2 * (Lq - 1) * n * 8 << " (bits = " << bits << ", level " << Lq - 1
                  << "); " << B * n << " slot products, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
