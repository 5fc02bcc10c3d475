// encrypted_seeded.cpp — seeded ciphertexts and a seeded relinearisation key between a client and a server (DESIGN.md §2.23).  The
// client encrypts two batches of BGV slots with SeededEncryptor and makes a seeded relinearisation key: only c0 and the key's b rows
// are written, as wire kinds 7 and 8, each with the 32-byte public seed in its prefix.  The server reads the two files, uploads them
// seeded (half the bytes of the full objects cross the bus; the `a` rows are regenerated on the device) and multiplies the batches
// with multiply_relin_grouped.  The client decrypts the products and checks them slot by slot mod t.  The server's buffers are on the
// device (the CUDA runtime's cudaMalloc / cudaMemcpy move the data, as in encrypted_deep_mlp.cpp).
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

// the 5-word prefix of a seeded wire kind: the public seed as four little-endian words, then first_index or the item number
std::vector<std::uint64_t> with_prefix(const Evaluator::Seed &a_seed, std::uint64_t number, const std::vector<std::uint64_t> &rows) {
    std::vector<std::uint64_t> out(kSeededPrefixWords + rows.size());
    for (int w = 0; w < 4; ++w)
        for (int b = 0; b < 8; ++b) out[w] |= std::uint64_t(a_seed[8 * w + b]) << (8 * b);
    out[4] = number;
    std::memcpy(out.data() + kSeededPrefixWords, rows.data(), rows.size() * 8);
    return out;
}

Evaluator::Seed seed_of(const std::vector<std::uint64_t> &payload) {
    Evaluator::Seed s;
    for (int i = 0; i < 32; ++i) s[i] = static_cast<std::uint8_t>(payload[i / 8] >> (8 * (i % 8)));
    return s;
}

}  // namespace

int main(int argc, char **argv) {
    try {
        const unsigned Lq = 4, K = 2;                   // 4 ciphertext moduli + 2 special primes, N = 8192
        const std::size_t B = 3;                        // ciphertexts per operand batch
        const std::uint64_t t = 65537;                  // prime, 1 mod 2N
        const std::string dir = argc > 1 ? argv[1] : ".";
        EncryptionParameters parms;
        parms.n_limbs = Lq + K;
        Evaluator ev(parms);
        const std::size_t n = ev.poly_degree(), Pq = Lq * n, P = ev.poly_words();
        std::vector<std::uint64_t> moduli;
        for (unsigned l = 0; l < Lq + K; ++l) moduli.push_back(ev.modulus(l));

        // ---- the client: secret, seeded ciphertexts of 2B slot vectors at level Lq, a seeded relinearisation key
        const Evaluator::Seed seed = Evaluator::random_seed();
        std::vector<std::uint64_t> secret(P);
        ev.generate_secret(seed, secret.data());
        std::mt19937_64 rng(3);
        std::vector<std::int64_t> slots(2 * B * n);
        for (auto &v : slots) v = static_cast<std::int64_t>(rng() % t);
        std::vector<std::uint64_t> plain(2 * B * Pq), c0(2 * B * Pq), b(ev.seeded_key_words(K));
        ev.encode_bgv(Lq, slots.data(), 2 * B, t, plain.data());
        SeededEncryptor enc(ev, SeededEncryptor::Memory::host, Lq, secret.data(), seed, t, 1000);
        enc.encrypt(plain.data(), 2 * B, c0.data());
        ev.generate_relin_key_seeded(K, t, secret.data(), seed, b.data());
        const std::string f_ct = dir + "/seeded_ct.dpfhe", f_key = dir + "/seeded_relin.dpfhe";
        write_wire_file(f_ct, make_wire_header(13, Lq, WireKind::SeededCiphertexts, 2 * B, moduli.data()),
                        with_prefix(enc.public_seed(), 1000, c0).data());
        write_wire_file(f_key, make_wire_header(13, Lq + K, WireKind::SeededSwitchKey, K, moduli.data()), with_prefix(enc.public_seed(), 0, b).data());

        // ---- the server: reads the files, uploads them seeded, multiplies batch 0 by batch 1
        std::vector<std::uint64_t> ct_file, key_file;
        const WireHeader hc = read_wire_file(f_ct, ct_file), hk = read_wire_file(f_key, key_file);
        if (hc.kind != 7 || hk.kind != 8 || hc.count != 2 * B || hk.count != K) throw std::runtime_error("unexpected wire files");
        DeviceWords d_ct(2 * B * 2 * Pq), d_key(ev.key_words(K)), d_out(B * 2 * Pq);
        ev.upload_seeded_ciphertexts(Lq, seed_of(ct_file), ct_file[4], ct_file.data() + kSeededPrefixWords, CiphertextBatch{d_ct.p, 2 * B});
        ev.upload_seeded_switch_keys(K, seed_of(key_file), {key_file[4]}, key_file.data() + kSeededPrefixWords, d_key.p);
        ev.multiply_relin_grouped_device(K, d_ct.p, d_ct.p + B * 2 * Pq, d_key.p, d_out.p, B, t);
        std::vector<std::uint64_t> prod(B * 2 * Pq);
        cuda_check(cudaDeviceSynchronize());
        cuda_check(cudaMemcpy(prod.data(), d_out.p, prod.size() * 8, cudaMemcpyDeviceToHost));

        // ---- the client: decrypts and decodes the products
        std::vector<std::uint64_t> phase(B * Pq), out(B * n);
        ev.decrypt(Lq, secret.data(), ConstCiphertextBatch(prod.data(), B), phase.data());
        ev.decode_bgv(Lq, phase.data(), B, t, out.data());
        std::size_t wrong = 0;
        for (std::size_t i = 0; i < B * n; ++i)
            if (out[i] != static_cast<std::uint64_t>(slots[i]) * static_cast<std::uint64_t>(slots[B * n + i]) % t) ++wrong;
        std::cout << "seeded: " << c0.size() * 8 << " + " << b.size() * 8 << " bytes sent for " << 2 * c0.size() * 8 << " + " << 2 * b.size() * 8
                  << "; " << B * n << " slot products, " << wrong << " wrong" << std::endl;
        return wrong ? 2 : 0;
    } catch (const std::exception &e) {
        std::cerr << "Error: " << e.what() << std::endl;
        return 1;
    }
}
