// emu_compact.cpp — host emulator of the compact-ciphertext tile bodies (TEST INFRASTRUCTURE ONLY).
//
// Runs the bodies of deeppowers_b200/csrc/compact.cuh tile by tile as compact_pack_kernel and compact_unpack_kernel do: the 32 lanes
// of a tile's warp one after another, each phase for every lane before the next, with the launch constants of the product's
// build_compact_args.  Built by tests/test_compact_emu_cpu.py in both arithmetic variants; never linked into libdpfhe.so.
#include <cstdint>
#include <cstdlib>

#include "compact.cuh"
#include "host_params.hpp"

using namespace dpfhe;
using namespace dpfhe::DPFHE_VNS;

extern "C" {

// x [n_polys][N] (coefficient form, [0, q0)) -> out [n_polys][N bits / 64]
void emu_compact_pack(uint64_t q0, unsigned log_n, unsigned bits, uint64_t t_plain, const uint64_t *x, uint64_t *out, size_t n_polys) {
    CompactArgs A;
    build_compact_args(q0, log_n, bits, t_plain, A);
    u64 y[64];
    for (size_t tile = 0; tile < n_polys * A.tiles; ++tile) {
        for (int lane = 0; lane < 32; ++lane) compact_pack_values(x + tile * 64, y, A, lane);
        for (int lane = 0; lane < 32; ++lane) compact_pack_store(y, out + tile * bits, A, lane);
    }
}

// finish = 0: the c1' rows of cct [n][2][N bits / 64] lifted into dst [n][N]; finish = 1: the c0' rows and prod [n][N] into the
// plaintexts dst [n][N] (coefficient form)
void emu_compact_unpack(int finish, uint64_t q0, unsigned log_n, unsigned bits, uint64_t t_plain, const uint64_t *cct, const uint64_t *prod,
                        uint64_t *dst, size_t n) {
    CompactArgs A;
    build_compact_args(q0, log_n, bits, t_plain, A);
    u64 w[64];
    for (size_t tile = 0; tile < n * A.tiles; ++tile) {
        const size_t item = tile / A.tiles, in_poly = tile % A.tiles;
        const u64 *src = cct + ((2 * item + (finish ? 0 : 1)) * A.tiles + in_poly) * bits;
        for (int lane = 0; lane < 32; ++lane) compact_load_words(src, w, A, lane);
        for (int lane = 0; lane < 32; ++lane) {
            if (finish) compact_finish_tile(w, prod + tile * 64, dst + tile * 64, A, lane);
            else compact_lift_tile(w, dst + tile * 64, A, lane);
        }
    }
}
}
