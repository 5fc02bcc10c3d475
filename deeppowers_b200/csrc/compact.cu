// compact.cu — sm_90a kernels and launchers of compact ciphertexts (DESIGN.md §2.24): the scale-and-pack of level-1 pairs and the
// client's unpack-and-lift / unpack-and-finish.  The transforms, modulus switches and the product by the secret around them are the
// existing launchers'.
//
// Compiled once per arithmetic variant (-DDPFHE_FAST=0 / 1, namespace dpfhe::gen / dpfhe::fast), like keys.cu and eval.cu.  A
// separate compilation unit: no kernel of the other units shares a body with these.
#include <cuda_runtime.h>

#include "compact.cuh"
#include "launch_util.hpp"

namespace dpfhe {
namespace DPFHE_VNS {

namespace {
constexpr int WARPS = 8;   // tiles per CTA of 256 threads: one warp each
}

// x [n_tiles][64] (coefficient form, [0, q0)) -> out [n_tiles][bits]
__global__ void __launch_bounds__(256) compact_pack_kernel(const __grid_constant__ CompactArgs A, const u64 *__restrict__ x, u64 *__restrict__ out,
                                                           size_t n_tiles) {
    __shared__ u64 y[WARPS][64];
    const int lane = (int)(threadIdx.x & 31), wid = (int)(threadIdx.x >> 5);
    for (size_t tile = (size_t)blockIdx.x * WARPS + wid; tile < n_tiles; tile += (size_t)gridDim.x * WARPS) {
        compact_pack_values(x + tile * 64, y[wid], A, lane);
        __syncwarp();
        compact_pack_store(y[wid], out + tile * A.bits, A, lane);
        __syncwarp();
    }
}

// FINISH = false: the c1' rows of the compact ciphertexts cct [n][2][tiles * bits] lifted into dst [n][N];
// FINISH = true: the c0' rows and prod [n][N] (c1' s mod q0) into the plaintexts dst [n][N], both in coefficient form
template <bool FINISH>
__global__ void __launch_bounds__(256) compact_unpack_kernel(const __grid_constant__ CompactArgs A, const u64 *__restrict__ cct,
                                                             const u64 *__restrict__ prod, u64 *__restrict__ dst, size_t n_tiles) {
    __shared__ u64 w[WARPS][64];
    const int lane = (int)(threadIdx.x & 31), wid = (int)(threadIdx.x >> 5);
    for (size_t tile = (size_t)blockIdx.x * WARPS + wid; tile < n_tiles; tile += (size_t)gridDim.x * WARPS) {
        const size_t item = tile / A.tiles, in_poly = tile % A.tiles;
        compact_load_words(cct + ((2 * item + (FINISH ? 0 : 1)) * A.tiles + in_poly) * A.bits, w[wid], A, lane);
        __syncwarp();
        if (FINISH) compact_finish_tile(w[wid], prod + tile * 64, dst + tile * 64, A, lane);
        else compact_lift_tile(w[wid], dst + tile * 64, A, lane);
        __syncwarp();
    }
}

namespace {
unsigned tile_grid(const LaunchCtx &lc, size_t n_tiles) { return ew_grid(lc, (n_tiles + WARPS - 1) / WARPS * 256); }
}  // namespace

// n_polys polynomials x [n_polys][N] (coefficient form modulo q0) switched to 2^bits and packed into out [n_polys][N bits / 64]; one launch
cudaError_t launch_compact_pack(const LaunchCtx &lc, const CompactArgs &A, const u64 *x, u64 *out, size_t n_polys, cudaStream_t st) {
    const size_t n_tiles = n_polys * A.tiles;
    if (!n_tiles) return cudaSuccess;
    compact_pack_kernel<<<tile_grid(lc, n_tiles), 256, 0, st>>>(A, x, out, n_tiles);
    return cudaGetLastError();
}

// finish = false: c1' of the n compact ciphertexts cct lifted into dst [n][N]; finish = true: c0' and prod [n][N] into the level-1
// plaintexts dst [n][N] (coefficient form); one launch
cudaError_t launch_compact_unpack(const LaunchCtx &lc, bool finish, const CompactArgs &A, const u64 *cct, const u64 *prod, u64 *dst, size_t n,
                                  cudaStream_t st) {
    const size_t n_tiles = n * A.tiles;
    if (!n_tiles) return cudaSuccess;
    auto k = finish ? compact_unpack_kernel<true> : compact_unpack_kernel<false>;
    k<<<tile_grid(lc, n_tiles), 256, 0, st>>>(A, cct, prod, dst, n_tiles);
    return cudaGetLastError();
}

}  // namespace DPFHE_VNS
}  // namespace dpfhe
