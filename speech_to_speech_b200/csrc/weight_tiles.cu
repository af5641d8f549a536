// weight_tiles.cu -- re-lay a row-major 16-bit weight matrix [N, K] into the fragment-major "tiled" layout the
// decode kernels stream (decode_common.cuh): tile = 8 rows, window = 32 k,
//   element (row 8*tile + g, k 32*w + 8*t + e)  ->  ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e
// so that (a) any run of k windows of a tile is one contiguous block = one cp.async.bulk, and (b) the 16-byte
// fragment loads of a warp read 512 consecutive bytes of shared memory.  Rows N..roundup8(N) are zero.  Done once
// at finalize; the row-major copy stays for the TMA/wgmma GEMMs (prefill, encoder) and the embedding lookup.
#include <algorithm>

#include "kernels.cuh"

namespace {
__global__ void tile_weights_kernel(const uint4* __restrict__ W, int N, int K, uint4* __restrict__ Wt, long long n_vec) {
  const int wpr = K >> 5;  // windows per row
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n_vec; v += (long long)gridDim.x * blockDim.x) {
    const int lane = (int)(v & 31);
    const long long tw = v >> 5;
    const int w = (int)(tw % wpr);
    const long long tile = tw / wpr;
    const long long row = tile * 8 + (lane >> 2);
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (row < N) val = W[(row * K + (long long)w * 32 + (lane & 3) * 8) >> 3];
    Wt[v] = val;
  }
}
}  // namespace

size_t tiled_weight_elems(int N, int K) { return (size_t)((N + 7) / 8) * 8 * (size_t)K; }

int tile_weights_launch(const void* W, int N, int K, void* Wt, cudaStream_t stream) {
  S2S_REQUIRE(K % 32 == 0, "tile_weights: K=%d must be a multiple of 32", K);
  const long long n_vec = (long long)tiled_weight_elems(N, K) / 8;
  const int blocks = (int)std::min<long long>((n_vec + 255) / 256, 132 * 16);
  tile_weights_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(W), N, K, reinterpret_cast<uint4*>(Wt), n_vec);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}
