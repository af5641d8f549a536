// weight_tiles.cu -- lay row-major 16-bit weight rows [rows, K] into the fragment-major "tiled" layout of a [N, K] matrix
// that the decode kernels stream (decode_common.cuh): tile = 8 rows, window = 32 k,
//   element (row 8*tile + g, k 32*w + 8*t + e)  ->  ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e
// so that (a) any run of k windows of a tile is one contiguous block = one cp.async.bulk, and (b) the 16-byte
// fragment loads of a warp read 512 consecutive bytes of shared memory, and (c) each 32-k window of a tile is an 8 x 64 B
// row-major block, which the wgmma prefill GEMM loads with a 4-D TMA map (gemm_tc.cu).  Rows N..roundup8(N) stay zero.
// The Llama family keeps its projections and lm_head in this layout only, and Whisper its decoder matrices and token
// embedding: bind / init_random tile each tensor's rows into place (tile_rows_launch, weight_arena.cu), so no row-major
// copy exists.  Llama's prefill and decode read the same copy.
//
// FP8 E4M3 weight-only storage (Llama-family decode, llama_decode.cu): per row n the integer exponent e_n is the smallest
// with max_k |W[n,k]| * 2^-e_n <= 448 (not below FP8_MIN_EXP; 0 for an all-zero row), the code is
// Q[n,k] = e4m3_rn_satfinite(W[n,k] * 2^-e_n) and the row scale 2^e_n.  A power-of-two scale makes dq(Q)[n,k] = Q[n,k] * 2^e_n
// a bf16 number: the prefill GEMM expands the codes to exactly dq(Q) in shared memory, so prefill and the FP8 decode
// launch multiply by the same weight values.  A row's scale depends on that row alone, so a tensor is quantised by
// itself, at bind time.  The codes use the same tiling at one byte per element,
//   element (row 8*tile + g, k 32*w + 8*t + e)  ->  byte ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e,
// and the roundup8(N) fp32 scales follow them (1 for the padding rows).
#include <cuda_fp8.h>

#include <algorithm>

#include "kernels.cuh"

namespace {
// lowest row exponent: keeps the smallest dequantised value (2^-9 * 2^e_n) a normal bf16 number.  Rows whose largest
// magnitude is below 448 * 2^-100 lose precision instead; trained weights are nowhere near.
constexpr int FP8_MIN_EXP = -100;

// rows r of a row-major 16-bit source -> rows row0 + r * rstride of a tiled matrix; one 16-byte vector per thread
__global__ void tile_rows_kernel(const uint4* __restrict__ src, long long n_vec, int K, uint4* __restrict__ Wt, int row0,
                                 int rstride) {
  const int vpr = K >> 3, wpr = K >> 5;   // vectors, windows per row
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n_vec; v += (long long)gridDim.x * blockDim.x) {
    const long long r = v / vpr;
    const int c = (int)(v - r * vpr);
    const long long dr = row0 + r * rstride;
    Wt[((dr >> 3) * wpr + (c >> 2)) * 32 + 4 * (dr & 7) + (c & 3)] = src[v];
  }
}

// one warp per source row: row maximum -> exponent -> tiled codes and the row scale of row row0 + r * rstride
__global__ void __launch_bounds__(256) quantize_rows_fp8_kernel(const __nv_bfloat16* __restrict__ src, int rows, int K, int row0,
                                                                int rstride, unsigned char* __restrict__ Wq,
                                                                float* __restrict__ scale) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const long long dr = row0 + (long long)r * rstride;
  uint2* qt = reinterpret_cast<uint2*>(Wq) + (dr >> 3) * (K >> 5) * 32 + 4 * (dr & 7);   // + w * 32 + t
  const uint4* wr = reinterpret_cast<const uint4*>(src + (long long)r * K);
  float amax = 0.f;
  for (int v = lane; v < (K >> 3); v += 32) {
    const uint4 x = wr[v];
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = DT<__nv_bfloat16>::to_f2(xs[i]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  amax = warp_max(amax);
  int e = 0;
  if (amax > 0.f) {   // amax = m * 2^x, m in [0.5, 1); 448 = 0.875 * 2^9
    int x;
    const float m = frexpf(amax, &x);
    e = max(m <= 0.875f ? x - 9 : x - 8, FP8_MIN_EXP);
  }
  const float inv = exp2f((float)-e);   // exact power of two, normal fp32
  if (lane == 0) scale[dr] = exp2f((float)e);
  for (int v = lane; v < (K >> 3); v += 32) {
    const uint4 x = wr[v];
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
    uint32_t q[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = DT<__nv_bfloat16>::to_f2(xs[i]);
      const uint32_t c0 = __nv_cvt_float_to_fp8(f.x * inv, __NV_SATFINITE, __NV_E4M3);
      const uint32_t c1 = __nv_cvt_float_to_fp8(f.y * inv, __NV_SATFINITE, __NV_E4M3);
      q[i >> 1] |= (c0 | (c1 << 8)) << (16 * (i & 1));
    }
    qt[(v >> 2) * 32 + (v & 3)] = make_uint2(q[0], q[1]);
  }
}
}  // namespace

size_t tiled_fp8_weight_bytes(int N, int K) { return tiled_weight_elems(N, K) + (size_t)((N + 7) / 8) * 8 * sizeof(float); }

int tile_rows_launch(const void* src, int rows, int K, void* Wt, int N, int row0, int rstride, bool fp8, cudaStream_t stream) {
  S2S_REQUIRE(K % 32 == 0, "tile_rows: K=%d must be a multiple of 32", K);
  S2S_REQUIRE(rows >= 1 && rstride >= 1 && row0 >= 0 && row0 + (long long)(rows - 1) * rstride < N,
              "tile_rows: rows %d, first %d, stride %d outside the %d rows of the matrix", rows, row0, rstride, N);
  if (fp8) {
    unsigned char* q = reinterpret_cast<unsigned char*>(Wt);
    quantize_rows_fp8_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(src), rows, K, row0, rstride,
                                                                  q, reinterpret_cast<float*>(q + tiled_weight_elems(N, K)));
  } else {
    const long long n_vec = (long long)rows * K / 8;
    const int blocks = (int)std::min<long long>((n_vec + 255) / 256, 132 * 16);
    tile_rows_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(src), n_vec, K, reinterpret_cast<uint4*>(Wt), row0, rstride);
  }
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

size_t tiled_weight_elems(int N, int K) { return (size_t)((N + 7) / 8) * 8 * (size_t)K; }
