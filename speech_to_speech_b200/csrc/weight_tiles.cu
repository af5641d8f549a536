// weight_tiles.cu -- re-lay a row-major 16-bit weight matrix [N, K] into the fragment-major "tiled" layout the
// decode kernels stream (decode_common.cuh): tile = 8 rows, window = 32 k,
//   element (row 8*tile + g, k 32*w + 8*t + e)  ->  ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e
// so that (a) any run of k windows of a tile is one contiguous block = one cp.async.bulk, and (b) the 16-byte
// fragment loads of a warp read 512 consecutive bytes of shared memory.  Rows N..roundup8(N) are zero.  Done once
// at finalize; the row-major copy stays for the TMA/wgmma GEMMs (prefill, encoder) and the embedding lookup.
//
// FP8 E4M3 weight-only storage (Llama-family decode, llama_decode.cu): per row n the integer exponent e_n is the smallest
// with max_k |W[n,k]| * 2^-e_n <= 448 (not below FP8_MIN_EXP; 0 for an all-zero row), the code is
// Q[n,k] = e4m3_rn_satfinite(W[n,k] * 2^-e_n) and the row scale 2^e_n.  A power-of-two scale makes dq(Q)[n,k] = Q[n,k] * 2^e_n
// a bf16 number, so the row-major matrix is overwritten with dq(Q): the 16-bit prefill GEMMs and the FP8 decode launch
// multiply by the same weight values.  The codes use the same tiling at one byte per element,
//   element (row 8*tile + g, k 32*w + 8*t + e)  ->  byte ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e,
// and the roundup8(N) fp32 scales follow them (1 for the padding rows).
#include <cuda_fp8.h>

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

// lowest row exponent: keeps the smallest dequantised value (2^-9 * 2^e_n) a normal bf16 number.  Rows whose largest
// magnitude is below 448 * 2^-100 lose precision instead; trained weights are nowhere near.
constexpr int FP8_MIN_EXP = -100;

// one CTA per tile of 8 rows, one warp per row: row maximum -> exponent -> codes (tiled), scale, dequantised row
__global__ void __launch_bounds__(256) quantize_tile_fp8_kernel(__nv_bfloat16* __restrict__ W, int N, int K,
                                                                unsigned char* __restrict__ Wq, float* __restrict__ scale) {
  const int tile = blockIdx.x, g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)tile * 8 + g;
  uint2* qt = reinterpret_cast<uint2*>(Wq) + (long long)tile * (K >> 5) * 32 + 4 * g;   // + w * 32 + t
  if (row >= N) {
    for (int v = lane; v < (K >> 3); v += 32) qt[(v >> 2) * 32 + (v & 3)] = make_uint2(0u, 0u);
    if (lane == 0) scale[row] = 1.f;
    return;
  }
  uint4* wr = reinterpret_cast<uint4*>(W + row * K);
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
  const float inv = exp2f((float)-e), sc = exp2f((float)e);   // exact powers of two, both normal fp32
  if (lane == 0) scale[row] = sc;
  for (int v = lane; v < (K >> 3); v += 32) {
    const uint4 x = wr[v];
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
    uint32_t dq[4], q[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = DT<__nv_bfloat16>::to_f2(xs[i]);
      const uint32_t c0 = __nv_cvt_float_to_fp8(f.x * inv, __NV_SATFINITE, __NV_E4M3);
      const uint32_t c1 = __nv_cvt_float_to_fp8(f.y * inv, __NV_SATFINITE, __NV_E4M3);
      q[i >> 1] |= (c0 | (c1 << 8)) << (16 * (i & 1));
      const __half_raw h0 = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)c0, __NV_E4M3);
      const __half_raw h1 = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)c1, __NV_E4M3);
      dq[i] = DT<__nv_bfloat16>::pack2(__half2float(__half(h0)) * sc, __half2float(__half(h1)) * sc);
    }
    qt[(v >> 2) * 32 + (v & 3)] = make_uint2(q[0], q[1]);
    wr[v] = make_uint4(dq[0], dq[1], dq[2], dq[3]);
  }
}
}  // namespace

size_t tiled_fp8_weight_bytes(int N, int K) { return tiled_weight_elems(N, K) + (size_t)((N + 7) / 8) * 8 * sizeof(float); }

int quantize_tile_weights_fp8_launch(void* W, int N, int K, void* Wq, cudaStream_t stream) {
  S2S_REQUIRE(K % 32 == 0, "quantize_tile_weights_fp8: K=%d must be a multiple of 32", K);
  unsigned char* q = reinterpret_cast<unsigned char*>(Wq);
  quantize_tile_fp8_kernel<<<(N + 7) / 8, 256, 0, stream>>>(reinterpret_cast<__nv_bfloat16*>(W), N, K, q,
                                                           reinterpret_cast<float*>(q + tiled_weight_elems(N, K)));
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

size_t tiled_weight_elems(int N, int K) { return (size_t)((N + 7) / 8) * 8 * (size_t)K; }

int tile_weights_launch(const void* W, int N, int K, void* Wt, cudaStream_t stream) {
  S2S_REQUIRE(K % 32 == 0, "tile_weights: K=%d must be a multiple of 32", K);
  const long long n_vec = (long long)tiled_weight_elems(N, K) / 8;
  const int blocks = (int)std::min<long long>((n_vec + 255) / 256, 132 * 16);
  tile_weights_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(W), N, K, reinterpret_cast<uint4*>(Wt), n_vec);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}
