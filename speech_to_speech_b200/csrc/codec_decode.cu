// codec_decode.cu -- TTS codec decoder: 16 codebook ids per 12.5 Hz frame -> 24 kHz waveform, fp32, time-major.
//
// Reference path: Qwen3TTSHandler._process_custom_voice -> model.generate_custom_voice_streaming(...) yields
// (audio_f32, 24000, timing) every `chunk_size` frames (S/TTS/qwen3_tts_handler.py:946-978); the arithmetic lives in
// the absent faster-qwen3-tts.  Structural oracle: transformers Qwen3OmniMoeCode2Wav
// (modeling_qwen3_omni_moe.py:3283-3790), restated in oracle/code2wav_ref.py:
//   mean of the frame's code embeddings -> 8 sliding-window RoPE transformer layers (LayerScale) -> RMSNorm
//   -> 2 x [transposed conv (k = stride) -> ConvNeXt block]                       (x4 in time)
//   -> causal conv 7 -> 4 x [SnakeBeta -> causal transposed conv (k = 2 stride) -> 3 dilated residual units]
//   -> SnakeBeta -> causal conv 7 -> clamp                                        (x480 in time: 1920 samples / frame)
// and chunked_decode(:3779-3790): decode `chunk` new frames behind `left_context` frames of history, drop the history.
//
// Everything convolutional is ONE contraction kernel over time-major [T, C] activations (conv1d_f32_kernel):
//   causal conv (k taps, dilation)   : rows t - (k-1-j) * dil, zero rows before the start
//   transposed conv, k = 2 s         : out[(t0-1) * s + r, o] = X[t0-1] . W[:, o, r + s] + X[t0] . W[:, o, r]  for t0 = 1..T-1
//                                      = a 2-tap contraction with N = s * C_out whose [T-1, s * C_out] result IS the
//                                      time-major [(T-1) * s, C_out] output (trim of k - s samples at both ends included)
//   transposed conv, k = s           : a 1-tap contraction with N = s * C_out
//   linear layers (transformer, ConvNeXt MLP): 1 tap.
// fp32 CUDA-core FMA with shared-memory tiles: the decoder is held to 1e-4-level waveform parity with the fp32 oracle;
// its cost is ~5 GFLOP per frame (DESIGN.md), far from the H100's limits at the session counts the talker sustains.
#include <math.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "codec_decode.cuh"
#include "kernels.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ contraction kernel
constexpr int CV_BM = 64, CV_BK = 16, CV_THREADS = 256;
constexpr int CODEC_MAX_BATCH = 16;   // sequences per launch sequence (one per concurrently speaking session)

template <int BN>
__global__ void __launch_bounds__(CV_THREADS) conv1d_f32_kernel(const ConvArgs a) {
  constexpr int TN = BN / 16;   // outputs per thread along n (4 or 2); 4 along m
  __shared__ float As[CV_BK][CV_BM + 4];
  __shared__ float Bs[CV_BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * CV_BM + a.t0, n0 = blockIdx.x * BN, z = blockIdx.z;
  const float* X = a.x + (long long)z * a.x_bs;
  float acc[4][TN];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  // loaders: A tile 64 rows x 16 c (thread -> row tid / 4, 4 consecutive c), B tile 16 c x BN n
  const int a_row = tid >> 2, a_c = (tid & 3) * 4;
  for (int j = 0; j < a.k; ++j) {
    const int xr = m0 + a_row + a.x_row0 + j * a.dil;
    const bool row_ok = (m0 + a_row) < a.T_out && xr >= 0 && xr < a.T_in;
    const float* xrow = X + (long long)xr * a.ldx;
    const float* wj = a.w + (long long)j * a.C_in * a.N;
    for (int c0 = 0; c0 < a.C_in; c0 += CV_BK) {
      float av[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + a_c + i;
        av[i] = (row_ok && c < a.C_in) ? xrow[c] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) As[a_c + i][a_row] = av[i];
      for (int e = tid; e < CV_BK * BN; e += CV_THREADS) {
        const int kk = e / BN, nn = e % BN;
        const int c = c0 + kk, n = n0 + nn;
        Bs[kk][nn] = (c < a.C_in && n < a.N) ? __ldg(wj + (long long)c * a.N + n) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < CV_BK; ++kk) {
        float ar[4], br[TN];
#pragma unroll
        for (int i = 0; i < 4; ++i) ar[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int jn = 0; jn < TN; ++jn) br[jn] = Bs[kk][tx * TN + jn];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int jn = 0; jn < TN; ++jn) acc[i][jn] = fmaf(ar[i], br[jn], acc[i][jn]);
      }
      __syncthreads();
    }
  }
  float* Y = a.y + (long long)z * a.y_bs;
  const float* R = a.resid ? a.resid + (long long)z * a.r_bs : nullptr;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = m0 + ty * 4 + i;
    if (t >= a.T_out) continue;
#pragma unroll
    for (int jn = 0; jn < TN; ++jn) {
      const int n = n0 + tx * TN + jn;
      if (n >= a.N) continue;
      float v = acc[i][jn];
      if (a.bias) v += __ldg(a.bias + (n % a.bias_mod));
      if (a.act == 1) v = gelu_erf(v);
      else if (a.act == 2) v = v / (1.0f + expf(-v));
      if (a.scale) v *= __ldg(a.scale + n);
      if (R) v += R[(long long)t * a.ldr + n];
      Y[(long long)t * a.ldy + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ tensor-core contraction
// The same contraction on the tensor cores: fp16 operands (activations converted while they are staged, weights stored as
// fp16 k-pairs at bind time), fp32 accumulate, fp32 epilogue (bias / activation / scale / residual) and fp32 output.
// mma.sync.m16n8k16, CTA tile 128 (time) x 64 (channels) x 32 (k), 8 warps as 4 x 2, warp tile 32 x 32.  The codec
// decoder is ~5 GFLOP per frame and every chunk re-decodes its 25 frames of left context (chunked_decode): on the CUDA
// cores it was the largest share of a turn (bench.py stage_ms), here it is weight- and activation-stream bound.
// wgmma is not used: the operand is a strided gather of fp32 rows (dilated taps, causal zero rows) that has to be
// converted on the way in, which the generic-proxy staging path does and a TMA descriptor does not.
constexpr int TC_BM = 128, TC_BN = 64, TC_BK = 32, TC_THREADS = 256;
constexpr int TC_APAD = 8;     // halves: row stride 40 halves = 80 B -> conflict-free 32-bit fragment loads
constexpr int TC_BPAD = 8;     // half2 words

__device__ __forceinline__ void mma_f16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// wh: weights as half2 k-pairs, [k][C_in_pad / 2][N] (C_in_pad = C_in rounded up to 2, zero padded)
__global__ void __launch_bounds__(TC_THREADS) conv1d_tc_kernel(const ConvArgs a, const __half2* __restrict__ wh, int c_pairs) {
  __shared__ __half As[2][TC_BM][TC_BK + TC_APAD];
  __shared__ uint32_t Bs[2][TC_BK / 2][TC_BN + TC_BPAD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;                 // warp tile origin: rows 32 wm, cols 32 wn
  const int m0 = blockIdx.y * TC_BM + a.t0, n0 = blockIdx.x * TC_BN, z = blockIdx.z;
  const float* X = a.x + (long long)z * a.x_bs;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;
  const int kt_per_tap = (a.C_in + TC_BK - 1) / TC_BK;
  const int n_kt = a.k * kt_per_tap;
  // A staging: 128 rows x 32 channels fp32 -> fp16.  8 consecutive lanes read one row's 128 contiguous bytes (fully coalesced
  // float4 loads); a thread handles rows a_row + 32 v, v = 0..3, channels a_c .. a_c + 3
  const int a_row = tid >> 3, a_c = (tid & 7) * 4;
  // B staging: 16 k-pairs x 64 n words; thread -> pair tid / 16, 4 consecutive n
  const int b_kp = tid >> 4, b_n = (tid & 15) * 4;
  float4 areg[4];
  uint32_t breg[4];
  auto load_tile = [&](int kt) {
    const int j = kt / kt_per_tap, c0 = (kt - j * kt_per_tap) * TC_BK;
    const bool vec = (c0 + a_c + 4 <= a.C_in) && ((a.ldx & 3) == 0);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int r = a_row + 32 * v;
      const int xr = m0 + r + a.x_row0 + j * a.dil;
      const bool ok = (m0 + r) < a.T_out && xr >= 0 && xr < a.T_in;
      const float* xp = X + (long long)xr * a.ldx + c0 + a_c;
      if (ok && vec && ((reinterpret_cast<uintptr_t>(xp) & 15) == 0)) {
        areg[v] = *reinterpret_cast<const float4*>(xp);
      } else {
        float t4[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) t4[e] = (ok && c0 + a_c + e < a.C_in) ? xp[e] : 0.f;
        areg[v] = make_float4(t4[0], t4[1], t4[2], t4[3]);
      }
    }
    const int kp = (j * c_pairs) + (c0 >> 1) + b_kp;          // pair row of the weight matrix
    const bool kok = (c0 >> 1) + b_kp < c_pairs;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int n = n0 + b_n + v;
      breg[v] = (kok && n < a.N) ? __ldg(reinterpret_cast<const uint32_t*>(wh + (long long)kp * a.N + n)) : 0u;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      __half2* dst = reinterpret_cast<__half2*>(&As[buf][a_row + 32 * v][a_c]);
      dst[0] = __floats2half2_rn(areg[v].x, areg[v].y);
      dst[1] = __floats2half2_rn(areg[v].z, areg[v].w);
    }
#pragma unroll
    for (int v = 0; v < 4; ++v) Bs[buf][b_kp][b_n + v] = breg[v];
  };
  load_tile(0);
  store_tile(0);
  __syncthreads();
  for (int kt = 0; kt < n_kt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_kt) load_tile(kt + 1);              // global loads of the next tile fly during the MMAs
#pragma unroll
    for (int ks = 0; ks < TC_BK; ks += 16) {
      uint32_t af[2][4], bf[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = wm * 32 + i * 16 + g;
        af[i][0] = *reinterpret_cast<const uint32_t*>(&As[buf][r][ks + 2 * t]);
        af[i][1] = *reinterpret_cast<const uint32_t*>(&As[buf][r + 8][ks + 2 * t]);
        af[i][2] = *reinterpret_cast<const uint32_t*>(&As[buf][r][ks + 8 + 2 * t]);
        af[i][3] = *reinterpret_cast<const uint32_t*>(&As[buf][r + 8][ks + 8 + 2 * t]);
      }
#pragma unroll
      for (int jn = 0; jn < 4; ++jn) {
        const int n = wn * 32 + jn * 8 + g;
        bf[jn][0] = Bs[buf][(ks >> 1) + t][n];
        bf[jn][1] = Bs[buf][(ks >> 1) + 4 + t][n];
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) mma_f16_16816(acc[i][jn], af[i][0], af[i][1], af[i][2], af[i][3], bf[jn][0], bf[jn][1]);
    }
    if (kt + 1 < n_kt) store_tile(buf ^ 1);
    __syncthreads();
  }
  float* Y = a.y + (long long)z * a.y_bs;
  const float* R = a.resid ? a.resid + (long long)z * a.r_bs : nullptr;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int jn = 0; jn < 4; ++jn)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int tt = m0 + wm * 32 + i * 16 + g + (r >> 1) * 8;
        const int n = n0 + wn * 32 + jn * 8 + 2 * t + (r & 1);
        if (tt >= a.T_out || n >= a.N) continue;
        float v = acc[i][jn][r];
        if (a.bias) v += __ldg(a.bias + (n % a.bias_mod));
        if (a.act == 1) v = gelu_erf(v);
        else if (a.act == 2) v = v / (1.0f + expf(-v));
        if (a.scale) v *= __ldg(a.scale + n);
        if (R) v += R[(long long)tt * a.ldr + n];
        Y[(long long)tt * a.ldy + n] = v;
      }
}

// The same contraction fed from fp16 ACTIVATIONS (a.x16): the producers whose output is consumed by a contraction only -- the
// SnakeBeta activations in front of every convolution of the decoder blocks -- store fp16 directly, i.e. the rounding the
// staging above applies moves into the producer (same values, same k order, same accumulation: bit-identical results), the
// operand stream halves and both operands travel global -> shared through a 3-stage cp.async pipeline with no register staging.
constexpr int TCH_STAGES = 3;
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst_s, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;   // src-size 0: the 16 destination bytes are zero-filled, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_s), "l"(src), "r"(sz) : "memory");
}
__global__ void __launch_bounds__(TC_THREADS) conv1d_tc16_kernel(const ConvArgs a, const __half* __restrict__ x16, const __half2* __restrict__ wh,
                                                                 int c_pairs) {
  __shared__ __align__(16) __half As[TCH_STAGES][TC_BM][TC_BK + TC_APAD];
  __shared__ __align__(16) uint32_t Bs[TCH_STAGES][TC_BK / 2][TC_BN + TC_BPAD];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const int m0 = blockIdx.y * TC_BM + a.t0, n0 = blockIdx.x * TC_BN, z = blockIdx.z;
  const __half* X = x16 + (long long)z * a.x_bs;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;
  const int kt_per_tap = (a.C_in + TC_BK - 1) / TC_BK;
  const int n_kt = a.k * kt_per_tap;
  // A: 128 rows x 4 chunks of 8 halves; thread -> rows a_row, a_row + 64, chunk a_ch.  B: 16 pair rows x 16 chunks of 4 words.
  const int a_row = tid >> 2, a_ch = (tid & 3) * 8;
  const int b_kp = tid >> 4, b_n = (tid & 15) * 4;
  auto issue = [&](int kt, int buf) {
    const int j = kt / kt_per_tap, c0 = (kt - j * kt_per_tap) * TC_BK;
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const int r = a_row + 64 * v;
      const int xr = m0 + r + a.x_row0 + j * a.dil;
      const bool ok = (m0 + r) < a.T_out && xr >= 0 && xr < a.T_in && (c0 + a_ch + 8) <= a.C_in;
      const __half* src = ok ? X + (long long)xr * a.ldx + c0 + a_ch : X;
      cp_async16_zfill(smem_u32(&As[buf][r][a_ch]), src, ok);
    }
    const bool kok = (c0 >> 1) + b_kp < c_pairs && (n0 + b_n + 4) <= a.N;
    const __half2* wsrc = kok ? wh + (long long)(j * c_pairs + (c0 >> 1) + b_kp) * a.N + n0 + b_n : wh;
    cp_async16_zfill(smem_u32(&Bs[buf][b_kp][b_n]), wsrc, kok);
  };
#pragma unroll
  for (int s = 0; s < TCH_STAGES - 1; ++s) {
    if (s < n_kt) issue(s, s);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int kt = 0; kt < n_kt; ++kt) {
    const int buf = kt % TCH_STAGES;
    asm volatile("cp.async.wait_group %0;" ::"n"(TCH_STAGES - 2) : "memory");
    __syncthreads();                                       // tile kt landed for every thread; tile kt-1's buffer is free
    if (kt + TCH_STAGES - 1 < n_kt) issue(kt + TCH_STAGES - 1, (kt + TCH_STAGES - 1) % TCH_STAGES);
    asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll
    for (int ks = 0; ks < TC_BK; ks += 16) {
      uint32_t af[2][4], bf[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = wm * 32 + i * 16 + g;
        af[i][0] = *reinterpret_cast<const uint32_t*>(&As[buf][r][ks + 2 * t]);
        af[i][1] = *reinterpret_cast<const uint32_t*>(&As[buf][r + 8][ks + 2 * t]);
        af[i][2] = *reinterpret_cast<const uint32_t*>(&As[buf][r][ks + 8 + 2 * t]);
        af[i][3] = *reinterpret_cast<const uint32_t*>(&As[buf][r + 8][ks + 8 + 2 * t]);
      }
#pragma unroll
      for (int jn = 0; jn < 4; ++jn) {
        const int n = wn * 32 + jn * 8 + g;
        bf[jn][0] = Bs[buf][(ks >> 1) + t][n];
        bf[jn][1] = Bs[buf][(ks >> 1) + 4 + t][n];
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) mma_f16_16816(acc[i][jn], af[i][0], af[i][1], af[i][2], af[i][3], bf[jn][0], bf[jn][1]);
    }
  }
  float* Y = a.y + (long long)z * a.y_bs;
  const float* R = a.resid ? a.resid + (long long)z * a.r_bs : nullptr;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int jn = 0; jn < 4; ++jn)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int tt = m0 + wm * 32 + i * 16 + g + (r >> 1) * 8;
        const int n = n0 + wn * 32 + jn * 8 + 2 * t + (r & 1);
        if (tt >= a.T_out || n >= a.N) continue;
        float v = acc[i][jn][r];
        if (a.bias) v += __ldg(a.bias + (n % a.bias_mod));
        if (a.act == 1) v = gelu_erf(v);
        else if (a.act == 2) v = v / (1.0f + expf(-v));
        if (a.scale) v *= __ldg(a.scale + n);
        if (R) v += R[(long long)tt * a.ldr + n];
        Y[(long long)tt * a.ldy + n] = v;
      }
}

// fp32 [k][C_in][N] -> half2 pairs [k][ceil(C_in / 2)][N]
__global__ void pack_weight_pairs_kernel(const float* __restrict__ w, int k, int C_in, int N, __half2* __restrict__ out) {
  const int cp = (C_in + 1) >> 1;
  const long long total = (long long)k * cp * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i % N);
    const long long r = i / N;
    const int p = (int)(r % cp), j = (int)(r / cp);
    const int c = 2 * p;
    const float lo = w[((long long)j * C_in + c) * N + n];
    const float hi = c + 1 < C_in ? w[((long long)j * C_in + c + 1) * N + n] : 0.f;
    out[i] = __floats2half2_rn(lo, hi);
  }
}

// ------------------------------------------------------------------------------------------------ small kernels
// x[b * T + t, :] = mean_q E[q * cb + codes_b[t][q], :]   (one code pointer per sequence of the batch)
struct CodePtrs { const int* p[CODEC_MAX_BATCH]; };
__global__ void code_embed_mean_kernel(CodePtrs cp, int T, int Q, int cb, const float* __restrict__ E, int H, float* __restrict__ x) {
  const int b = blockIdx.x / T, t = blockIdx.x % T;
  const int* codes = cp.p[b];
  const float inv = 1.0f / (float)Q;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < Q; ++q) s += E[((long long)q * cb + codes[t * Q + q]) * H + i];
    x[(long long)blockIdx.x * H + i] = s * inv;
  }
}

// y = w * x * rsqrt(mean(x^2) + eps), one warp per row
__global__ void rmsnorm_rows_f32_kernel(const float* __restrict__ x, const float* __restrict__ w, float eps, int rows, int d,
                                        float* __restrict__ y) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (long long)row * d;
  float ss = 0.f;
  for (int i = lane; i < d; i += 32) ss = fmaf(xr[i], xr[i], ss);
  ss = warp_sum(ss);
  const float r = 1.0f / sqrtf(ss / (float)d + eps);
  for (int i = lane; i < d; i += 32) y[(long long)row * d + i] = w[i] * (xr[i] * r);
}

// RoPE (rotate_half pairs (j, j + hd/2)) on q and k in place; qkv [T, (H + 2 KV) * hd], position = row index
__global__ void rope_rows_f32_kernel(float* __restrict__ qkv, int T, int n_rot_heads, int hd, int ld, float theta) {
  const int t = blockIdx.x % T;              // rows of a batch are [b * T + t]: the position restarts with every sequence
  qkv += (long long)(blockIdx.x - t) * ld;
  const int half = hd >> 1;
  for (int i = threadIdx.x; i < n_rot_heads * half; i += blockDim.x) {
    const int h = i / half, j = i % half;
    const float inv = 1.0f / powf(theta, (float)(2 * j) / (float)hd);
    const float ang = (float)t * inv;
    const float c = cosf(ang), s = sinf(ang);
    float* p = qkv + (long long)t * ld + h * hd;
    const float a = p[j], b = p[j + half];
    p[j] = a * c - b * s;
    p[j + half] = b * c + a * s;
  }
}

// causal sliding-window attention, one warp per (query t, head h); keys t - W + 1 .. t; fp32 softmax
__global__ void swa_attention_f32_kernel(const float* __restrict__ qkv, int B, int T, int H, int KV, int hd, int W, float* __restrict__ o) {
  extern __shared__ float sm[];   // per warp: q[hd] + p[W]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int item = blockIdx.x * nw + warp;
  if (item >= B * T * H) return;
  const int bt = item / H, h = item % H, g = H / KV;
  const int b = bt / T, t = bt % T;          // sequence b of the batch: keys never cross a sequence boundary
  const int ld = (H + 2 * KV) * hd;
  qkv += (long long)b * T * ld;
  o += (long long)b * T * (H * hd);
  float* qs = sm + (size_t)warp * (hd + W);
  float* ps = qs + hd;
  const float* q = qkv + (long long)t * ld + h * hd;
  for (int i = lane; i < hd; i += 32) qs[i] = q[i];
  __syncwarp();
  const int lo = max(0, t - W + 1), n = t - lo + 1;
  const float scale = rsqrtf((float)hd);
  float mx = -INFINITY;
  for (int s = lane; s < n; s += 32) {
    const float* k = qkv + (long long)(lo + s) * ld + (H + h / g) * hd;
    float d = 0.f;
    for (int i = 0; i < hd; ++i) d = fmaf(qs[i], k[i], d);
    d *= scale;
    ps[s] = d;
    mx = fmaxf(mx, d);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int s = lane; s < n; s += 32) { const float e = expf(ps[s] - mx); ps[s] = e; sum += e; }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.0f / sum;
  for (int i = lane; i < hd; i += 32) {
    float acc = 0.f;
    for (int s = 0; s < n; ++s) acc = fmaf(ps[s], qkv[(long long)(lo + s) * ld + (H + KV + h / g) * hd + i], acc);
    o[(long long)t * (H * hd) + h * hd + i] = acc * inv;
  }
}

// h = silu(g) * u ; gu [T, 2 * inter] as [gate | up]
__global__ void silu_mul_kernel(const float* __restrict__ gu, int inter, long long n, float* __restrict__ h) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long t = i / inter, c = i % inter;
  const float g = gu[t * 2 * inter + c], u = gu[t * 2 * inter + inter + c];
  h[i] = (g / (1.0f + expf(-g))) * u;
}

// SnakeBeta: y = x + ib[c] * sin(x * a[c])^2 with a = exp(alpha), ib = 1 / (exp(beta) + 1e-9) (precomputed at bind)
// rows [first, len) of each of the B sequences (sequence stride len * C)
__global__ void snake_beta_kernel(const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ ib, int C,
                                  int len, int first, long long n_per_seq, long long n, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long b = i / n_per_seq, r = i - b * n_per_seq;
  const long long idx = b * (long long)len * C + (long long)first * C + r;
  const int c = (int)(r % C);
  const float v = x[idx], s = sinf(v * a[c]);
  y[idx] = v + ib[c] * (s * s);
}

// the same, stored as fp16 for a tensor-core contraction (conv1d_tc16_kernel); 4 channels per thread (C % 4 == 0)
__global__ void snake_beta_h_kernel(const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ ib, int C,
                                    int len, int first, long long n_per_seq, long long n, __half* __restrict__ y) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  const long long b = i / n_per_seq, r = i - b * n_per_seq;
  const long long idx = b * (long long)len * C + (long long)first * C + r;
  const int c = (int)(r % C);
  const float4 v = *reinterpret_cast<const float4*>(x + idx);
  const float4 av = *reinterpret_cast<const float4*>(a + c), bv = *reinterpret_cast<const float4*>(ib + c);
  const float s0 = sinf(v.x * av.x), s1 = sinf(v.y * av.y), s2 = sinf(v.z * av.z), s3 = sinf(v.w * av.w);
  __half2* dst = reinterpret_cast<__half2*>(y + idx);
  dst[0] = __floats2half2_rn(v.x + bv.x * (s0 * s0), v.y + bv.y * (s1 * s1));
  dst[1] = __floats2half2_rn(v.z + bv.z * (s2 * s2), v.w + bv.w * (s3 * s3));
}

// ConvNeXt front: depthwise causal conv 7 + LayerNorm(eps) over channels; one CTA per time step
__global__ void dwconv7_ln_kernel(const float* __restrict__ x, int T, int first, int C, const float* __restrict__ wd, const float* __restrict__ bd,
                                  const float* __restrict__ lw, const float* __restrict__ lb, float eps, float* __restrict__ y) {
  extern __shared__ float hs[];   // [C]
  __shared__ float red[2][32];
  // grid = B x (T - first) rows; the causal window restarts with every sequence of the batch
  const int per = T - first, b = blockIdx.x / per, t = first + blockIdx.x % per;
  x += (long long)b * T * C;
  y += (long long)b * T * C;
  float s1 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v = bd[c];
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const int r = t - 6 + j;
      if (r >= 0) v = fmaf(x[(long long)r * C + c], wd[c * 7 + j], v);
    }
    hs[c] = v;
    s1 += v;
  }
  s1 = warp_sum(s1);
  if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = s1;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[0][w];
  const float mean = tot / (float)C;
  float s2 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float dlt = hs[c] - mean; s2 = fmaf(dlt, dlt, s2); }
  s2 = warp_sum(s2);
  if ((threadIdx.x & 31) == 0) red[1][threadIdx.x >> 5] = s2;
  __syncthreads();
  float var = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) var += red[1][w];
  const float rstd = 1.0f / sqrtf(var / (float)C + eps);
  for (int c = threadIdx.x; c < C; c += blockDim.x) y[(long long)t * C + c] = (hs[c] - mean) * rstd * lw[c] + lb[c];
}

// wav[b][i] = clamp(x[b][skip + i], -1, 1)
__global__ void clamp_out_kernel(const float* __restrict__ x, long long x_bs, int skip, int n, float* __restrict__ wav, long long wav_bs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) wav[(long long)blockIdx.y * wav_bs + i] = fminf(1.0f, fmaxf(-1.0f, x[(long long)blockIdx.y * x_bs + skip + i]));
}

__global__ void exp_prep_kernel(float* a, float* b, int n) {   // alpha -> exp(alpha); beta -> 1 / (exp(beta) + 1e-9)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { a[i] = expf(a[i]); b[i] = 1.0f / (expf(b[i]) + 1e-9f); }
}

inline float src_f32(const void* data, int64_t i, int dtype) {
  if (dtype == S2S_F32) return reinterpret_cast<const float*>(data)[i];
  uint16_t u = reinterpret_cast<const uint16_t*>(data)[i];
  if (dtype == S2S_BF16) { uint32_t w = (uint32_t)u << 16; float f; memcpy(&f, &w, 4); return f; }
  __half h; memcpy(&h, &u, 2); return __half2float(h);
}

enum CSlotKind { C_PLAIN = 0, C_LINEAR = 1 /* [N,K] -> [K][N] */, C_CONV = 2 /* [O,C,k] -> [k][C][O] */,
                 C_TCONV = 3 /* [C,O,k] -> taps x [C][s*O] */ };
struct CSlot {
  float* dst = nullptr;
  int64_t n = 0;
  int kind = C_PLAIN;
  int d0 = 0, d1 = 0, d2 = 0, stride = 0;   // source dims
  bool bound = false;
  float rnd_scale = 0.02f, rnd_offset = 0.f;
};

}  // namespace

int conv1d_tc_launch(const ConvArgs& a, const void* w_pairs, cudaStream_t st) {
  if (a.T_out - a.t0 <= 0 || a.N <= 0) return S2S_OK;
  const int batch = a.batch > 0 ? a.batch : 1;
  dim3 grid((a.N + TC_BN - 1) / TC_BN, (a.T_out - a.t0 + TC_BM - 1) / TC_BM, batch);
  if (a.x16) {
    S2S_REQUIRE(a.C_in % 8 == 0 && a.N % 4 == 0 && a.ldx % 8 == 0 && a.x_bs % 8 == 0, "conv1d_tc16: C_in %d / N %d / ldx %lld not 16-byte tileable",
                a.C_in, a.N, a.ldx);
    conv1d_tc16_kernel<<<grid, TC_THREADS, 0, st>>>(a, reinterpret_cast<const __half*>(a.x16), reinterpret_cast<const __half2*>(w_pairs),
                                                    (a.C_in + 1) >> 1);
    S2S_LAUNCH_CHECK();
    return S2S_OK;
  }
  conv1d_tc_kernel<<<grid, TC_THREADS, 0, st>>>(a, reinterpret_cast<const __half2*>(w_pairs), (a.C_in + 1) >> 1);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

int conv1d_f32_launch(const ConvArgs& a, cudaStream_t st) {
  if (a.T_out - a.t0 <= 0 || a.N <= 0) return S2S_OK;
  const int batch = a.batch > 0 ? a.batch : 1;
  const int mt = (a.T_out - a.t0 + CV_BM - 1) / CV_BM;
  // few time tiles (transformer / first decoder stages): narrower n tiles put more SMs on the weight stream
  static const int num_sms = [] {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 0;
    return n;
  }();
  if ((long long)mt * ((a.N + 63) / 64) * batch < num_sms) {
    dim3 grid((a.N + 31) / 32, mt, batch);
    conv1d_f32_kernel<32><<<grid, CV_THREADS, 0, st>>>(a);
  } else {
    dim3 grid((a.N + 63) / 64, mt, batch);
    conv1d_f32_kernel<64><<<grid, CV_THREADS, 0, st>>>(a);
  }
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

// ------------------------------------------------------------------------------------------------ the model
struct CodecLayer {   // transformer layer
  float *w_qkv, *w_o, *w_gu, *w_down, *n1, *n2, *ls_attn, *ls_mlp;
};
struct CodecConvNeXt { float *up_w, *up_b, *dw_w, *dw_b, *ln_w, *ln_b, *pw1_w, *pw1_b, *pw2_w, *pw2_b, *gamma; };
struct CodecResUnit { float *a1, *b1, *c1_w, *c1_b, *a2, *b2, *c2_w, *c2_b; };
struct CodecBlock { float *a0, *b0, *tc_w, *tc_b; CodecResUnit u[3]; int cin, cout, rate; };

struct s2s_codec {
  s2s_ctx* ctx = nullptr;
  s2s_codec_config cfg{};
  bool finalized = false;
  std::vector<void*> allocs;
  std::unordered_map<std::string, CSlot> slots;
  std::vector<std::pair<float*, float*>> snake_pairs;   // (alpha, beta) buffers and their length, transformed at finalize
  std::vector<int> snake_len;
  float* embed = nullptr;
  std::vector<CodecLayer> layers;
  float* norm_f = nullptr;
  std::vector<CodecConvNeXt> ups;
  float *d0_w = nullptr, *d0_b = nullptr;
  std::vector<CodecBlock> blocks;
  float *fa = nullptr, *fb = nullptr, *f_w = nullptr, *f_b = nullptr;
  // workspace
  float *x = nullptr, *xn = nullptr, *qkv = nullptr, *att = nullptr, *gu = nullptr, *hmid = nullptr;
  float *bufX = nullptr, *bufA = nullptr, *bufH = nullptr;
  size_t buf_elems = 0;
  int total_up = 1;
  // tensor-core path: fp16 k-pair copies of the contraction weights, keyed by the fp32 matrix they were packed from
  struct TcW { int k, C_in, N; void* packed; };
  std::unordered_map<const float*, TcW> tc_w;
};

namespace {

void tc_register(CodecDecoder* m, const float* w, int k, int C_in, int N) { m->tc_w[w] = CodecDecoder::TcW{k, C_in, N, nullptr}; }

int calloc_f(CodecDecoder* m, float** out, size_t n) {
  void* p = nullptr;
  S2S_CHECK_CUDA(cudaMalloc(&p, (n ? n : 4) * 4));
  S2S_CHECK_CUDA(cudaMemset(p, 0, (n ? n : 4) * 4));
  m->allocs.push_back(p);
  *out = reinterpret_cast<float*>(p);
  return S2S_OK;
}

int cslot(CodecDecoder* m, const std::string& name, float** out, int kind, int d0, int d1, int d2, int stride, float rs,
          float ro = 0.f) {
  CSlot s;
  s.kind = kind; s.d0 = d0; s.d1 = d1; s.d2 = d2; s.stride = stride; s.rnd_scale = rs; s.rnd_offset = ro;
  s.n = (int64_t)d0 * (d1 ? d1 : 1) * (d2 ? d2 : 1);
  S2S_CHECK(calloc_f(m, &s.dst, (size_t)s.n));
  *out = s.dst;
  m->slots[name] = s;
  return S2S_OK;
}

// sequence lengths along the decoder for T frames
void codec_lengths(const s2s_codec_config& c, int T, std::vector<int>& L) {
  int len = T;
  for (int i = 0; i < c.n_upsampling_ratios; ++i) len *= c.upsampling_ratios[i];
  L.clear();
  L.push_back(len);
  for (int i = 0; i < c.n_upsample_rates; ++i) { len = (len - 1) * c.upsample_rates[i]; L.push_back(len); }
}

int build(CodecDecoder* m) {
  const auto& c = m->cfg;
  const int H = c.hidden, hd = H / c.heads, qd = c.heads * hd, kvd = c.kv_heads * hd, I = c.inter;
  float* dummy;
  S2S_CHECK(cslot(m, "code_embedding.weight", &m->embed, C_PLAIN, c.codebook_size * c.quantizers, H, 0, 0, 1.0f));
  m->layers.resize(c.layers);
  const float sh = 1.0f / sqrtf((float)H);
  for (int l = 0; l < c.layers; ++l) {
    const std::string p = "pre_transformer.layers." + std::to_string(l) + ".";
    CodecLayer& L = m->layers[l];
    // q, k, v share one [H][qd + 2 kvd] matrix; gate and up one [H][2 I] matrix (column blocks)
    S2S_CHECK(calloc_f(m, &L.w_qkv, (size_t)H * (qd + 2 * kvd)));
    S2S_CHECK(calloc_f(m, &L.w_gu, (size_t)H * 2 * I));
    auto sub = [&](const std::string& name, float* base, int N_total, int col0, int N, int K, float rs) {
      CSlot s; s.dst = base; s.kind = C_LINEAR; s.d0 = N; s.d1 = K; s.d2 = N_total; s.stride = col0; s.n = (int64_t)N * K; s.rnd_scale = rs;
      m->slots[name] = s;
    };
    sub(p + "self_attn.q_proj.weight", L.w_qkv, qd + 2 * kvd, 0, qd, H, sh);
    sub(p + "self_attn.k_proj.weight", L.w_qkv, qd + 2 * kvd, qd, kvd, H, sh);
    sub(p + "self_attn.v_proj.weight", L.w_qkv, qd + 2 * kvd, qd + kvd, kvd, H, sh);
    sub(p + "mlp.gate_proj.weight", L.w_gu, 2 * I, 0, I, H, sh);
    sub(p + "mlp.up_proj.weight", L.w_gu, 2 * I, I, I, H, sh);
    S2S_CHECK(cslot(m, p + "self_attn.o_proj.weight", &L.w_o, C_LINEAR, H, qd, 0, 0, sh));
    S2S_CHECK(cslot(m, p + "mlp.down_proj.weight", &L.w_down, C_LINEAR, H, I, 0, 0, 1.0f / sqrtf((float)I)));
    tc_register(m, L.w_qkv, 1, H, qd + 2 * kvd); tc_register(m, L.w_gu, 1, H, 2 * I);
    tc_register(m, L.w_o, 1, qd, H); tc_register(m, L.w_down, 1, I, H);
    S2S_CHECK(cslot(m, p + "input_layernorm.weight", &L.n1, C_PLAIN, H, 0, 0, 0, 0.1f, 1.0f));
    S2S_CHECK(cslot(m, p + "post_attention_layernorm.weight", &L.n2, C_PLAIN, H, 0, 0, 0, 0.1f, 1.0f));
    S2S_CHECK(cslot(m, p + "self_attn_layer_scale.scale", &L.ls_attn, C_PLAIN, H, 0, 0, 0, 0.1f, 0.5f));
    S2S_CHECK(cslot(m, p + "mlp_layer_scale.scale", &L.ls_mlp, C_PLAIN, H, 0, 0, 0, 0.1f, 0.5f));
  }
  S2S_CHECK(cslot(m, "pre_transformer.norm.weight", &m->norm_f, C_PLAIN, H, 0, 0, 0, 0.1f, 1.0f));
  m->ups.resize(c.n_upsampling_ratios);
  m->total_up = 1;
  for (int i = 0; i < c.n_upsampling_ratios; ++i) {
    const int f = c.upsampling_ratios[i];
    m->total_up *= f;
    const std::string p = "upsample." + std::to_string(i) + ".";
    CodecConvNeXt& U = m->ups[i];
    S2S_CHECK(cslot(m, p + "0.conv.weight", &U.up_w, C_TCONV, H, H, f, f, sh));
    S2S_CHECK(cslot(m, p + "0.conv.bias", &U.up_b, C_PLAIN, H, 0, 0, 0, 0.02f));
    S2S_CHECK(cslot(m, p + "1.dwconv.conv.weight", &U.dw_w, C_PLAIN, H, 7, 0, 0, 0.378f));
    S2S_CHECK(cslot(m, p + "1.dwconv.conv.bias", &U.dw_b, C_PLAIN, H, 0, 0, 0, 0.02f));
    S2S_CHECK(cslot(m, p + "1.norm.weight", &U.ln_w, C_PLAIN, H, 0, 0, 0, 0.1f, 1.0f));
    S2S_CHECK(cslot(m, p + "1.norm.bias", &U.ln_b, C_PLAIN, H, 0, 0, 0, 0.05f));
    S2S_CHECK(cslot(m, p + "1.pwconv1.weight", &U.pw1_w, C_LINEAR, 4 * H, H, 0, 0, sh));
    S2S_CHECK(cslot(m, p + "1.pwconv1.bias", &U.pw1_b, C_PLAIN, 4 * H, 0, 0, 0, 0.02f));
    S2S_CHECK(cslot(m, p + "1.pwconv2.weight", &U.pw2_w, C_LINEAR, H, 4 * H, 0, 0, 0.5f * sh));
    S2S_CHECK(cslot(m, p + "1.pwconv2.bias", &U.pw2_b, C_PLAIN, H, 0, 0, 0, 0.02f));
    S2S_CHECK(cslot(m, p + "1.gamma", &U.gamma, C_PLAIN, H, 0, 0, 0, 0.05f, 0.3f));
    tc_register(m, U.up_w, 1, H, f * H); tc_register(m, U.pw1_w, 1, H, 4 * H); tc_register(m, U.pw2_w, 1, 4 * H, H);
  }
  const int D = c.decoder_dim;
  S2S_CHECK(cslot(m, "decoder.0.conv.weight", &m->d0_w, C_CONV, D, H, 7, 0, 1.0f / sqrtf(7.0f * H)));
  S2S_CHECK(cslot(m, "decoder.0.conv.bias", &m->d0_b, C_PLAIN, D, 0, 0, 0, 0.02f));
  tc_register(m, m->d0_w, 7, H, D);
  m->blocks.resize(c.n_upsample_rates);
  auto snake = [&](const std::string& pa, const std::string& pb, float** a, float** b, int n) -> int {
    S2S_CHECK(cslot(m, pa, a, C_PLAIN, n, 0, 0, 0, 0.2f));
    S2S_CHECK(cslot(m, pb, b, C_PLAIN, n, 0, 0, 0, 0.2f));
    m->snake_pairs.push_back({*a, *b});
    m->snake_len.push_back(n);
    return S2S_OK;
  };
  for (int i = 0; i < c.n_upsample_rates; ++i) {
    CodecBlock& B = m->blocks[i];
    B.cin = D >> i; B.cout = D >> (i + 1); B.rate = c.upsample_rates[i];
    m->total_up *= B.rate;
    const std::string p = "decoder." + std::to_string(i + 1) + ".block.";
    S2S_CHECK(snake(p + "0.alpha", p + "0.beta", &B.a0, &B.b0, B.cin));
    S2S_CHECK(cslot(m, p + "1.conv.weight", &B.tc_w, C_TCONV, B.cin, B.cout, 2 * B.rate, B.rate, 1.0f / sqrtf(2.0f * B.cin)));
    S2S_CHECK(cslot(m, p + "1.conv.bias", &B.tc_b, C_PLAIN, B.cout, 0, 0, 0, 0.02f));
    tc_register(m, B.tc_w, 2, B.cin, B.rate * B.cout);
    for (int u = 0; u < 3; ++u) {
      const std::string q = p + std::to_string(u + 2) + ".";
      CodecResUnit& R = B.u[u];
      S2S_CHECK(snake(q + "act1.alpha", q + "act1.beta", &R.a1, &R.b1, B.cout));
      S2S_CHECK(cslot(m, q + "conv1.conv.weight", &R.c1_w, C_CONV, B.cout, B.cout, 7, 0, 1.0f / sqrtf(7.0f * B.cout)));
      S2S_CHECK(cslot(m, q + "conv1.conv.bias", &R.c1_b, C_PLAIN, B.cout, 0, 0, 0, 0.02f));
      S2S_CHECK(snake(q + "act2.alpha", q + "act2.beta", &R.a2, &R.b2, B.cout));
      S2S_CHECK(cslot(m, q + "conv2.conv.weight", &R.c2_w, C_CONV, B.cout, B.cout, 1, 0, 1.0f / sqrtf((float)B.cout)));
      S2S_CHECK(cslot(m, q + "conv2.conv.bias", &R.c2_b, C_PLAIN, B.cout, 0, 0, 0, 0.02f));
      tc_register(m, R.c1_w, 7, B.cout, B.cout); tc_register(m, R.c2_w, 1, B.cout, B.cout);
    }
  }
  const int n = c.n_upsample_rates, cl = D >> n;
  S2S_CHECK(snake("decoder." + std::to_string(n + 1) + ".alpha", "decoder." + std::to_string(n + 1) + ".beta", &m->fa, &m->fb, cl));
  S2S_CHECK(cslot(m, "decoder." + std::to_string(n + 2) + ".conv.weight", &m->f_w, C_CONV, 1, cl, 7, 0, 0.5f / sqrtf(7.0f * cl)));
  S2S_CHECK(cslot(m, "decoder." + std::to_string(n + 2) + ".conv.bias", &m->f_b, C_PLAIN, 1, 0, 0, 0, 0.02f));
  (void)dummy;
  // workspace for max_batch sequences of max_frames
  const int T = c.max_frames * (c.max_batch > 0 ? c.max_batch : 1);
  std::vector<int> L;
  codec_lengths(c, c.max_frames, L);
  const size_t nb = (size_t)(c.max_batch > 0 ? c.max_batch : 1);
  for (int& v : L) v = (int)((size_t)v * nb);
  size_t mx = (size_t)L[0] * std::max(4 * H, D);
  for (int i = 0; i < c.n_upsample_rates; ++i) mx = std::max(mx, (size_t)L[i + 1] * (size_t)(D >> (i + 1)));
  mx = std::max(mx, (size_t)L[0] * (size_t)D);
  m->buf_elems = mx;
  S2S_CHECK(calloc_f(m, &m->bufX, mx));
  S2S_CHECK(calloc_f(m, &m->bufA, mx));
  S2S_CHECK(calloc_f(m, &m->bufH, mx));
  S2S_CHECK(calloc_f(m, &m->x, (size_t)T * H));
  S2S_CHECK(calloc_f(m, &m->xn, (size_t)T * H));
  S2S_CHECK(calloc_f(m, &m->qkv, (size_t)T * (qd + 2 * kvd)));
  S2S_CHECK(calloc_f(m, &m->att, (size_t)T * qd));
  S2S_CHECK(calloc_f(m, &m->gu, (size_t)T * 2 * I));
  S2S_CHECK(calloc_f(m, &m->hmid, (size_t)T * I));
  return S2S_OK;
}

// one contraction: tensor cores (fp16 operands) unless the model runs in parity mode or the shape has no packed weights
int contract(CodecDecoder* m, const ConvArgs& a, cudaStream_t st) {
  if (m->cfg.precision != 0) {
    auto it = m->tc_w.find(a.w);
    if (it != m->tc_w.end() && it->second.packed) return conv1d_tc_launch(a, it->second.packed, st);
  }
  return conv1d_f32_launch(a, st);
}

ConvArgs linear_args(const float* x, int T, int K, const float* w, int N, float* y) {
  ConvArgs a{};
  a.x = x; a.ldx = K; a.T_in = T; a.x_row0 = 0; a.w = w; a.k = 1; a.dil = 1; a.C_in = K; a.N = N; a.bias = nullptr; a.bias_mod = N;
  a.y = y; a.ldy = N; a.T_out = T; a.batch = 1;
  return a;
}
ConvArgs causal_conv_args(const float* x, int T, int C_in, const float* w, const float* b, int k, int dil, int C_out, float* y) {
  ConvArgs a{};
  a.x = x; a.ldx = C_in; a.T_in = T; a.x_row0 = -(k - 1) * dil; a.w = w; a.k = k; a.dil = dil; a.C_in = C_in; a.N = C_out;
  a.bias = b; a.bias_mod = C_out; a.y = y; a.ldy = C_out; a.T_out = T; a.batch = 1;
  return a;
}

// SnakeBeta whose only consumer is a tensor-core contraction: fp16 output (conv1d_tc16_kernel reads it with cp.async)
int snake_launch_h(const float* x, const float* a, const float* ib, int C, int B, int len, int first, void* y16, cudaStream_t st) {
  const long long per = (long long)(len - first) * C, n = per * B;
  if (n <= 0) return S2S_OK;
  snake_beta_h_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>(x, a, ib, C, len, first, per, n, reinterpret_cast<__half*>(y16));
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}
// may the contraction with weights w (C_in = C, N outputs) take an fp16 operand?  (tensor-core mode, packed weights, 16-byte tiles)
bool fp16_operand_ok(const CodecDecoder* m, const float* w, int C, int N) {
  if (m->cfg.precision == 0 || C % 8 != 0 || N % 4 != 0) return false;
  if (const char* e = getenv("S2S_CODEC_FP16_OPERANDS")) { if (e[0] == '0') return false; }   // A/B switch (tests: bit-identical)
  auto it = m->tc_w.find(w);
  return it != m->tc_w.end() && it->second.packed != nullptr;
}

int snake_launch(const float* x, const float* a, const float* ib, int C, int B, int len, int first, float* y, cudaStream_t st) {
  const long long per = (long long)(len - first) * C, n = per * B;
  if (n <= 0) return S2S_OK;
  snake_beta_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, a, ib, C, len, first, per, n, y);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

}  // namespace

int codec_total_upsample(const CodecDecoder* m) { return m->total_up; }
int codec_samples_for(const CodecDecoder* m, int T) {
  std::vector<int> L;
  codec_lengths(m->cfg, T, L);
  return L.back();
}

int codec_create(s2s_ctx* ctx, const s2s_codec_config* cfg, CodecDecoder** out) {
  S2S_REQUIRE(ctx && cfg && out, "codec_create: null argument");
  S2S_REQUIRE(cfg->hidden % cfg->heads == 0 && cfg->heads % cfg->kv_heads == 0, "codec: bad head geometry");
  S2S_REQUIRE(cfg->n_upsample_rates >= 1 && cfg->n_upsample_rates <= 8 && cfg->n_upsampling_ratios >= 0 && cfg->n_upsampling_ratios <= 4,
              "codec: bad upsampling lists");
  S2S_REQUIRE(cfg->max_frames >= 1 && cfg->layers >= 0 && cfg->sliding_window >= 1, "codec: bad capacity");
  S2S_REQUIRE((cfg->decoder_dim >> cfg->n_upsample_rates) >= 1, "codec: decoder_dim too small for %d blocks", cfg->n_upsample_rates);
  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  CodecDecoder* m = new s2s_codec();
  m->ctx = ctx;
  m->cfg = *cfg;
  const int r = build(m);
  if (r != S2S_OK) { codec_destroy(m); return r; }
  *out = m;
  return S2S_OK;
}

int codec_destroy(CodecDecoder* m) {
  if (!m) return S2S_OK;
  for (void* p : m->allocs) cudaFree(p);
  delete m;
  return S2S_OK;
}

int codec_bind_tensor(CodecDecoder* m, const char* name, const void* data_h, const int64_t* shape, int ndim, int dtype) {
  S2S_REQUIRE(m && name && data_h && shape, "codec bind_tensor: null argument");
  auto it = m->slots.find(name);
  if (it == m->slots.end()) { s2s_set_error("codec bind_tensor: unknown tensor '%s'", name); return S2S_ERR_NOT_FOUND; }
  CSlot& s = it->second;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  S2S_REQUIRE(n == s.n, "codec bind_tensor: '%s' has %lld elements, expected %lld", name, (long long)n, (long long)s.n);
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  if (s.kind == C_LINEAR && s.d2 > 0) {
    // column block [col0, col0 + N) of a shared [K][N_total] matrix: one strided 2-D copy
    const int N = s.d0, K = s.d1, Nt = s.d2, col0 = s.stride;
    std::vector<float> tmp((size_t)K * N);
    for (int nn = 0; nn < N; ++nn)
      for (int k = 0; k < K; ++k) tmp[(size_t)k * N + nn] = src_f32(data_h, (int64_t)nn * K + k, dtype);
    S2S_CHECK_CUDA(cudaMemcpy2D(s.dst + col0, (size_t)Nt * 4, tmp.data(), (size_t)N * 4, (size_t)N * 4, K, cudaMemcpyHostToDevice));
    s.bound = true;
    return S2S_OK;
  }
  std::vector<float> tmp((size_t)n);
  if (s.kind == C_LINEAR) {
    const int N = s.d0, K = s.d1;
    for (int nn = 0; nn < N; ++nn)
      for (int k = 0; k < K; ++k) tmp[(size_t)k * N + nn] = src_f32(data_h, (int64_t)nn * K + k, dtype);
  } else if (s.kind == C_CONV) {
    const int O = s.d0, C = s.d1, k = s.d2;
    for (int o = 0; o < O; ++o)
      for (int c = 0; c < C; ++c)
        for (int j = 0; j < k; ++j) tmp[((size_t)j * C + c) * O + o] = src_f32(data_h, ((int64_t)o * C + c) * k + j, dtype);
  } else if (s.kind == C_TCONV) {
    // [C, O, k] with k = s or 2 s.  k = s: one tap, W'[c][r * O + o] = W[c][o][r].
    // k = 2 s: tap 0 multiplies X[t0 - 1] -> W[c][o][r + s]; tap 1 multiplies X[t0] -> W[c][o][r].
    const int C = s.d0, O = s.d1, k = s.d2, st = s.stride, taps = k / st;
    for (int c = 0; c < C; ++c)
      for (int o = 0; o < O; ++o)
        for (int r = 0; r < st; ++r) {
          if (taps == 1) tmp[(size_t)c * st * O + (size_t)r * O + o] = src_f32(data_h, ((int64_t)c * O + o) * k + r, dtype);
          else {
            tmp[((size_t)0 * C + c) * st * O + (size_t)r * O + o] = src_f32(data_h, ((int64_t)c * O + o) * k + r + st, dtype);
            tmp[((size_t)1 * C + c) * st * O + (size_t)r * O + o] = src_f32(data_h, ((int64_t)c * O + o) * k + r, dtype);
          }
        }
  } else {
    for (int64_t i = 0; i < n; ++i) tmp[(size_t)i] = src_f32(data_h, i, dtype);
  }
  S2S_CHECK_CUDA(cudaMemcpy(s.dst, tmp.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  s.bound = true;
  return S2S_OK;
}

int codec_init_random(CodecDecoder* m, uint64_t seed) {
  S2S_REQUIRE(m, "codec init_random: null model");
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  for (auto& kv : m->slots) {
    CSlot& s = kv.second;
    uint64_t hsh = 1469598103934665603ull;
    for (char ch : kv.first) hsh = (hsh ^ (uint64_t)(unsigned char)ch) * 1099511628211ull;
    if (s.kind == C_LINEAR && s.d2 > 0) {
      // column block of a shared matrix: fill row by row
      std::vector<float> tmp((size_t)s.d0 * s.d1);
      uint64_t st = seed ^ hsh;
      for (auto& v : tmp) { st = st * 6364136223846793005ull + 1442695040888963407ull; v = s.rnd_scale * (((st >> 40) & 0xffff) / 32768.0f - 1.0f); }
      S2S_CHECK_CUDA(cudaMemcpy2D(s.dst + s.stride, (size_t)s.d2 * 4, tmp.data(), (size_t)s.d0 * 4, (size_t)s.d0 * 4, s.d1, cudaMemcpyHostToDevice));
    } else {
      S2S_CHECK(fill_random_launch(s.dst, s.n, S2S_F32, s.rnd_scale, s.rnd_offset, seed ^ hsh, 0));
    }
    s.bound = true;
  }
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  return S2S_OK;
}

int codec_finalize(CodecDecoder* m) {
  S2S_REQUIRE(m, "codec finalize: null model");
  for (auto& kv : m->slots)
    if (!kv.second.bound) { s2s_set_error("codec finalize: tensor '%s' was never bound", kv.first.c_str()); return S2S_ERR_INVALID; }
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  if (!m->finalized)   // SnakeBeta parameters -> (exp(alpha), 1 / (exp(beta) + 1e-9)), once
    for (size_t i = 0; i < m->snake_pairs.size(); ++i) {
      exp_prep_kernel<<<(m->snake_len[i] + 255) / 256, 256>>>(m->snake_pairs[i].first, m->snake_pairs[i].second, m->snake_len[i]);
      S2S_LAUNCH_CHECK();
    }
  // fp16 k-pair copies for the tensor-core contraction (rebuilt on every (re)load)
  for (auto& kv : m->tc_w) {
    CodecDecoder::TcW& t = kv.second;
    const size_t words = (size_t)t.k * ((t.C_in + 1) / 2) * t.N;
    if (!t.packed) {
      S2S_CHECK_CUDA(cudaMalloc(&t.packed, words * 4));
      m->allocs.push_back(t.packed);
    }
    pack_weight_pairs_kernel<<<(unsigned)std::min<size_t>((words + 255) / 256, 4096), 256>>>(kv.first, t.k, t.C_in, t.N,
                                                                                               reinterpret_cast<__half2*>(t.packed));
    S2S_LAUNCH_CHECK();
  }
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  m->finalized = true;
  return S2S_OK;
}

// B sequences of the same shape (T frames, ctx_frames of history) through ONE launch sequence: the linear layers see
// B * T rows, the causal convolutions run one sequence per blockIdx.z.  codes_d[b]: [T][Q]; wav_out_d + b * wav_stride.
int codec_decode_batch(CodecDecoder* m, const int32_t* const* codes_d, int B, int T, int ctx_frames, float* wav_out_d,
                       long long wav_stride, int32_t* n_out_h, float* hidden_out_d, cudaStream_t st) {
  S2S_REQUIRE(m && m->finalized && codes_d && wav_out_d, "codec decode: null argument / not finalized");
  const auto& c = m->cfg;
  const int maxB = c.max_batch > 0 ? c.max_batch : 1;
  S2S_REQUIRE(B >= 1 && B <= maxB && B <= CODEC_MAX_BATCH, "codec decode: batch %d outside [1,%d]", B, std::min(maxB, CODEC_MAX_BATCH));
  S2S_REQUIRE(T >= 1 && T <= c.max_frames, "codec decode: T=%d outside [1,%d]", T, c.max_frames);
  S2S_REQUIRE(ctx_frames >= 0 && ctx_frames < T, "codec decode: context %d must be smaller than T=%d", ctx_frames, T);
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  const int H = c.hidden, hd = H / c.heads, qd = c.heads * hd, kvd = c.kv_heads * hd, I = c.inter, ldq = qd + 2 * kvd;
  const int R = B * T;   // rows of the transformer part
  CodePtrs cp{};
  for (int b = 0; b < B; ++b) cp.p[b] = codes_d[b];
  code_embed_mean_kernel<<<R, 256, 0, st>>>(cp, T, c.quantizers, c.codebook_size, m->embed, H, m->x);
  S2S_LAUNCH_CHECK();
  for (int l = 0; l < c.layers; ++l) {
    const CodecLayer& L = m->layers[l];
    rmsnorm_rows_f32_kernel<<<(R + 7) / 8, 256, 0, st>>>(m->x, L.n1, c.rms_eps, R, H, m->xn);
    S2S_LAUNCH_CHECK();
    S2S_CHECK(contract(m, linear_args(m->xn, R, H, L.w_qkv, ldq, m->qkv), st));
    rope_rows_f32_kernel<<<R, 256, 0, st>>>(m->qkv, T, c.heads + c.kv_heads, hd, ldq, c.rope_theta);
    S2S_LAUNCH_CHECK();
    {
      const int nw = 8;
      const size_t sm = (size_t)nw * (hd + c.sliding_window) * 4;
      swa_attention_f32_kernel<<<(R * c.heads + nw - 1) / nw, nw * 32, sm, st>>>(m->qkv, B, T, c.heads, c.kv_heads, hd, c.sliding_window, m->att);
      S2S_LAUNCH_CHECK();
    }
    {
      ConvArgs a = linear_args(m->att, R, qd, L.w_o, H, m->x);
      a.scale = L.ls_attn; a.resid = m->x; a.ldr = H;
      S2S_CHECK(contract(m, a, st));
    }
    rmsnorm_rows_f32_kernel<<<(R + 7) / 8, 256, 0, st>>>(m->x, L.n2, c.rms_eps, R, H, m->xn);
    S2S_LAUNCH_CHECK();
    S2S_CHECK(contract(m, linear_args(m->xn, R, H, L.w_gu, 2 * I, m->gu), st));
    silu_mul_kernel<<<(unsigned)(((long long)R * I + 255) / 256), 256, 0, st>>>(m->gu, I, (long long)R * I, m->hmid);
    S2S_LAUNCH_CHECK();
    {
      ConvArgs a = linear_args(m->hmid, R, I, L.w_down, H, m->x);
      a.scale = L.ls_mlp; a.resid = m->x; a.ldr = H;
      S2S_CHECK(contract(m, a, st));
    }
  }
  rmsnorm_rows_f32_kernel<<<(R + 7) / 8, 256, 0, st>>>(m->x, m->norm_f, c.rms_eps, R, H, m->bufX);
  S2S_LAUNCH_CHECK();
  if (hidden_out_d) S2S_CHECK_CUDA(cudaMemcpyAsync(hidden_out_d, m->bufX, (size_t)R * H * 4, cudaMemcpyDeviceToDevice, st));
  // ---- causal trimming ---------------------------------------------------------------------------------------------
  // Only the samples of frames >= ctx_frames are returned, and every layer below the transformer is causal with a finite
  // receptive field: a layer only has to produce the rows its consumers read.  `need` is walked backwards from the first
  // returned sample through the layer list (conv k taps, dilation d: rows o - (k-1)d .. o; transposed conv of stride r: rows
  // floor(o / r), +1; k = stride: floor(o / f)); the kept region is computed with exactly the arithmetic of the full decode,
  // so the result is bit-identical to decoding all T frames and dropping the history -- at ~1/3 of the work for 8 new
  // frames behind 25 (blocks 2-4, most of the FLOPs, run over ~9 frames instead of 33).
  const int n_up = c.n_upsampling_ratios, n_blk = c.n_upsample_rates;
  std::vector<int> Ls;
  codec_lengths(c, T, Ls);                       // Ls[0] = rows entering decoder.0, Ls[i + 1] = rows after block i
  const int skip = ctx_frames * m->total_up;
  const int n_out = Ls.back() - skip;
  S2S_REQUIRE(n_out > 0, "codec decode: nothing left after dropping %d context frames", ctx_frames);
  static const int dil[3] = {1, 3, 9};
  // rows that must exist (first needed row) of: each block's output, each residual unit's output, each block's transposed-conv
  // output and input; decoder.0's output; each upsampler's output and input
  std::vector<int> need_blk_out(n_blk), need_unit(n_blk * 3), need_blk_in(n_blk), need_up_out(n_up), need_up_in(n_up);
  const int need_final_in = std::max(0, skip - 6);                 // final conv 7 reads rows o - 6 .. o
  {
    int need = need_final_in;
    for (int i = n_blk - 1; i >= 0; --i) {
      need_blk_out[i] = need;
      for (int u = 2; u >= 0; --u) { need_unit[i * 3 + u] = need; need = std::max(0, need - 6 * dil[u]); }   // conv 7, dilation d
      need_blk_in[i] = need / c.upsample_rates[i];                  // transposed conv: out row o reads in rows floor(o / r), + 1
      need = need_blk_in[i];
    }
    need = std::max(0, need - 6);                                   // decoder.0 conv 7
    for (int i = n_up - 1; i >= 0; --i) {
      need_up_out[i] = need;
      need_up_in[i] = std::max(0, need - 6) / c.upsampling_ratios[i];   // depthwise conv 7, then k = stride transposed conv
      need = need_up_in[i];
    }
  }
  // upsampling stages: transposed conv (k = stride) + ConvNeXt, one sequence per blockIdx.z from here on
  float *X = m->bufX, *A = m->bufA, *Hb = m->bufH;
  int len = T;   // per sequence
  auto batched = [&](ConvArgs a, int cin, int cout_row, int rows_in, int rows_out, int t0) {
    a.batch = B; a.x_bs = (long long)rows_in * cin; a.y_bs = (long long)rows_out * cout_row; a.r_bs = a.y_bs; a.t0 = t0;
    return a;
  };
  for (int i = 0; i < n_up; ++i) {
    const CodecConvNeXt& U = m->ups[i];
    const int f = c.upsampling_ratios[i], f_out = need_up_out[i];
    {
      ConvArgs a = linear_args(X, len, H, U.up_w, f * H, A);            // input row t produces output rows t f .. t f + f - 1
      a.bias = U.up_b; a.bias_mod = H;
      S2S_CHECK(contract(m, batched(a, H, f * H, len, len, need_up_in[i]), st));
    }
    len *= f;   // A is [B][len, H], valid from row need_up_in[i] * f <= f_out - 6
    dwconv7_ln_kernel<<<B * (len - f_out), 256, (size_t)H * 4, st>>>(A, len, f_out, H, U.dw_w, U.dw_b, U.ln_w, U.ln_b, 1e-6f, Hb);
    S2S_LAUNCH_CHECK();
    {
      ConvArgs a = linear_args(Hb, len, H, U.pw1_w, 4 * H, X);
      a.bias = U.pw1_b; a.act = 1;
      S2S_CHECK(contract(m, batched(a, H, 4 * H, len, len, f_out), st));
    }
    {
      ConvArgs a = linear_args(X, len, 4 * H, U.pw2_w, H, A);
      a.bias = U.pw2_b; a.scale = U.gamma; a.resid = A; a.ldr = H;
      S2S_CHECK(contract(m, batched(a, 4 * H, H, len, len, f_out), st));
    }
    std::swap(X, A);   // X = stage output [B][len, H], valid from row f_out
  }
  const int D = c.decoder_dim;
  const int need_d0 = n_blk ? need_blk_in[0] : need_final_in;
  S2S_CHECK(contract(m, batched(causal_conv_args(X, len, H, m->d0_w, m->d0_b, 7, 1, D, A), H, D, len, len, need_d0), st));
  std::swap(X, A);
  for (int i = 0; i < n_blk; ++i) {
    const CodecBlock& Bk = m->blocks[i];
    const int t_first = need_blk_in[i];                               // first input row (= first transposed-conv "row")
    const bool h0 = fp16_operand_ok(m, Bk.tc_w, Bk.cin, Bk.rate * Bk.cout);
    if (h0) S2S_CHECK(snake_launch_h(X, Bk.a0, Bk.b0, Bk.cin, B, len, t_first, A, st));
    else S2S_CHECK(snake_launch(X, Bk.a0, Bk.b0, Bk.cin, B, len, t_first, A, st));
    {
      ConvArgs a{};
      a.x = A; a.x16 = h0 ? A : nullptr; a.ldx = Bk.cin; a.T_in = len; a.x_row0 = 0; a.w = Bk.tc_w; a.k = 2; a.dil = 1; a.C_in = Bk.cin; a.N = Bk.rate * Bk.cout;
      a.bias = Bk.tc_b; a.bias_mod = Bk.cout; a.y = X; a.ldy = (long long)Bk.rate * Bk.cout; a.T_out = len - 1;
      S2S_CHECK(contract(m, batched(a, Bk.cin, Bk.rate * Bk.cout, len, len - 1, t_first), st));
    }
    len = (len - 1) * Bk.rate;            // X is [B][len, cout], valid from row t_first * rate
    int have = t_first * Bk.rate;         // first valid row of the block's residual stream
    for (int u = 0; u < 3; ++u) {
      const CodecResUnit& Ru = Bk.u[u];
      const int f_u = need_unit[i * 3 + u];                            // rows this unit must produce (reads f_u - 6 d >= have)
      const bool h1 = fp16_operand_ok(m, Ru.c1_w, Bk.cout, Bk.cout), h2 = fp16_operand_ok(m, Ru.c2_w, Bk.cout, Bk.cout);
      if (h1) S2S_CHECK(snake_launch_h(X, Ru.a1, Ru.b1, Bk.cout, B, len, have, A, st));
      else S2S_CHECK(snake_launch(X, Ru.a1, Ru.b1, Bk.cout, B, len, have, A, st));
      {
        ConvArgs a1 = causal_conv_args(A, len, Bk.cout, Ru.c1_w, Ru.c1_b, 7, dil[u], Bk.cout, Hb);
        a1.x16 = h1 ? A : nullptr;
        S2S_CHECK(contract(m, batched(a1, Bk.cout, Bk.cout, len, len, f_u), st));
      }
      if (h2) S2S_CHECK(snake_launch_h(Hb, Ru.a2, Ru.b2, Bk.cout, B, len, f_u, A, st));
      else S2S_CHECK(snake_launch(Hb, Ru.a2, Ru.b2, Bk.cout, B, len, f_u, A, st));
      ConvArgs a = linear_args(A, len, Bk.cout, Ru.c2_w, Bk.cout, X);
      a.x16 = h2 ? A : nullptr;
      a.bias = Ru.c2_b; a.resid = X; a.ldr = Bk.cout;
      S2S_CHECK(contract(m, batched(a, Bk.cout, Bk.cout, len, len, f_u), st));
      have = f_u;
    }
  }
  const int cl = D >> n_blk;
  S2S_CHECK(snake_launch(X, m->fa, m->fb, cl, B, len, need_final_in, A, st));
  S2S_CHECK(contract(m, batched(causal_conv_args(A, len, cl, m->f_w, m->f_b, 7, 1, 1, Hb), cl, 1, len, len, skip), st));
  S2S_REQUIRE(B == 1 || wav_stride >= n_out, "codec decode: wav_stride %lld < %d samples", wav_stride, n_out);
  clamp_out_kernel<<<dim3((n_out + 255) / 256, B), 256, 0, st>>>(Hb, len, skip, n_out, wav_out_d, wav_stride);
  S2S_LAUNCH_CHECK();
  if (n_out_h) *n_out_h = n_out;
  return S2S_OK;
}

int codec_decode(CodecDecoder* m, const int32_t* codes_d, int T, int ctx_frames, float* wav_out_d, int32_t* n_out_h,
                 float* hidden_out_d, cudaStream_t st) {
  return codec_decode_batch(m, &codes_d, 1, T, ctx_frames, wav_out_d, 0, n_out_h, hidden_out_d, st);
}

extern "C" {
int s2s_codec_create(s2s_ctx* ctx, const s2s_codec_config* cfg, s2s_codec** out) { return codec_create(ctx, cfg, out); }
int s2s_codec_destroy(s2s_codec* m) { return codec_destroy(m); }
int s2s_codec_bind_tensor(s2s_codec* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim, int32_t dtype) {
  return codec_bind_tensor(m, name, data_h, shape, ndim, dtype);
}
int s2s_codec_init_random(s2s_codec* m, uint64_t seed) { return codec_init_random(m, seed); }
int s2s_codec_finalize(s2s_codec* m) { return codec_finalize(m); }
int s2s_codec_decode(s2s_codec* m, const int32_t* codes_d, int32_t T, int32_t ctx_frames, float* wav_out_d, int32_t* n_out_h,
                     float* hidden_out_d, void* stream) {
  return codec_decode(m, codes_d, T, ctx_frames, wav_out_d, n_out_h, hidden_out_d, (cudaStream_t)stream);
}
int32_t s2s_codec_samples(s2s_codec* m, int32_t T) { return m ? codec_samples_for(m, T) : 0; }
int32_t s2s_codec_total_upsample(s2s_codec* m) { return m ? codec_total_upsample(m) : 0; }
}  // extern "C"
