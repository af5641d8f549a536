// kernels.cuh -- launch interfaces of the non-GEMM kernels (internal to libs2s_b200).
#pragma once
#include "common.cuh"

// ---- logmel.cu ----
struct LogmelTables {
  const float* hann;     // [400]
  const float* twiddle;  // [2][400] cos, sin of 2*pi*i/400
  const float* fb;       // [n_mels][201] slaney filter bank
  const int2* fb_range;  // [n_mels] non-zero bin range [lo, hi)
};
int logmel_launch(const LogmelTables& tb, const float* pcm_d, long long pcm_stride, const int* n_samples_d, int B,
                  int n_mels, float* mel_f32, float* mel_max, void* mel_t, int dtype, cudaStream_t stream);
int logmel_finalize_launch(const float* src, const float* mel_max, int normalize, int B, int n_mels, float* dst_f32,
                           void* mel_t, int dtype, cudaStream_t stream);

// ---- attention_tc.cu (wgmma / TMA) ----
size_t attention_tc_scratch_elems(int B, int Tk, int kv_heads, int hd);  // 16-bit elements of V^T scratch
int attention_tc_launch(s2s_ctx* ctx, const void* q, const void* k, const void* v, void* o, int B, int Tq, int Tk,
                        int heads, int kv_heads, int hd, long long ldq, long long ldk, long long ldv, long long ldo,
                        float scale, int causal, int dtype, void* vt_scratch, size_t vt_elems, cudaStream_t stream);
// ---- elementwise.cu ----
// y = LayerNorm(x) (bias != null) or RMSNorm(x) (bias == null); x fp32 [rows, d]; out_h 16-bit and/or out_f fp32
int norm_rows_launch(const float* x, const float* w, const float* bias, float eps, long long rows, int d, void* out_h,
                     float* out_f, int dtype, cudaStream_t stream);
int convert_f32_launch(const float* src, void* dst, long long n, int dtype, cudaStream_t stream);
int fill_random_launch(void* dst, long long n, int dtype, float scale, float offset, uint64_t seed,
                       cudaStream_t stream);
// ---- weight_tiles.cu ----
// row-major 16-bit [N, K] -> fragment-major tiled layout streamed by the decode kernels (see decode_common.cuh)
size_t tiled_weight_elems(int N, int K);
int tile_weights_launch(const void* W, int N, int K, void* Wt, cudaStream_t stream);
