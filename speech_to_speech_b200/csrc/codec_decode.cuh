// codec_decode.cuh -- the TTS codec decoder (codes -> 24 kHz waveform) and its building-block kernels (internal).
#pragma once
#include "common.cuh"

// Y[t, n] = epilogue( bias[n % bias_mod] + sum_{j < k} sum_{c < C_in} X[t + x_row0 + j * dil, c] * W[j][c][n] ), fp32.
// Rows of X outside [0, T_in) read as zero (causal left padding).  Time-major activations: a transposed convolution of
// stride s is the same contraction with N = s * C_out and the output read as [(T - 1) * s, C_out] (see codec_decode.cu).
struct ConvArgs {
  const float* x; long long ldx; int T_in; int x_row0;
  const void* x16;                          // optional fp16 copy of x (same shape / strides in elements): tensor-core mode only
  const float* w; int k, dil, C_in, N;
  const float* bias; int bias_mod;
  int act;                                  // 0 none, 1 exact GELU, 2 SiLU
  const float* scale;                       // [N] or null (LayerScale / ConvNeXt gamma), applied after act
  const float* resid; long long ldr;        // [T_out, N] or null, added last (may alias y)
  float* y; long long ldy; int T_out;
  int t0;                                   // first output row computed (rows below it are never read downstream: causal trimming)
  int batch; long long x_bs, y_bs, r_bs;    // independent sequences along blockIdx.z
};
int conv1d_f32_launch(const ConvArgs& a, cudaStream_t st);
// the same contraction on the tensor cores; w_pairs = fp16 k-pair copy of a.w (pack_weight_pairs_kernel)
int conv1d_tc_launch(const ConvArgs& a, const void* w_pairs, cudaStream_t st);

typedef s2s_codec CodecDecoder;   // the C-ABI handle is the model object
int codec_create(s2s_ctx* ctx, const s2s_codec_config* cfg, CodecDecoder** out);
// a codec that reads source's weights (source finalized; cfg equal to source's but for max_frames and max_batch), finalized
int codec_create_shared(s2s_ctx* ctx, CodecDecoder* source, const s2s_codec_config* cfg, CodecDecoder** out);
// s2s_llama_device_bytes' meaning: weights = the (possibly shared) weight store, total = that + the object's own state
int codec_device_bytes(const CodecDecoder* m, int64_t* weights, int64_t* total);
int codec_destroy(CodecDecoder* m);
int codec_bind_tensor(CodecDecoder* m, const char* name, const void* data_h, const int64_t* shape, int ndim, int dtype);
int codec_init_random(CodecDecoder* m, uint64_t seed);
int codec_finalize(CodecDecoder* m);
// codes_d [T][Q] int32 -> the waveform of frames [ctx_frames, T) (the first ctx_frames * total_upsample samples are dropped:
// Qwen3OmniMoeCode2Wav.chunked_decode); *n_out_h = samples written to wav_out_d.  hidden_out_d optional [T, hidden].
int codec_decode(CodecDecoder* m, const int32_t* codes_d, int T, int ctx_frames, float* wav_out_d, int32_t* n_out_h,
                 float* hidden_out_d, cudaStream_t st);
int codec_decode_batch(CodecDecoder* m, const int32_t* const* codes_d, int B, int T, int ctx_frames, float* wav_out_d,
                       long long wav_stride, int32_t* n_out_h, float* hidden_out_d, cudaStream_t st);
int codec_samples_for(const CodecDecoder* m, int T);   // waveform length of a T-frame decode (before the context drop)
int codec_total_upsample(const CodecDecoder* m);
