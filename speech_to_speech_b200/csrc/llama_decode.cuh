// llama_decode.cuh -- parameters of the persistent Llama-family greedy-decode kernel.
#pragma once
#include "common.cuh"
#include "sampling.cuh"

struct LlamaDecLayer {          // device pointers; 16-bit weights [out, in]: TILED layout (weight_tiles.cu) in the kernel's table,
                                // or (weight format S2S_FP8_E4M3) tiled E4M3 codes followed by the fp32 row scales
  const void* w_qkv;            // [(H + 2 KV) * hd, d]; q and k rows stored pair-adjacent for RoPE (see llama.cu)
  const void* w_o;              // [d, H * hd]
  const void* w_gu;             // [2 * ffn, d], rows interleaved (gate_i, up_i)
  const void* w_down;           // [d, ffn]
  const float *norm1, *norm2;   // RMSNorm weights [d]
  const float *q_norm, *k_norm; // Qwen3 (qk_norm): per-head RMSNorm weights [hd], stored pair-adjacent like the q/k rows; else null
};

struct LlamaDecParams {
  int d, heads, kv_heads, hd, layers, ffn, vocab, B, max_pos;
  float eps;
  const LlamaDecLayer* lw;      // [layers] device
  const void* embed;            // [vocab, d] 16-bit
  const void* lm_head;          // [vocab, d] TILED layout, 16-bit or FP8 like the layers' matrices
  const float* norm_f;          // [d]
  const float2* rope;           // [max_pos][hd/2] (cos, sin)
  // state
  float* x;                     // [B, d] residual stream
  float* q;                     // [B, H*hd]
  void* h;                      // [B, ffn] 16-bit (SwiGLU output)
  void* kv;                     // [slots][layers][2][max_pos][KV*hd] 16-bit
  long long kv_slot_stride, kv_layer_stride, kv_which_stride;
  float* part;                  // [B][H][s_max][hd + 4] split records of the attention phase
  int s_max;
  void* attn16;                 // [B, H*hd] 16-bit attention output (input of o_proj)
  unsigned int* attn_cnt;       // [B * H] finished splits per (session, head); zero between phases
  const int* slot;              // [B]
  int* pos;                     // [B] position of the token being processed (advanced by the kernel)
  int max_len;                  // max over b of (pos[b] + 1) at step 0
  // token bookkeeping
  const int* first_ids;         // [B]
  int n_steps, eos;
  int* out_ids;                 // [B][n_steps]
  int* out_len;                 // [B]
  const int* forced;            // [B][n_steps] or null
  float* logits_out;            // [n_steps][B][vocab] or null
  int* done; int* n_done;
  float* cand_val; int* cand_idx;   // [B][grid]
  unsigned int* sync_counter;
  // ---- Qwen3 family (qk_norm): the qkv phase stores raw q / k rows; the attention items apply RMSNorm(head_dim) + RoPE
  int qk_norm;
  float* kraw;                  // [B][KV*hd] fp32 raw k rows of the current token
  float* qn;                    // [B][H*hd] fp32 normalised, rotated, scaled q rows (written and read inside the attention phase)
  // ---- embedding-driven use (Qwen3-TTS talker and code predictor, qwen3tts.cu) ----
  const float* x_in;            // [B][d] fp32 or null: the input of step 0 is this vector instead of embed[first_ids]
  float* hidden_out;            // [n_steps][B][d] fp32 or null: the residual stream BEFORE the final norm of every step
  const unsigned char* suppress;// [vocab] or null: bit0 = never predict this id (EPI_LOGITS mask)
  // multi-table mode (code predictor: one embedding table and one output head per codebook): step 0 consumes x_in and
  // predicts nothing, then feeds first_ids through `embed0`; step s >= 1 predicts with lm_head + (s-1)*head_stride and
  // feeds its argmax through embed + (s-1)*embed_stride (strides in elements; 0 = single-table mode)
  long long embed_stride, head_stride;
  const void* embed0;           // [vocab0, d] 16-bit
  int ring_slots;               // weight-ring slots per warp (set by the launcher)
  int norm_rg;                  // rows of the fp32 statistics copy resident at a time (set by the launcher; B = all at once;
                                // DEC_NORM_L2 = no copy, rows read from L2 into registers)
  int down_kc;                  // > 0: the down-projection operand is staged in K-chunks of this many columns (large batches)
  int assoc_b;                  // the batch whose plan fixes the attention split plan (set by the launcher, see LlamaDecPlan)
  unsigned long long* trace;    // optional [2][cap][6] globaltimer stamps (profiling aid, dec_run)
  int trace_cap;
  // ---- per-session token choice (sampling.cuh); samp == null: every session takes the argmax-candidate path ----
  const SampSlot* samp;         // [B] or null
  float* samp_rows;             // [B][vocab] fp32 logits rows of the step (used when logits_out is null)
  unsigned int* seen;           // [slots][seen_words] ids seen by each slot (repetition penalty)
  int seen_words;
  int seen_fixed;               // 1: the caller maintains the seen sets (Qwen3-TTS talker); the launch adds no fed id
};

// dtype: the compute type (S2S_BF16 / S2S_F16); weight_format: dtype, or S2S_FP8_E4M3 (bf16 compute, single-table only)
int llama_decode_launch(s2s_ctx* ctx, const LlamaDecParams& p, int dtype, int weight_format, int debug_phases, cudaStream_t stream);
// largest batch per launch on `grid` CTAs that has a shared-memory plan (llama_decode_plan.cuh) on `device`
int llama_decode_max_batch(int device, int dtype, int weight_format, int d, int ffn, int qd, int grid);
