// llama_decode.cuh -- parameters of the persistent Llama-family greedy-decode kernel.
#pragma once
#include "common.cuh"

struct LlamaDecLayer {          // device pointers; 16-bit weights [out, in]: TILED layout (weight_tiles.cu) in the kernel's table
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
  const void* lm_head;          // [vocab, d] 16-bit, TILED layout
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
  int norm_rg;                  // rows of the fp32 statistics copy resident at a time (set by the launcher; B = all at once)
  int down_kc;                  // > 0: the down-projection operand is staged in K-chunks of this many columns (large batches)
  unsigned long long* trace;    // optional [cap][3] globaltimer stamps of CTA 0 (phase begin, body end, barrier exit)
  int trace_cap;
  int sync_relaxed;             // 1: barrier waits without the acquire fence (A/B measurement aid)
};

int llama_decode_launch(s2s_ctx* ctx, const LlamaDecParams& p, int dtype, int debug_phases, cudaStream_t stream);
// largest batch per launch on `grid` CTAs that keeps >= 2 weight-ring slots per warp in shared memory
int llama_decode_max_batch(int d, int ffn, int qd, int grid);
// shared-memory plan of a batch: kmax = widest operand staged whole, rg = statistics rows per group, kc = down-projection chunk
// (0 = unchunked); returns false when the batch does not fit
bool llama_decode_plan(int B, int d, int ffn, int qd, int grid, int* kmax, int* rg, int* kc, int* ring_slots);
