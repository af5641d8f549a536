// whisper_decode.cuh -- parameters of the persistent Whisper greedy-decode kernel.
#pragma once
#include "common.cuh"

constexpr int ATT_CHUNK_KEYS = 64;  // keys per attention work item (== ATT_CHUNK in decode_common.cuh)

struct WhisperDecLayer {      // all device pointers; 16-bit weights [out, in] in the tiled layout (weight_tiles.cu)
  const void* w_qkv; const float* b_qkv;   // [3d, d]; q rows pre-scaled by head_dim^-0.5, k bias = 0
  const void* w_o;   const float* b_o;     // [d, d]
  const void* w_cq;  const float* b_cq;    // cross-attention q [d, d] (pre-scaled)
  const void* w_co;  const float* b_co;    // cross-attention out [d, d]
  const void* w_fc1; const float* b_fc1;   // [ffn, d]
  const void* w_fc2; const float* b_fc2;   // [d, ffn]
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *ln3_w, *ln3_b;
};

struct WhisperDecParams {
  int d, heads, layers, ffn, vocab, B, max_pos, n_ctx;
  const WhisperDecLayer* lw;   // [layers] device
  const void* embed;           // [vocab, d] 16-bit, tiled: token embedding lookup (gv_tiled_elem) and tied output projection
  const float* pos;            // [max_pos, d]
  const float *lnf_w, *lnf_b;
  // state
  float* x;                    // [B, d] residual stream (X0)
  float* x_alt;                // [B, d] second residual buffer (X1) -- cluster kernel
  float* part_x0;              // [heads][B][d] per-head partial out-projections (self block) -- cluster kernel
  float* part_x1;              // [heads][B][d] ... (cross block)
  int cluster_size;            // CTAs per cluster in the cluster kernel (0: 8-phase kernel)
  float* q;                    // [B, d]
  void* h;                     // [B, ffn] 16-bit (fc1 + GELU output)
  void* self_kv;               // [B][layers][2][max_pos][d] 16-bit
  const void* cross_kv;        // [B][layers][k|v][heads][n_ctx][64] 16-bit (head-major: GEMM epilogue head_major_rows)
  float* part;                 // [B][heads][s_max][64 + 4] split records of an attention phase
  int s_max;
  void* attn16;                // [B, d] 16-bit attention output (input of the out-projections)
  unsigned int* attn_cnt;      // [B * heads] finished splits per (session, head); zero between phases
  int cross_plan;              // item plan of the cross-attention phases (launcher: attn_plan)
  unsigned char self_plan[32]; // ... of self-attention, indexed by the number of 32-key blocks
  // token bookkeeping
  int* tokens;                 // [B][max_pos]
  int n_prefix, max_new, eos;
  const unsigned char* suppress;  // [vocab]: bit0 suppress always, bit1 suppress at the first generated position
  int* out_ids;                // [B][max_new]
  int* out_len;                // [B]
  const int* forced;           // [B][max_new] or null
  float* logits_out;           // [max_new][B][vocab] or null
  int* done;                   // [B]
  int* n_done;                 // [1]
  float* cand_val;             // [B][grid]
  int* cand_idx;               // [B][grid]
  unsigned int* sync_counter;  // [1], zeroed before launch
  int ring_slots;               // weight-ring slots per warp (set by the launcher from the shared-memory budget)
  unsigned long long* trace;   // optional [2][trace_cap][6] globaltimer stamps (profiling aid, dec_run)
  int trace_cap;
};

int whisper_decode_launch(s2s_ctx* ctx, const WhisperDecParams& p, int dtype, int debug_phases, cudaStream_t stream);
// largest batch per launch that keeps >= 2 weight-ring slots per warp in shared memory
int whisper_decode_max_batch(int d, int ffn);
