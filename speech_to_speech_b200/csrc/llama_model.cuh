// llama_model.cuh -- the Llama-family model object (internal to libs2s_b200): shared by llama.cu (C ABI of the LLM slot)
// and qwen3tts.cu (Qwen3-TTS talker and code predictor are Qwen3-style decoders driven by embeddings).
#pragma once
#include <vector>

#include "common.cuh"
#include "llama_decode.cuh"
#include "weight_arena.cuh"

struct s2s_llama {
  s2s_ctx* ctx = nullptr;
  s2s_llama_config cfg{};
  bool finalized = false;
  bool matrices = false;                 // the tiled matrices are allocated: the weight format is fixed
  int weight_format = 0;                 // storage of the projections and lm_head: cfg.compute_dtype, or S2S_FP8_E4M3
  int debug_phases = 0;
  WeightArena arena;
  bool lm_head_bound = false;
  // weights
  void* embed = nullptr;                 // row-major (a lookup)
  float* norm_f = nullptr;
  // the projections in the one tiled layout (weight_tiles.cu) that prefill and decode both read: 16-bit, or FP8 codes +
  // row scales
  std::vector<LlamaDecLayer> layers_h;
  LlamaDecLayer* layers_d = nullptr;     // device copy of layers_h
  void* lm_head_t = nullptr;             // tiled like the projections; n_tables heads of head_t_table_elems
  float2* rope = nullptr;
  // KV + sessions
  void* kv = nullptr;
  long long kv_slot_stride = 0, kv_layer_stride = 0, kv_which_stride = 0;
  std::vector<int> len;  // tokens in each slot
  // prefill workspace
  int* ids_d = nullptr;
  float *x = nullptr, *last_logits = nullptr, *batch_logits = nullptr;   // batch_logits: [MAX_DEC_B][vocab] (batched prefill)
  void *xn = nullptr, *qkv = nullptr, *attn = nullptr, *hbuf = nullptr, *vt = nullptr;
  size_t vt_elems = 0;
  // decode state
  float *dx = nullptr, *dq = nullptr, *dh = nullptr, *part = nullptr, *cand_val = nullptr;
  void* attn16 = nullptr;
  unsigned int* attn_cnt = nullptr;
  int *slot_d = nullptr, *pos_d = nullptr, *done = nullptr, *n_done = nullptr, *cand_idx = nullptr, *out_ids = nullptr,
      *out_len = nullptr, *next_id = nullptr;
  unsigned int* sync_counter = nullptr;
  int s_max = 0;
  unsigned long long* trace = nullptr;
  int trace_cap = 0;
  int n_tables = 1;                      // > 1: one embedding table and one output head per codebook (code predictor)
  size_t embed_table_elems = 0, head_t_table_elems = 0;
  float* qn = nullptr;                   // qk_norm: normalised q rows of the decode step [B][H*hd]
  float* kraw = nullptr;                 // qk_norm: raw k rows of the decode step [B][KV*hd]
  // token choice per slot (s2s_llama_set_sampling); active == 0: argmax
  std::vector<SampSlot> samp;            // [max_sessions]
  SampSlot* samp_d = nullptr;            // [MAX_DEC_B] the launch's packed parameters
  float* samp_rows = nullptr;            // [MAX_DEC_B][vocab]
  unsigned int* seen = nullptr;          // [max_sessions][seen_words]
  int seen_words = 0;
  std::vector<char> seen_stale;          // [max_sessions] reset since the seen set was last emptied
};


constexpr int LLAMA_MAX_DEC_B = 16;  // upper bound; the shared-memory budget of the geometry may allow fewer

// Run the decoder stack over the n fp32 rows already in m->x (embeddings), appending to `slot`'s KV cache.
// logits_out_d optional [n, vocab]; next_id_d optional [1] = argmax of the last position (table 0);
// hidden_out_d optional [d] fp32 = the last position's residual stream BEFORE the final norm.
int llama_prefill_rows(s2s_llama* m, int slot, int n, float* logits_out_d, int32_t* next_id_d, float* hidden_out_d,
                       cudaStream_t st);
// Everything of LlamaDecParams that does not depend on the call (geometry, weights, workspace).
void llama_fill_dec_params(s2s_llama* m, LlamaDecParams& p);
int llama_max_decode_batch_of(const s2s_llama* m);
// s2s_sampling -> SampSlot with the range checks of s2s_llama_set_sampling (NULL = greedy); errors are prefixed by `who`
int samp_from_abi(const s2s_sampling* s, int vocab, const char* who, SampSlot* out);
