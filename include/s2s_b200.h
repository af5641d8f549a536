/*
 * s2s_b200.h -- C ABI of libs2s_b200.so, the H100 (sm_90a) engine behind
 * huggingface/speech-to-speech's STT / LLM / TTS handler slots.
 *
 * The reference has no FFI of its own (pure Python); the calls this library replaces are
 * the third-party model-runtime calls inside the three handler process() methods:
 *
 *   s2s_whisper_*   <- processor(...) + model.generate(...)            S/STT/whisper_stt_handler.py:83-87, 166-197, 243
 *   s2s_llama_*     <- pipeline("text-generation")(prompt, ...)        S/LLM/language_model.py:800-892
 *   s2s_tts_*       <- _resample_to_pipeline_sr/_to_int16/_stream      S/TTS/qwen3_tts_handler.py:612-613, 674-680, 695-749
 *   (S/ = src/speech_to_speech of huggingface/speech-to-speech)
 *
 * Conventions: plain pointers and sizes only; every call returns 0 on success or a negative
 * S2S_ERR_* code (message via s2s_last_error(), thread-local).  Pointers suffixed _d are
 * device pointers, _h host pointers.  `stream` is a cudaStream_t passed as void*; device
 * work is enqueued on it and is asynchronous unless the call documents a host result.
 * The library owns its weights and workspaces (allocated at create/finalize); it never
 * frees caller memory.  A model handle may be used from one thread at a time; different
 * handles are independent.
 */
#ifndef S2S_B200_H
#define S2S_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define S2S_OK 0
#define S2S_ERR_INVALID -1   /* bad argument / shape / state */
#define S2S_ERR_CUDA -2      /* CUDA runtime or driver error */
#define S2S_ERR_NOT_FOUND -3 /* unknown tensor name */
#define S2S_ERR_UNSUPPORTED -4

/* element types for bind_tensor sources */
#define S2S_F32 0
#define S2S_F16 1
#define S2S_BF16 2
/* weight storage format only (s2s_llama_set_weight_format); never a bind_tensor source or a compute type */
#define S2S_FP8_E4M3 3

typedef struct s2s_ctx s2s_ctx;
typedef struct s2s_whisper s2s_whisper;
typedef struct s2s_llama s2s_llama;

/* ---- context ------------------------------------------------------------------------- */
int s2s_init(int device, s2s_ctx** out);
int s2s_destroy(s2s_ctx* ctx);
/* SM partition ("lane") of a context: the persistent cooperative decode kernels of the models created on `ctx` use `ctas`
 * CTAs (0 = one per SM, the default).  Contexts with disjoint partitions (e.g. two of 66 CTAs on a 132-SM H100), driven
 * from different CUDA streams, run their decode launches concurrently; a decode step is a chain of latency-bound phases, so
 * two half-grid launches take about as long as one whole-grid launch.  No reference counterpart (the reference runs one
 * session per model call). */
int s2s_set_sm_partition(s2s_ctx* ctx, int32_t ctas);
const char* s2s_last_error(void);
/* number of kernels this library launched in this process (all contexts, all host threads) since the last reset */
int64_t s2s_launch_count(s2s_ctx* ctx, int reset);
/* *out = device bytes the model objects of this process hold right now (all contexts, all host threads): weights,
 * workspaces and the staging buffer of bind_tensor / init_random, counted when allocated and when freed.  Unlike the
 * device's free memory it is not moved by other processes (tests, measurements). */
int s2s_allocated_bytes(int64_t* out);

/* ---- shared weights ---------------------------------------------------------------------
 * s2s_{whisper,llama,qwen3tts}_create_shared make an object on `ctx` that reads the weights of `source` instead of a copy
 * of its own -- e.g. one copy per GPU for the engines of two SM partitions (s2s_set_sm_partition) -- and keeps its own KV
 * cache, workspaces and decode state.  It computes bit for bit what an object bound to the same weights computes.
 * `source` must be finalized and on ctx's device; `cfg` must equal the source's configuration except for capacities
 * (llama: max_sessions, max_positions, max_prefill; whisper: max_batch; qwen3tts: max_sessions, max_positions, max_text,
 * codec.max_frames, codec.max_batch) -- any other difference is S2S_ERR_INVALID naming the field.  The llama weight format
 * comes from the source.  The new object comes back finalized; its decode plans follow its own context's CTA budget.
 * The weights are read-only while more than one object holds them: bind_tensor, init_random, finalize and
 * s2s_llama_set_weight_format return S2S_ERR_INVALID on an object made this way, and on its source while such an object
 * lives.  Objects are destroyed in any order; the weights are freed with the last of them.
 * *_device_bytes: *weights = the weight bytes the object reads (its own or the shared ones), *total = that plus what the
 * object allocated itself, so a set of objects sharing one source holds weights + sum(total - weights). */

/* ---- Whisper (STT) ---------------------------------------------------------------------
 * Geometry mirrors transformers WhisperConfig.  compute_dtype: S2S_F16 (reference default
 * stt_torch_dtype=float16) or S2S_BF16 = storage type of weights and GEMM operands;
 * accumulation, LayerNorm, softmax and the residual stream are fp32.                      */
typedef struct {
  int32_t d_model, heads, enc_layers, dec_layers, ffn, n_mels, vocab;
  int32_t max_source_positions; /* 1500 */
  int32_t max_target_positions; /* 448  */
  int32_t compute_dtype;
  int32_t max_batch; /* concurrent utterances per call */
} s2s_whisper_config;

int s2s_whisper_create(s2s_ctx* ctx, const s2s_whisper_config* cfg, s2s_whisper** out);
int s2s_whisper_destroy(s2s_whisper* m);
/* Copy one parameter (transformers state-dict name, e.g. "model.encoder.conv1.weight") from
 * HOST memory into the library's arena, converting to compute_dtype and to the kernel layout. */
int s2s_whisper_bind_tensor(s2s_whisper* m, const char* name, const void* data_h, const int64_t* shape,
                            int32_t ndim, int32_t dtype);
/* Fill every parameter with seeded pseudo-random values on the device (bench only). */
int s2s_whisper_init_random(s2s_whisper* m, uint64_t seed);
int s2s_whisper_finalize(s2s_whisper* m);
int s2s_whisper_create_shared(s2s_ctx* ctx, s2s_whisper* source, const s2s_whisper_config* cfg, s2s_whisper** out);
/* *weights = encoder and decoder weights (the tiled decoder matrices and embedding, cross-attention K/V projections,
 * positional tables); *total = that plus the log-mel tables, workspaces, KV caches and decode state (see shared weights) */
int s2s_whisper_device_bytes(s2s_whisper* m, int64_t* weights, int64_t* total);

/* decoding controls = what WhisperGenerationMixin.generate derives from generation_config */
typedef struct {
  const int32_t* prefix_h; /* forced decoder prompt, e.g. [sot, lang, transcribe, notimestamps] */
  int32_t n_prefix;
  int32_t max_new_tokens;
  int32_t eos_id;
  const int32_t* suppress_h; /* SuppressTokensLogitsProcessor */
  int32_t n_suppress;
  const int32_t* begin_suppress_h; /* SuppressTokensAtBeginLogitsProcessor */
  int32_t n_begin_suppress;
  const int32_t* prefix_rows_h;    /* optional [B][n_prefix]: one prompt per utterance (per-utterance language after
                                      detect_language on the SAME encoder output, whisper_stt_handler.py:236-241); NULL = prefix_h */
} s2s_whisper_decode_opts;

/* pcm_d: [B, pcm_stride] f32 mono 16 kHz, n_samples_h[b] valid samples each (rest ignored, padded
 * with zeros to 30 s like WhisperFeatureExtractor).  mel_out_d: optional [B, n_mels, 3000] f32. */
int s2s_whisper_logmel(s2s_whisper* m, const float* pcm_d, int64_t pcm_stride, const int32_t* n_samples_h,
                       int32_t B, float* mel_out_d, void* stream);
/* mel_in_d: optional [B, n_mels, 3000] f32 (NULL = use the features left by s2s_whisper_logmel).
 * enc_out_d: optional [B, 1500, d_model] f32 copy of the encoder output (after final LayerNorm).
 * Also computes the decoder cross-attention K/V for every decoder layer.                     */
int s2s_whisper_encode(s2s_whisper* m, const float* mel_in_d, int32_t B, float* enc_out_d, void* stream);
/* Greedy decode of the B utterances encoded last.  ids_out_d: [B, max_new_tokens] i32 (generated
 * tokens incl. EOS, then EOS padding), len_out_d: [B] i32.  forced_d (optional, [B, max_new_tokens]):
 * teacher-forced feedback tokens for parity tests.  logits_out_d (optional): [max_new_tokens, B, vocab]
 * f32 processed logits of every generation step (B <= s2s_whisper_max_decode_batch).  Up to 16 sessions share one
 * persistent launch (larger B is split); a single session uses the thread-block-cluster kernel.     */
int s2s_whisper_decode(s2s_whisper* m, const s2s_whisper_decode_opts* opts, int32_t B, int32_t* ids_out_d,
                       int32_t* len_out_d, const int32_t* forced_d, float* logits_out_d, void* stream);
/* One decoder step from <|sot|>, logits restricted to lang_ids -> lang_out_d[B] (detect_language). */
int s2s_whisper_detect_language(s2s_whisper* m, int32_t sot_id, const int32_t* lang_ids_h, int32_t n_lang,
                                int32_t B, int32_t* lang_out_d, void* stream);
/* Profiling aid: when trace_d != NULL the next decode launches record, for CTA 0 and the last CTA, the
 * %globaltimer (ns) at [phase begin, inputs staged, arrived at the grid barrier, next phase prepared, phase body end,
 * barrier exit] (the cluster kernel uses slots 2 and 3 for its intra-phase milestones) of the first
 * `capacity` phases into trace_d[2][capacity][6] (u64).  NULL disables tracing.                                          */
int s2s_whisper_set_trace(s2s_whisper* m, uint64_t* trace_d, int32_t capacity);
/* Sessions one persistent decode launch can carry for this geometry (<= 16; larger batches are split by the library).
 * The session batcher (speech_to_speech_b200/batcher.py) sizes its batches with it. */
int32_t s2s_whisper_max_decode_batch(s2s_whisper* m);
/* End-to-end with HOST buffers: H2D of pcm, log-mel, encode, greedy decode, D2H of ids; synchronous.
 * pcm_h: [B, pcm_stride] f32 (pinned or pageable), ids_out_h: [B, max_new_tokens], len_out_h: [B].  */
int s2s_whisper_transcribe(s2s_whisper* m, const s2s_whisper_decode_opts* opts, const float* pcm_h,
                           int64_t pcm_stride, const int32_t* n_samples_h, int32_t B, int32_t* ids_out_h,
                           int32_t* len_out_h, void* stream);

/* ---- the prefill / encoder GEMM by itself (exposed for tests / roofline benches) ----------
 * The wgmma + TMA kernel every Whisper encoder op and every Llama-family prefill projection runs, in any form those call
 * sites use (fields as the library's own GemmProblem):
 *   v[b][m][n] = sum_k A[b][m][k] W[n][k] (+ bias[n]),   A[b][m][k] at a + b*a_batch_stride + m*a_row_stride + k,
 * fp32 accumulation; a_row_stride < K reads overlapping windows (Whisper's convolutions without im2col).  W: w_layout 0
 * row-major [N][ldw]; 1 the 16-bit tiles of s2s_tile_weights (K % 32 == 0); 2 its FP8 codes + row scales (bf16 only),
 * computing exactly the bf16 GEMM over dq(Q).  Epilogue per output row orow = b*out_batch_rows + out_row_offset + m:
 * act 1 exact GELU, act 2 SwiGLU over interleaved (gate, up) columns -> out_h[orow*ldo_h + n/2] (16-bit only); fp32
 * out_f[orow*ldo_f + n] = v + resid (resid_mode 1: resid row orow, may be out_f itself; 2: resid row m, a table broadcast
 * over the batch); 16-bit out_h[orow*ldo_h + n], or with head_major_rows R > 0 at
 * ((orow/R * N/64 + n/64) * R + orow%R) * 64 + n%64.  dtype S2S_F16 / S2S_BF16 (A, W and out_h).  bn: the N tile,
 * 0 = the library's rule, 64 or 128 to force one (128 needs N % 128 == 0).  S2S_ERR_INVALID, with nothing launched, on
 * N % 64, K % 8 (K % 32 tiled), a row stride that is not a multiple of 8, operands not 16-byte aligned, FP8 without bf16,
 * no output, a residual without out_f or with resid_mode outside {1, 2}, act 2 with out_f / head_major_rows or without
 * out_h, head_major_rows without out_h, bn outside {0, 64, 128}.  Asynchronous on `stream`. */
#define S2S_GEMM_W_ROW_MAJOR 0
#define S2S_GEMM_W_TILED16 1
#define S2S_GEMM_W_TILED_FP8 2
typedef struct {
  const void* a; int64_t a_row_stride, a_batch_stride;
  const void* w; int64_t ldw;
  int32_t w_layout;
  int32_t M, N, K, batch;
  const float* bias; int32_t act;
  void* out_h; int64_t ldo_h;
  float* out_f; int64_t ldo_f;
  const float* resid; int64_t ld_resid; int32_t resid_mode;
  int64_t out_batch_rows, out_row_offset;
  int32_t head_major_rows;
  int32_t dtype, bn;
} s2s_gemm_args;
int s2s_gemm_ex(s2s_ctx* ctx, const s2s_gemm_args* args, void* stream);
/* The tiled weight layout the Llama-family engines store their projections in, which both the decode kernel and the
 * prefill GEMMs read: element (row 8t+g, k 32w+8j+e) of a row-major [N, K] matrix at ((t*K/32 + w)*32 + 4g + j)*8 + e.
 * format S2S_F16 / S2S_BF16: 16-bit elements; S2S_FP8_E4M3: one E4M3 code per element, Q = e4m3(W * 2^-e_n) with the
 * smallest integer e_n that keeps the row's largest magnitude <= 448, followed by the N fp32 row scales 2^e_n.
 * s2s_tiled_weight_bytes: the buffer size (0 for an invalid shape or format).  s2s_tile_weights: row-major w_d [N, K]
 * (bf16 for FP8) -> out_d; N a multiple of 8, K of 32.  s2s_gemm_ex reads it with w_layout 1 / 2. */
int64_t s2s_tiled_weight_bytes(int32_t N, int32_t K, int32_t format);
int s2s_tile_weights(s2s_ctx* ctx, const void* w_d, int32_t N, int32_t K, int32_t format, void* out_d, void* stream);
/* O = softmax(Q K^T * scale [+causal]) V ; q/k/v/o row-major [T, heads*hd] slices with row strides
 * (elements); kv_heads <= heads (GQA).  hd in {64, 128}.                                     */
int s2s_attention(s2s_ctx* ctx, const void* q_d, const void* k_d, const void* v_d, void* o_d, int32_t B,
                  int32_t Tq, int32_t Tk, int32_t heads, int32_t kv_heads, int32_t hd, int64_t ldq,
                  int64_t ldk, int64_t ldv, int64_t ldo, float scale, int32_t causal, int32_t dtype,
                  void* stream);
/* One attention phase of the Llama-family decode by itself (exposed for tests): the production device function of the
 * persistent decode kernel, cut into (session, head, key split) items by the same plan, run in a plain launch of `grid`
 * CTAs.  Session b attends its first lens_h[b] cached keys (the step's own key included) with the fp32 query q[b]:
 *   out[b][h] = sum_j softmax_j(q[b][h] . K[j]) V[j],   K / V = the kv head h / (heads / kv_heads) of slot slots_h[b].
 * kv holds one layer of the model's cache layout, [slots][2][max_pos][kv_heads * hd] (K rows, then V rows, per slot).
 * grid 0 = the context's decode grid (s2s_set_sm_partition); assoc_b 0 = B, else the batch whose plan fixes the split
 * plan (the decode launch uses 8 at 13 to 16 Llama-3-8B sessions).  *plan_out_h (may be NULL) = the plan: key splits per
 * (session, head) in bits 0-6, bit 7 set for warp-level items.  Split records and counters are allocated per call, and a
 * counter the merge left non-zero is an error.  Synchronous: returns after the stream has finished.
 * Qwen3 mode (qk_norm = 1), the attention phase of the Qwen3 / Qwen3-TTS decode: q is the RAW q row, the cache holds keys
 * [0, len - 1) and kraw[b] the raw key of the step.  At the head of every item the kernel's ld_qk_prepare normalises
 * (RMSNorm over hd with q_norm / k_norm and eps, fp32 statistics), rotates (rope [max_pos][hd / 2] fp32 (cos, sin) at
 * position len - 1) and scales (1 / sqrt(hd)) q; the item whose key split holds key len - 1 normalises and rotates kraw and
 * writes it to cache row len - 1 first.  q_norm / k_norm are stored pair-adjacent like the q / k rows (the model's layout).
 * qn_out (may be NULL): the normalised, rotated, scaled q [B][heads][hd].  Pointers 16-byte aligned. */
typedef struct {
  const float* q;        /* [B][heads][hd] fp32, softmax scale applied (qk_norm: raw) */
  void* kv;              /* 16-bit (dtype), [slots][2][max_pos][kv_heads * hd]; qk_norm: K row len - 1 is written */
  int32_t max_pos;
  const int32_t* slots_h; const int32_t* lens_h; int32_t B;   /* lens_h[b] in [1, max_pos]; B in [1, 16] */
  int32_t heads, kv_heads, hd, dtype;                         /* hd 64 or 128; dtype S2S_F16 or S2S_BF16 */
  int32_t grid;          /* CTAs; 0 = the context's decode grid */
  int32_t assoc_b;       /* 0 = B */
  void* out;             /* [B][heads][hd] 16-bit */
  int32_t qk_norm;       /* 0: q is final (the fields below are ignored); 1: Qwen3 mode */
  const float* kraw;     /* [B][kv_heads][hd] fp32 raw keys of the step */
  const float* q_norm;   /* [hd] */
  const float* k_norm;   /* [hd] */
  const float* rope;     /* [max_pos][hd / 2] (cos, sin) pairs */
  float eps;
  float* qn_out;         /* [B][heads][hd] fp32 or NULL */
} s2s_dec_attn_args;
int s2s_decode_attention(s2s_ctx* ctx, const s2s_dec_attn_args* args, int32_t* plan_out_h, void* stream);
/* The skinny GEMM of the persistent decode kernels by itself (exposed for tests): the production device functions
 * (gemv_mma / gemv_mma_chunked, their staging routines and epilogues) in one plain launch of `grid` CTAs, running n_proj
 * <= 3 projections back to back with one weight ring per warp, so ring slot and parity carry over between them as between
 * the phases of a decode launch.  Projection i computes, for sessions b < B,
 *   v[b][n] = sum_k W[n][k] x[b][k] (+ bias[n]),   W from s2s_tile_weights (16-bit, or FP8 codes + row scales),
 * with x staged from `input`: COPY 16-bit rows x16 [B][K]; NORM fp32 rows xf [B][K] normalised (norm 1 LayerNorm with
 * norm_w / norm_b, 2 RMSNorm with norm_w; eps; rg rows of the fp32 copy resident at a time, 0 = B, -1 = read from L2,
 * K <= 4096); NORM_SUM xf + add_bias + sum of n_parts partials parts [n_parts][B][K], summed in that order, written to
 * x_out by CTA 0 (may be NULL) and normalised as NORM; CHUNKED 16-bit rows x16 [B][K] staged kc columns at a time.  The
 * epilogue `mode` is the decode kernels' (0 STORE out[b*ldo + n]; 1 GELU 16-bit out_h[b*ldh + n]; 2 RESID out += v;
 * 3 QKV: q rows -> out, k / v rows -> the 16-bit cache kv0 + which*kv_which + b*kv_batch + c; 4 LOGITS: suppress bits
 * 1 always / 2 at first_step set a row to -inf, optional logits_out[b*logits_ld + n], argmax (lowest id on ties) ->
 * argmax_out[b]; 5 QKV_ROPE: rows [0, q_rows) rotated with rope[pos[b]] (fp32 (cos, sin) pairs, hd/2 per position) and
 * scaled by q_scale -> out, [q_rows, q_rows + k_rows) rotated -> K cache, the rest -> V cache, cache element (b, c) at
 * kv0 + which*kv_which + slot[b]*kv_slot + pos[b]*kv_ld + c; kraw != NULL stores q and k raw (q -> out, k -> kraw[b][k_rows]);
 * 6 SWIGLU: row pairs (gate, up) -> out_h[b*ldh + n/2]).  Modes 1 and 3 exist with llama = 0 only, 5 and 6 with llama = 1.
 * Pointers are device pointers.  The projections of one call must not read what an earlier one writes (no grid barrier).
 * grid 0 = the context's decode grid; slots 1..4 ring slots per warp (0 = as many as fit); prefetch: issue a projection's
 * first weight units before its input is staged, as the decode kernels' look-ahead does (not for CHUNKED); use_plans:
 * plans computed once at kernel start, else on the fly; drain: before the last projection, issue projection 0's first
 * units and wait for them unused (an early exit's gemv_drain).  staged (may be NULL): CTA 0's staged 16-bit operand
 * [B][K].  plans_out_h (may be NULL): int32 [n_proj][5] = n_tiles, main_rounds, ks_log, slice, tail_rounds of CTA 0 (for
 * CHUNKED, the plan of [N, kc] as the host recomputes it from the same inputs).
 * Virtual clusters (cluster > 0; the per-head plans of the Whisper single-session kernel without cluster hardware): CTA i is
 * rank i % cluster of cluster cid = i / cluster, which owns head cid when cid < heads; grid % cluster == 0 and
 * grid / cluster >= heads.  A projection with head_plan 1 (the q, k, v rows of head cid of a [3d, d] QKV projection, K = d),
 * 2 (the q rows of head cid of a [d, d] projection) or 3 (all d rows of a [d, d] matrix times the head's 64 columns, K = 64,
 * N = d) runs the cluster-local plan gemv_head_plan builds; x16 and out of cluster cid are offset by cid * x_cluster_stride
 * and cid * out_cluster_stride elements (min(cid, heads - 1) for clusters without a head).
 * S2S_ERR_INVALID on K % 32 != 0, B outside [1, 16], FP8 with anything but bf16 / llama = 1, a mode the instantiation
 * lacks, a kc gemv_chunk_ok rejects, odd N outside LOGITS, a bias with odd N.  Per-call scratch; synchronous. */
#define S2S_GEMV_IN_COPY 0
#define S2S_GEMV_IN_NORM 1
#define S2S_GEMV_IN_NORM_SUM 2
#define S2S_GEMV_IN_CHUNKED 3
typedef struct {
  const void* w; int32_t N, K; const float* bias;
  int32_t input;
  const void* x16; int32_t kc;
  const float* xf; int32_t norm; const float* norm_w; const float* norm_b; float eps; int32_t rg;
  const float* parts; int32_t n_parts; const float* add_bias; float* x_out;
  void* staged;
  int32_t mode;
  float* out; int32_t ldo; void* out_h; int32_t ldh;
  void* kv0; int64_t kv_which, kv_batch; int32_t d;
  const int32_t* pos; const int32_t* slot; int64_t kv_slot; int32_t kv_ld; const float* rope; int32_t hd, q_rows, k_rows;
  float q_scale; float* kraw;
  const uint8_t* suppress; int32_t first_step; float* logits_out; int64_t logits_ld; int32_t* argmax_out;
  int32_t head_plan; int64_t x_cluster_stride, out_cluster_stride;   /* virtual clusters only */
} s2s_dec_gemv_proj;
typedef struct {
  s2s_dec_gemv_proj proj[3]; int32_t n_proj;
  int32_t B, dtype, weight_format, llama;   /* weight_format = dtype, or S2S_FP8_E4M3 (bf16, llama = 1) */
  int32_t grid, slots, prefetch, use_plans, drain;
  int32_t cluster, heads;                   /* virtual clusters: 0 = whole-grid plans only */
} s2s_dec_gemv_args;
int s2s_decode_gemv(s2s_ctx* ctx, const s2s_dec_gemv_args* args, int32_t* plans_out_h, void* stream);
/* The prefill / encoder row norm by itself (exposed for tests): the launch every Whisper encoder layer and every
 * Llama-family prefill layer runs.  For each of `rows` fp32 rows x[r][0..d), two-pass fp32 statistics:
 *   bias != NULL: LayerNorm   y = (x - mean) / sqrt(var + eps) * w + bias
 *   bias == NULL: RMSNorm     y = x / sqrt(mean(x^2) + eps) * w
 * -> out_h [rows][d] 16-bit (dtype) and / or out_f [rows][d] fp32.  S2S_ERR_INVALID, with nothing launched, on d % 4 != 0,
 * rows < 1, no output, x / w / bias / out_f not 16-byte aligned, out_h not 8-byte aligned, dtype not S2S_F16 / S2S_BF16.
 * Asynchronous on `stream`. */
int s2s_norm_rows(s2s_ctx* ctx, const float* x, const float* w, const float* bias, float eps, int64_t rows, int32_t d,
                  void* out_h, float* out_f, int32_t dtype, void* stream);
/* The RoPE / KV-append step of a Llama-family prefill layer by itself (exposed for tests): the launch the prefill runs for
 * each segment.  qkv: n 16-bit rows [heads * hd | kv_heads * hd | kv_heads * hd] (q, k, v; q and k rows and q_norm / k_norm
 * stored pair-adjacent, element 2j, 2j + 1 of a head = rotate_half partners j, j + hd / 2).  Token t sits at position past + t:
 * with q_norm == k_norm == NULL (Llama) q and k are rotated with rope[past + t] ((cos, sin) fp32 pairs [max_pos][hd / 2]);
 * with both given (Qwen3) each q / k head is first RMS-normalised over hd (fp32 statistics, eps).  q is rewritten in place,
 * the rotated k row goes to kcache[past + t] and the v row to vcache[past + t] (caches [max_pos][kv_heads * hd]); the k and v
 * columns of qkv are left as they were.  S2S_ERR_INVALID, with nothing launched, on hd not 64 / 128, n < 1, past < 0,
 * past + n > max_pos, heads % kv_heads, one norm weight without the other, pointers not 16-byte aligned, dtype not
 * S2S_F16 / S2S_BF16.  Asynchronous on `stream`. */
int s2s_prefill_rope(s2s_ctx* ctx, void* qkv, int32_t n, int32_t heads, int32_t kv_heads, int32_t hd, int32_t past,
                     const float* rope, int32_t max_pos, const float* q_norm, const float* k_norm, float eps, void* kcache,
                     void* vcache, int32_t dtype, void* stream);
/* The greedy token choice after a prefill by itself (exposed for tests): *out_d = the argmax of logits_d[0..n), the lowest
 * id among equal maxima; NaN entries count as -inf, so a row without a number above -inf gives 0.  S2S_ERR_INVALID on
 * n < 1 or a null pointer.  Asynchronous on `stream`. */
int s2s_argmax_row(s2s_ctx* ctx, const float* logits_d, int32_t n, int32_t* out_d, void* stream);

/* ---- Llama-family LLM ------------------------------------------------------------------ */
typedef struct {
  int32_t d_model, layers, heads, kv_heads, head_dim, ffn, vocab;
  float rope_theta, rms_eps;
  int32_t compute_dtype;  /* S2S_BF16 (default) or S2S_F16 */
  int32_t max_sessions;   /* KV-cache slots */
  int32_t max_positions;  /* per session */
  int32_t max_prefill;    /* longest prompt chunk per call */
  int32_t qk_norm;        /* 1 = Qwen3-style per-head RMSNorm(head_dim) on q,k before RoPE (transformers
                             modeling_qwen3.py Qwen3Attention: the reference's default LLM family and the TTS talker); 0 = Llama */
  int32_t n_tables;       /* 0/1 = one embedding table + one output head; >1 = one pair per codebook
                             ("model.embed_tokens.<i>.weight", "lm_head.<i>.weight"), used by the TTS code predictor */
} s2s_llama_config;

int s2s_llama_create(s2s_ctx* ctx, const s2s_llama_config* cfg, s2s_llama** out);
int s2s_llama_destroy(s2s_llama* m);
int s2s_llama_bind_tensor(s2s_llama* m, const char* name, const void* data_h, const int64_t* shape,
                          int32_t ndim, int32_t dtype);
int s2s_llama_init_random(s2s_llama* m, uint64_t seed);
/* Storage format of the projection matrices (q/k/v, o, gate/up, down of every layer) and lm_head.  The model holds ONE copy
 * of them, in the tiled layout of s2s_tile_weights, which both the prefill GEMMs and the decode launch read; the embedding
 * table stays row-major, and a tied lm_head is tiled from it.  `format` = the model's compute_dtype (the default) or
 * S2S_FP8_E4M3: weight-only FP8 with one power-of-two scale per weight row, quantised from each bound 16-bit tensor as it
 * is bound.  Prefill expands the codes to the dequantised values, so prefill and decode run ONE model: bit for bit the
 * 16-bit engine bound to those dequantised weights, and a different model from the checkpoint's.  Halves the weight bytes
 * a decode step streams and the device memory of those matrices.  Call after create and before the first bind_tensor,
 * init_random or finalize (S2S_ERR_INVALID afterwards: the matrices are allocated in the format then in force); FP8 needs
 * bf16 compute and a single-table model (S2S_ERR_UNSUPPORTED otherwise). */
int s2s_llama_set_weight_format(s2s_llama* m, int32_t format);
int32_t s2s_llama_weight_format(s2s_llama* m);
int s2s_llama_finalize(s2s_llama* m);
int s2s_llama_create_shared(s2s_ctx* ctx, s2s_llama* source, const s2s_llama_config* cfg, s2s_llama** out);
/* Device bytes the model object holds: *weights = embedding table(s), norms and the tiled matrices; *total = that plus the
 * KV cache and every workspace (for an object sharing its weights, see shared weights).  The staging buffer of bind_tensor / init_random (as large as the largest matrix tensor)
 * is held from the first bind to finalize and is not counted. */
int s2s_llama_device_bytes(s2s_llama* m, int64_t* weights, int64_t* total);
/* Reset a KV-cache slot (new response).  Also empties the slot's seen-id set (repetition penalty), on the stream of the
 * slot's next prefill or decode. */
int s2s_llama_session_reset(s2s_llama* m, int32_t slot);
/* Token choice of a slot, in transformers' logits-processor order (generation/utils.py _get_logits_processor):
 * repetition penalty over every id the slot has seen (prompt and generated), EOS ids masked until min_new_tokens tokens were
 * produced since the slot's last prefill, then only when do_sample: temperature, top-k (0 = off), top-p (1 = off) and a
 * Gumbel-max draw whose uniforms come from Philox4x64-10 keyed by `seed` with counter (token id, position of the predicted
 * token) -- numpy.random.Philox(key=seed, counter=[id, position, 0, 0]), first output -- so a token depends only on (seed,
 * position, logits).  NULL = greedy argmax, which is also the state after create.  Every prefill adds its prompt ids to the
 * seen set; a token joins it when it is fed to a decode launch of a slot with a penalty (the choice after an intermediate
 * chunk of a long prompt does not).  Set it before the prefill of a response.                                          */
typedef struct {
  int32_t do_sample;
  float temperature;          /* > 0 when do_sample */
  int32_t top_k;              /* >= 0; 0 or >= vocab = off */
  float top_p;                /* (0, 1]; 1 = off */
  float repetition_penalty;   /* > 0; 1 = off */
  int32_t min_new_tokens;     /* >= 0 */
  int32_t n_eos;              /* <= 8 */
  int32_t eos_ids[8];
  uint64_t seed;
} s2s_sampling;
int s2s_llama_set_sampling(s2s_llama* m, int32_t slot, const s2s_sampling* s);
/* Prefill `n` prompt tokens (host ids) into `slot`; logits_out_d optional [n, vocab] f32;
 * next_id_d optional [1] i32 = the token chosen from the last position (argmax, or the slot's s2s_llama_set_sampling). */
int s2s_llama_prefill(s2s_llama* m, int32_t slot, const int32_t* ids_h, int32_t n, float* logits_out_d,
                      int32_t* next_id_d, void* stream);
/* Prefill of B sessions in ONE pass over the weights (the reference prefills one request per pipeline call,
 * LLM/language_model.py:883-888): ids_h holds the sessions' new prompt tokens back to back (n_h[b] tokens for slot slots_h[b],
 * sum <= max_prefill, B <= 16); the projections and the MLP run over all rows at once, RoPE / KV append / causal attention per
 * session.  next_ids_d [B] receives each session's next token (chosen as by s2s_llama_prefill).  Rows of a session produce the same values as
 * s2s_llama_prefill up to the tile shape the GEMM picks for the row count. */
int s2s_llama_prefill_batch(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* ids_h, const int32_t* n_h,
                            int32_t* next_ids_d, void* stream);

/* Decode for B (<= s2s_llama_max_decode_batch: 16, also for Llama-3-8B) sessions in one persistent launch, each token chosen as
 * its slot's s2s_llama_set_sampling says (argmax by default).  slots_h[B]; first_ids_d[B] are the tokens to
 * feed first (the prefill's choice); ids_out_d [B, n_steps] receives the n_steps tokens generated AFTER them; eos stops
 * a row (eos_id < 0 disables); forced_d optional [B, n_steps] teacher-forced feedback; logits_out_d optional
 * [n_steps, B, vocab].                                                                              */
int s2s_llama_decode(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* first_ids_d,
                     int32_t n_steps, int32_t eos_id, int32_t* ids_out_d, int32_t* len_out_d,
                     const int32_t* forced_d, float* logits_out_d, void* stream);
/* Profiling aid: the stamps of s2s_whisper_set_trace, trace_d[2][capacity][6] (stamp 1, inputs staged, stays 0). */
int s2s_llama_set_trace(s2s_llama* m, uint64_t* trace_d, int32_t capacity);
/* Largest B accepted by s2s_llama_decode for this geometry (shared-memory budget of the decode kernel, <= 16). */
int32_t s2s_llama_max_decode_batch(s2s_llama* m);
/* End-to-end with HOST buffers: (chunked) prefill + decode with the slot's token choice, synchronous.  ids_out_h[0] is
 * the token chosen from the prompt's last position, n_steps tokens in total (generate() semantics of the reference's pipeline call). */
int s2s_llama_generate(s2s_llama* m, int32_t slot, const int32_t* prompt_h, int32_t n_prompt, int32_t n_steps,
                       int32_t eos_id, int32_t* ids_out_h, int32_t* len_out_h, void* stream);

/* ---- TTS codec decoder: codebook ids -> 24 kHz waveform ---------------------------------------------
 * Replaces the codec-decode half of faster-qwen3-tts' `generate_*_streaming` (called from
 * S/TTS/qwen3_tts_handler.py:930-942, 968-976, 994-1001; the package is absent everywhere, so the arithmetic is pinned to
 * the published cousin transformers Qwen3OmniMoeCode2Wav, modeling_qwen3_omni_moe.py:3283-3790 -- unpinned vs upstream). */
typedef struct {
  int32_t codebook_size, hidden, heads, kv_heads, inter, layers, quantizers;
  int32_t n_upsample_rates, upsample_rates[8];       /* decoder blocks: (8, 5, 4, 3) */
  int32_t n_upsampling_ratios, upsampling_ratios[4]; /* ConvNeXt upsamplers: (2, 2)  */
  int32_t decoder_dim, sliding_window;
  float rope_theta, rms_eps;
  int32_t max_frames;   /* longest decode call: left context + chunk (33 for chunk_size 8 behind 25 frames of history) */
  int32_t max_batch;    /* sequences decoded by one launch sequence (concurrently speaking sessions, <= 16; 0 = 1) */
  int32_t precision;    /* 0 = fp32 FMA everywhere (the reference slot's `parity_mode`, qwen3_tts_arguments.py:99-101: waveform
                           within 1e-3 of the fp32 oracle); 1 = contractions on the tensor cores with fp16 operands and fp32
                           accumulation (waveform within 1e-2) */
} s2s_codec_config;
typedef struct s2s_codec s2s_codec;
int s2s_codec_create(s2s_ctx* ctx, const s2s_codec_config* cfg, s2s_codec** out);
int s2s_codec_destroy(s2s_codec* m);
/* names = the cousin's state dict ("code_embedding.weight", "pre_transformer.layers.0.self_attn.q_proj.weight", ...) */
int s2s_codec_bind_tensor(s2s_codec* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                          int32_t dtype);
int s2s_codec_init_random(s2s_codec* m, uint64_t seed);
int s2s_codec_finalize(s2s_codec* m);
/* codes_d [T][quantizers] i32 (frame-major) -> wav_out_d f32: the samples of frames [ctx_frames, T), i.e. one step of
 * Qwen3OmniMoeCode2Wav.chunked_decode (:3779-3790).  wav_out_d must hold s2s_codec_samples(m, T) floats;
 * *n_out_h = samples written; hidden_out_d optional [T, hidden] (pre-transformer output, for tests). */
int s2s_codec_decode(s2s_codec* m, const int32_t* codes_d, int32_t T, int32_t ctx_frames, float* wav_out_d,
                     int32_t* n_out_h, float* hidden_out_d, void* stream);
int32_t s2s_codec_samples(s2s_codec* m, int32_t T);   /* waveform length of a T-frame decode before the context drop */
int32_t s2s_codec_total_upsample(s2s_codec* m);       /* samples per frame (1920) */

/* One contraction of the codec decoder (exposed for tests / benches), on a chosen kernel:
 *   Y[t, n] = epi( bias[n % bias_mod] + sum_{j < k} sum_{c < C_in} X[t + x_row0 + j * dil, c] * W[j][c][n] )
 * for t in [t0, T_out) and n < N of each of `batch` sequences (sequence b: x + b * x_bs, y + b * y_bs, resid + b * r_bs;
 * all strides in elements).  Rows of X outside [0, T_in) read as zero.  X is [T_in rows, ldx] f32, W is [k][C_in][N] f32
 * (tap-major; a transposed convolution of stride s with kernel 2 s is the 2-tap contraction with N = s * C_out whose
 * [T_in - 1, s * C_out] output is the time-major [(T_in - 1) * s, C_out] result), bias [bias_mod] or NULL.  epi: act
 * (0 none, 1 exact GELU, 2 SiLU), then * scale[n] (scale NULL = 1), then + resid[t, n] (resid may alias y; NULL = 0).
 * Rows below t0, columns in [N, ldy) and rows past T_out are not written.
 * path 0: fp32 FMA (conv1d_f32_kernel); 1: tensor cores, fp16 operands converted while staged (conv1d_tc_kernel);
 * 2: tensor cores fed from x16, an fp16 copy of X with the same shape and strides (conv1d_tc16_kernel; needs
 * C_in % 8 == 0, N % 4 == 0, ldx % 8 == 0, x_bs % 8 == 0).  Paths 1 and 2 pack W into fp16 k-pairs in scratch memory of
 * their own.  Synchronous: returns after the stream has finished the contraction. */
typedef struct {
  const float* x; int64_t ldx; int32_t T_in; int32_t x_row0;
  const void* x16;
  const float* w; int32_t k, dil, C_in, N;
  const float* bias; int32_t bias_mod;
  int32_t act;
  const float* scale;
  const float* resid; int64_t ldr;
  float* y; int64_t ldy; int32_t T_out;
  int32_t t0;
  int32_t batch; int64_t x_bs, y_bs, r_bs;
} s2s_conv_args;
int s2s_codec_contract(s2s_ctx* ctx, const s2s_conv_args* args, int32_t path, void* stream);

/* ---- Qwen3-TTS talker + code predictor: text -> codebook ids, 12.5 frames per second of speech ------------------
 * Replaces the autoregressive half of faster-qwen3-tts' `generate_custom_voice_streaming(text, speaker, language,
 * instruct, chunk_size, max_new_tokens, non_streaming_mode)` (S/TTS/qwen3_tts_handler.py:946-978; warm-up :555-572).
 * The package is absent everywhere; the arithmetic is pinned to the published cousin, the Qwen3-Omni talker in
 * transformers (modeling_qwen3_omni_moe.py: talker :3029-3281, code predictor :2550-2731, prompt layout :3842-3905) with
 * a dense talker MLP (oracle/qwen3tts_ref.py) -- UNPINNED against the real Qwen3-TTS.  Codes are chosen greedily unless
 * s2s_qwen3tts_set_sampling asks for the cousin's sampling.
 * One frame = 1 talker step (first codebook, special ids suppressed) + n_groups code-predictor steps (residual
 * codebooks) + the next talker input (sum of the frame's code embeddings + the next text embedding / tts_pad). */
typedef struct {
  /* talker (Qwen3-style decoder over the codec vocabulary) */
  int32_t d_model, layers, heads, kv_heads, head_dim, ffn, vocab;
  /* code predictor (same width; one embedding table and one head per residual codebook) */
  int32_t cp_layers, cp_heads, cp_kv_heads, cp_head_dim, cp_ffn, cp_vocab;
  int32_t n_groups;                      /* codebooks per frame (16) */
  int32_t text_vocab, text_hidden;       /* text-side embedding table and its width (thinker_hidden_size) */
  float rope_theta, rms_eps;
  int32_t compute_dtype;                 /* S2S_BF16 / S2S_F16 for the decoder weights; projections / glue fp32 */
  int32_t max_sessions, max_positions, max_text;
  int32_t codec_eos, codec_nothink, codec_think_bos, codec_think_eos, codec_pad, codec_bos;
  int32_t tts_bos, tts_eos, tts_pad, im_start, assistant, newline;
  s2s_codec_config codec;                /* the waveform decoder owned by the same model object */
} s2s_qwen3tts_config;
typedef struct s2s_qwen3tts s2s_qwen3tts;
int s2s_qwen3tts_create(s2s_ctx* ctx, const s2s_qwen3tts_config* cfg, s2s_qwen3tts** out);
int s2s_qwen3tts_destroy(s2s_qwen3tts* m);
/* names: the cousin's talker state dict ("model.layers.0.self_attn.q_proj.weight", "model.codec_embedding.weight",
 * "codec_head.weight", "text_projection.linear_fc1.weight", "code_predictor.model.layers...",
 * "code_predictor.model.codec_embedding.<i>.weight", "code_predictor.lm_head.<i>.weight"), "text_embedding.weight", and
 * the codec decoder's names prefixed with "code2wav.". */
int s2s_qwen3tts_bind_tensor(s2s_qwen3tts* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                             int32_t dtype);
int s2s_qwen3tts_init_random(s2s_qwen3tts* m, uint64_t seed);
int s2s_qwen3tts_finalize(s2s_qwen3tts* m);
int s2s_qwen3tts_create_shared(s2s_ctx* ctx, s2s_qwen3tts* source, const s2s_qwen3tts_config* cfg, s2s_qwen3tts** out);
/* talker, code predictor, codec and text side together, with the meaning of s2s_llama_device_bytes (see shared weights) */
int s2s_qwen3tts_device_bytes(s2s_qwen3tts* m, int64_t* weights, int64_t* total);
/* Start an utterance in `slot`: builds the prompt ([im_start, assistant, newline] + text, codec prefix with the speaker
 * id), prefills the talker and stages the first frame's input.  text_ids_h: >= 1 text token ids.  Resets the slot's
 * token choice to greedy and empties its repetition-penalty set. */
int s2s_qwen3tts_prefill(s2s_qwen3tts* m, int32_t slot, const int32_t* text_ids_h, int32_t n_text, int32_t speaker_id,
                         void* stream);
/* Token choice of the utterance just prefilled in `slot` (call it after s2s_qwen3tts_prefill); NULL = greedy argmax.
 * The fields and range checks are those of s2s_llama_set_sampling, in the same logits-processor order (the talker's
 * suppressed special ids are -inf before any of it).  min_new_tokens must be 0 and the EOS ids are ignored: codec_eos is
 * the only stop.  The code predictor has no repetition penalty (anything but 1 is rejected).  The talker's penalty acts on
 * the first codes of the frames kept since prefill (the forced ones under teacher forcing), not on the prompt's codec ids
 * (the cousin's talker.generate gets no input_ids).  Draws: Philox4x64-10 keyed by the struct's seed (pass the same seed to
 * both) with counter [id, position, stream, 0] -- talker: stream 0, position of the predicted code in the talker's
 * sequence; predictor: stream 1 + the frame's index since prefill, position of the predicted code in the predictor's
 * sequence -- so a session's codes do not depend on its batch or on how its frames are split into calls. */
int s2s_qwen3tts_set_sampling(s2s_qwen3tts* m, int32_t slot, const s2s_sampling* talker, const s2s_sampling* predictor);
/* Generate n_frames frames for the B (<= s2s_qwen3tts_max_batch) sessions slots_h[B] in lock step: 3 persistent
 * launches per frame serve all of them.  codes_out_d [B][n_frames][n_groups] i32.  A session whose first code is
 * codec_eos has finished: the caller drops that frame and everything after it (frames_done is not advanced past it).
 * forced_codes_d (optional, [B][n_frames][n_groups]): teacher-forced feedback for parity tests -- the reported codes are
 * still the models' own decisions, the given codes are what is fed forward and kept.  Asynchronous on `stream`. */
int s2s_qwen3tts_decode_frames(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_frames,
                               int32_t* codes_out_d, const int32_t* forced_codes_d, void* stream);
/* Test hook: s2s_qwen3tts_decode_frames plus the logits rows each code was chosen from (optional, NULL = not stored):
 * talker_logits_out_d [n_frames][B][vocab] (suppressed ids -inf) and pred_logits_out_d [n_frames][n_groups][B][cp_vocab]
 * (step 0 predicts nothing and is left unwritten). */
int s2s_qwen3tts_decode_frames_logits(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_frames,
                                      int32_t* codes_out_d, const int32_t* forced_codes_d, float* talker_logits_out_d,
                                      float* pred_logits_out_d, void* stream);
/* Waveform of the newest `n_new` frames of `slot` (codes kept by the library since prefill), decoded behind up to
 * `left_context` frames of history (Qwen3OmniMoeCode2Wav.chunked_decode); wav_out_d f32 [n_new * 1920 (max)]. */
int s2s_qwen3tts_decode_audio(s2s_qwen3tts* m, int32_t slot, int32_t n_new, int32_t left_context, float* wav_out_d,
                              int32_t* n_out_h, void* stream);
/* The same for B sessions whose chunks have the same shape (same n_new and the same amount of history): ONE launch sequence,
 * the linear layers see B x T rows.  wav_out_d + b * wav_stride receives session b's samples. */
int s2s_qwen3tts_decode_audio_batch(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_new, int32_t left_context,
                                    float* wav_out_d, int64_t wav_stride, int32_t* n_out_h, void* stream);
/* Tell the library how many frames of `slot` are valid (after the caller saw codec_eos inside a chunk). */
int s2s_qwen3tts_set_frames(s2s_qwen3tts* m, int32_t slot, int32_t n_frames);
int32_t s2s_qwen3tts_frames(s2s_qwen3tts* m, int32_t slot);
int32_t s2s_qwen3tts_max_batch(s2s_qwen3tts* m);
/* Profiling aid (see s2s_llama_set_trace): phase stamps of the talker (which = 0) or code-predictor (1) launches,
 * trace_d[2][capacity][6]. */
int s2s_qwen3tts_set_trace(s2s_qwen3tts* m, int32_t which, uint64_t* trace_d, int32_t capacity);
s2s_codec* s2s_qwen3tts_codec(s2s_qwen3tts* m);

/* ---- TTS post-processing (Qwen3TTSHandler._stream) -------------------------------------
 * wav24k_d f32[n] -> polyphase resample 24k->16k (scipy.signal.resample_poly(x, 2, 3) taps supplied by
 * the host mirror) -> clip(x*32768) -> int16.  out16k_d must hold ceil(n*2/3) samples.          */
int s2s_tts_postproc(s2s_ctx* ctx, const float* wav24k_d, int32_t n, const float* taps_d, int32_t n_taps,
                     int16_t* out16k_d, int32_t* n_out_h, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* S2S_B200_H */
