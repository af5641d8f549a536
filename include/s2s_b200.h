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

/* ---- generic GEMM (exposed for tests / roofline benches) --------------------------------
 * C[M,N] = A[M,K] * W[N,K]^T (+bias), wgmma + TMA; dtype S2S_F16 or S2S_BF16, fp32 accumulate.
 * out_dtype: S2S_F32 or same as dtype.  act: 0 none, 1 exact GELU.                          */
int s2s_gemm(s2s_ctx* ctx, const void* a_d, const void* w_d, const float* bias_d, void* c_d, int32_t M,
             int32_t N, int32_t K, int32_t dtype, int32_t out_dtype, int32_t act, void* stream);
/* O = softmax(Q K^T * scale [+causal]) V ; q/k/v/o row-major [T, heads*hd] slices with row strides
 * (elements); kv_heads <= heads (GQA).  hd in {64, 128}.                                     */
int s2s_attention(s2s_ctx* ctx, const void* q_d, const void* k_d, const void* v_d, void* o_d, int32_t B,
                  int32_t Tq, int32_t Tk, int32_t heads, int32_t kv_heads, int32_t hd, int64_t ldq,
                  int64_t ldk, int64_t ldv, int64_t ldo, float scale, int32_t causal, int32_t dtype,
                  void* stream);

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
int s2s_llama_finalize(s2s_llama* m);
/* Reset a KV-cache slot (new response). */
int s2s_llama_session_reset(s2s_llama* m, int32_t slot);
/* Prefill `n` prompt tokens (host ids) into `slot`; logits_out_d optional [n, vocab] f32;
 * next_id_d optional [1] i32 = argmax of the last position.                                 */
int s2s_llama_prefill(s2s_llama* m, int32_t slot, const int32_t* ids_h, int32_t n, float* logits_out_d,
                      int32_t* next_id_d, void* stream);
/* Prefill of B sessions in ONE pass over the weights (the reference prefills one request per pipeline call,
 * LLM/language_model.py:883-888): ids_h holds the sessions' new prompt tokens back to back (n_h[b] tokens for slot slots_h[b],
 * sum <= max_prefill, B <= 16); the projections and the MLP run over all rows at once, RoPE / KV append / causal attention per
 * session.  next_ids_d [B] receives each session's greedy next token.  Rows of a session produce the same values as
 * s2s_llama_prefill up to the tile shape the GEMM picks for the row count. */
int s2s_llama_prefill_batch(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* ids_h, const int32_t* n_h,
                            int32_t* next_ids_d, void* stream);

/* Greedy decode for B (<= s2s_llama_max_decode_batch: 16, 4 for Llama-3-8B) sessions in one persistent launch.  slots_h[B]; first_ids_d[B] are the tokens to
 * feed first (the prefill argmax); ids_out_d [B, n_steps] receives the n_steps tokens generated AFTER them; eos stops
 * a row (eos_id < 0 disables); forced_d optional [B, n_steps] teacher-forced feedback; logits_out_d optional
 * [n_steps, B, vocab].                                                                              */
int s2s_llama_decode(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* first_ids_d,
                     int32_t n_steps, int32_t eos_id, int32_t* ids_out_d, int32_t* len_out_d,
                     const int32_t* forced_d, float* logits_out_d, void* stream);
/* Profiling aid (see s2s_whisper_set_trace): CTA 0's [phase begin, body end, barrier exit] stamps, trace_d[capacity][3]. */
int s2s_llama_set_trace(s2s_llama* m, uint64_t* trace_d, int32_t capacity);
/* Largest B accepted by s2s_llama_decode for this geometry (shared-memory budget of the decode kernel, <= 16). */
int32_t s2s_llama_max_decode_batch(s2s_llama* m);
/* End-to-end with HOST buffers: (chunked) prefill + greedy decode, synchronous.  ids_out_h[0] is the argmax of the
 * prompt's last position, n_steps tokens in total (generate() semantics of the reference's pipeline call). */
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

/* ---- Qwen3-TTS talker + code predictor: text -> codebook ids, 12.5 frames per second of speech ------------------
 * Replaces the autoregressive half of faster-qwen3-tts' `generate_custom_voice_streaming(text, speaker, language,
 * instruct, chunk_size, max_new_tokens, non_streaming_mode)` (S/TTS/qwen3_tts_handler.py:946-978; warm-up :555-572).
 * The package is absent everywhere; the arithmetic is pinned to the published cousin, the Qwen3-Omni talker in
 * transformers (modeling_qwen3_omni_moe.py: talker :3029-3281, code predictor :2550-2731, prompt layout :3842-3905) with
 * a dense talker MLP and greedy selection (oracle/qwen3tts_ref.py) -- UNPINNED against the real Qwen3-TTS.
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
/* Start an utterance in `slot`: builds the prompt ([im_start, assistant, newline] + text, codec prefix with the speaker
 * id), prefills the talker and stages the first frame's input.  text_ids_h: >= 1 text token ids. */
int s2s_qwen3tts_prefill(s2s_qwen3tts* m, int32_t slot, const int32_t* text_ids_h, int32_t n_text, int32_t speaker_id,
                         void* stream);
/* Generate n_frames frames for the B (<= s2s_qwen3tts_max_batch) sessions slots_h[B] in lock step: 3 persistent
 * launches per frame serve all of them.  codes_out_d [B][n_frames][n_groups] i32.  A session whose first code is
 * codec_eos has finished: the caller drops that frame and everything after it (frames_done is not advanced past it).
 * forced_codes_d (optional, [B][n_frames][n_groups]): teacher-forced feedback for parity tests -- the reported codes are
 * still the models' own decisions, the given codes are what is fed forward and kept.  Asynchronous on `stream`. */
int s2s_qwen3tts_decode_frames(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_frames,
                               int32_t* codes_out_d, const int32_t* forced_codes_d, void* stream);
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
/* Profiling aid (see s2s_llama_set_trace): phase stamps of the talker (which = 0) or code-predictor (1) launches. */
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
