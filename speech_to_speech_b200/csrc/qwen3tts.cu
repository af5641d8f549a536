// qwen3tts.cu -- Qwen3-TTS talker + code predictor behind the C ABI: text ids -> 16 codebook ids per 12.5 Hz frame.
//
// Reference path: Qwen3TTSHandler._process_custom_voice -> model.generate_custom_voice_streaming(text, speaker, ...,
// chunk_size, max_new_tokens) (S/TTS/qwen3_tts_handler.py:946-978).  The arithmetic lives in the absent
// faster-qwen3-tts; it is pinned to the published cousin (transformers Qwen3-Omni talker, modeling_qwen3_omni_moe.py)
// through oracle/qwen3tts_ref.py -- dense talker MLP, greedy selection by default, the cousin's sampling on request
// (s2s_qwen3tts_set_sampling) -- and UNPINNED against the real upstream.
//
// Both models are Qwen3-style decoders, i.e. the Llama-family engine of llama.cu with qk_norm:
//   talker    : s2s_llama over the codec vocabulary, driven by EMBEDDINGS: the prompt rows are prefilled through the
//               wgmma GEMM path (llama_prefill_rows), every frame is one step of the persistent decode kernel with
//               x_in = sum of the previous frame's 16 code embeddings + the next text embedding;
//   predictor : s2s_llama with one embedding table / output head per residual codebook (multi-table mode): one persistent
//               launch of n_groups steps per frame: [talker hidden, embed(code0)] then one step per residual codebook.
// A frame for up to 16 sessions is 3 persistent launches + 3 small glue kernels; nothing synchronises with the host.
// Sampling (sampling.cuh): the talker's draws use Philox stream 0 at the talker position, the predictor's stream 1 + the
// frame's index since prefill at the predictor position, so a session's codes depend only on (seed, prompt, settings),
// not on its batch or on how its frames are split into calls.  The talker's repetition penalty acts on the first codes of
// the frames kept since prefill: frame_finish_kernel adds each kept code0, the decode launch adds nothing (seen_fixed).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "codec_decode.cuh"
#include "kernels.cuh"
#include "llama_model.cuh"
#include "weight_arena.cuh"

extern "C" {
int s2s_llama_create(s2s_ctx* ctx, const s2s_llama_config* cfg, s2s_llama** out);
int s2s_llama_create_shared(s2s_ctx* ctx, s2s_llama* source, const s2s_llama_config* cfg, s2s_llama** out);
int s2s_llama_device_bytes(s2s_llama* m, int64_t* weights, int64_t* total);
int s2s_llama_destroy(s2s_llama* m);
int s2s_llama_bind_tensor(s2s_llama* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim, int32_t dtype);
int s2s_llama_init_random(s2s_llama* m, uint64_t seed);
int s2s_llama_finalize(s2s_llama* m);
}

namespace {

constexpr int TTS_MAX_B = LLAMA_MAX_DEC_B;
constexpr int PROMPT_ROWS = 9;   // transformers _get_talker_assistant_parts: 3 role tokens, 4 pads, bos, first text token

struct TtsBatch {   // passed by value to the glue kernels: no host <-> device synchronisation per frame
  int slot[TTS_MAX_B], pos0[TTS_MAX_B], frames0[TTS_MAX_B], n_trailing[TTS_MAX_B];
};

template <typename T>
__global__ void gather_rows_f32_kernel(const int* __restrict__ ids, const T* __restrict__ table, int d, float* __restrict__ out) {
  const T* e = table + (long long)ids[blockIdx.x] * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) out[(long long)blockIdx.x * d + i] = DT<T>::to_f(e[i]);
}

// Prompt rows (oracle build_prompt): P = projected [im_start, assistant, newline, text..., tts_bos, tts_eos, tts_pad].
//   rows 0-2: P[0..2]            rows 3-6: pad + E[nothink, think_bos, think_eos, speaker]
//   row 7   : bos + E[codec_pad] row 8   : P[3] + E[codec_bos]   (row 8 becomes the first frame's input)
//   trailing: P[4 .. n_text + 2], then eos
template <typename T>
__global__ void build_prompt_kernel(const float* __restrict__ P, int n_text, const T* __restrict__ codec_embed, int d,
                                    int nothink, int think_bos, int think_eos, int speaker, int cpad, int cbos,
                                    float* __restrict__ rows8, float* __restrict__ xnext, float* __restrict__ trailing) {
  const int r = blockIdx.x;   // 0 .. PROMPT_ROWS - 1 prompt rows, then n_text trailing rows
  const float* bos = P + (long long)(n_text + 3) * d;
  const float* eos = P + (long long)(n_text + 4) * d;
  const float* pad = P + (long long)(n_text + 5) * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    if (r < PROMPT_ROWS) {
      float v;
      int cid = -1;
      if (r < 3) v = P[(long long)r * d + i];
      else if (r < 7) { v = pad[i]; cid = r == 3 ? nothink : r == 4 ? think_bos : r == 5 ? think_eos : speaker; }
      else if (r == 7) { v = bos[i]; cid = cpad; }
      else { v = P[(long long)3 * d + i]; cid = cbos; }
      if (cid >= 0) v += DT<T>::to_f(codec_embed[(long long)cid * d + i]);
      if (r < PROMPT_ROWS - 1) rows8[(long long)r * d + i] = v; else xnext[i] = v;
    } else {
      const int t = r - PROMPT_ROWS;   // trailing row t
      trailing[(long long)t * d + i] = (t < n_text - 1) ? P[(long long)(4 + t) * d + i] : eos[i];
    }
  }
}

// before the talker step of frame f: inputs, cache slots and positions of the batch
__global__ void frame_prepare_kernel(TtsBatch tb, int f, const float* __restrict__ xnext_all, int d, float* __restrict__ x_in,
                                     int* __restrict__ slot_d, int* __restrict__ pos_d) {
  const int b = blockIdx.x;
  const float* src = xnext_all + (long long)tb.slot[b] * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) x_in[(long long)b * d + i] = src[i];
  if (threadIdx.x == 0) { slot_d[b] = tb.slot[b]; pos_d[b] = tb.pos0[b] + f; }
}

// between talker and predictor: predictor input 0 = final-norm(talker hidden) (the cousin feeds hidden_states[-1], which
// transformers ties to the post-norm last_hidden_state); predictor cache slot = batch index, position 0
__global__ void frame_mid_kernel(const float* __restrict__ hidden, const float* __restrict__ norm_w, float eps, int d,
                                 float* __restrict__ x_in_p, int* __restrict__ pslot_d, int* __restrict__ ppos_d,
                                 const int* __restrict__ code0, const int* __restrict__ forced /*[B][n_frames][G] or null*/, int f,
                                 int n_frames, int G, int* __restrict__ code0_feed, int* __restrict__ forced_frame /*[B][G]*/,
                                 SampSlot* __restrict__ psamp /*[B] or null*/, TtsBatch tb) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* h = hidden + (long long)b * d;
  float ss = 0.f;
  for (int i = threadIdx.x; i < d; i += blockDim.x) ss = fmaf(h[i], h[i], ss);
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const float r = 1.0f / sqrtf(tot / (float)d + eps);
  for (int i = threadIdx.x; i < d; i += blockDim.x) x_in_p[(long long)b * d + i] = norm_w[i] * (h[i] * r);
  if (threadIdx.x == 0) { pslot_d[b] = b; ppos_d[b] = 0; }
  // the predictor's positions restart every frame: its draws take the frame's own Philox stream
  // (frames since prefill = talker positions since prefill: set_frames after codec_eos does not move it)
  if (threadIdx.x == 0 && psamp) psamp[b].stream = 1ull + (unsigned long long)(tb.pos0[b] - (PROMPT_ROWS - 1) + f);
  // teacher forcing (parity tests): the code predictor is fed the given codes of this frame, its own argmax is still reported
  if (threadIdx.x < G) {
    if (forced) forced_frame[b * G + threadIdx.x] = forced[((long long)b * n_frames + f) * G + threadIdx.x];
    if (threadIdx.x == 0) code0_feed[b] = forced ? forced[((long long)b * n_frames + f) * G] : code0[b];
  }
}

// after the predictor: record the frame's codes and build the next talker input
//   xnext = E_talker[code0] + sum_{i >= 1} E_pred[i - 1][code_i] + (trailing[frame] | tts_pad)
template <typename T>
__global__ void frame_finish_kernel(TtsBatch tb, int f, int n_frames, int G, const int* __restrict__ pcodes /*[B][G]*/,
                                    const int* __restrict__ code0 /*[B] talker argmax*/, const int* __restrict__ forced_frame /*[B][G] or null*/,
                                    const T* __restrict__ talker_embed, const T* __restrict__ pred_embed, long long pred_stride,
                                    int d, const float* __restrict__ trailing_all, long long trailing_stride,
                                    const float* __restrict__ pad_all, float* __restrict__ xnext_all,
                                    int* __restrict__ codes_out, int* __restrict__ history, long long history_stride,
                                    unsigned int* __restrict__ tseen, int seen_words) {
  const int b = blockIdx.x, slot = tb.slot[b], fa = tb.frames0[b] + f;
  // reported: the models' own decisions (talker argmax, predictor argmaxes); fed forward / kept: the forced codes if given
  const int* pc = forced_frame ? forced_frame + b * G : pcodes + b * G;
  if (threadIdx.x < G) {
    codes_out[((long long)b * n_frames + f) * G + threadIdx.x] = threadIdx.x == 0 ? code0[b] : pcodes[b * G + threadIdx.x];
    history[(long long)slot * history_stride + (long long)fa * G + threadIdx.x] = pc[threadIdx.x];
  }
  // the kept first code joins the slot's talker seen set (repetition penalty over the generated code0s only)
  if (threadIdx.x == 0) atomicOr(tseen + (long long)slot * seen_words + (pc[0] >> 5), 1u << (pc[0] & 31));
  const float* extra = fa < tb.n_trailing[b] ? trailing_all + (long long)slot * trailing_stride + (long long)fa * d
                                              : pad_all + (long long)slot * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float v = DT<T>::to_f(talker_embed[(long long)pc[0] * d + i]);
    for (int g = 1; g < G; ++g) v += DT<T>::to_f(pred_embed[(long long)(g - 1) * pred_stride + (long long)pc[g] * d + i]);
    xnext_all[(long long)slot * d + i] = v + extra[i];
  }
}

}  // namespace

struct s2s_qwen3tts {
  s2s_ctx* ctx = nullptr;
  s2s_qwen3tts_config cfg{};
  bool finalized = false;
  s2s_llama *talker = nullptr, *pred = nullptr;
  CodecDecoder* codec = nullptr;
  WeightArena arena;   // the text side's tensors and every buffer below
  // text side
  void* text_embed = nullptr;                    // [text_vocab, text_hidden] 16-bit
  float *fc1_w = nullptr, *fc1_b = nullptr, *fc2_w = nullptr, *fc2_b = nullptr;   // [K][N] layouts
  // per session
  struct Sess { int n_trailing = 0, frames = 0, pos = 0; bool active = false; };
  std::vector<Sess> sess;
  float *trailing = nullptr, *pad_embed = nullptr, *xnext = nullptr;
  int* history = nullptr;
  long long trailing_stride = 0, history_stride = 0;
  // prefill workspace
  int* ids_d = nullptr;
  float *emb_rows = nullptr, *proj_mid = nullptr, *proj_out = nullptr;
  // frame workspace
  float *x_in_t = nullptr, *hidden = nullptr, *x_in_p = nullptr;
  int *tslot_d = nullptr, *tpos_d = nullptr, *pslot_d = nullptr, *ppos_d = nullptr, *code0 = nullptr, *pcodes = nullptr,
      *tlen = nullptr, *plen = nullptr, *code0_feed = nullptr, *forced_frame = nullptr;
  unsigned char* suppress = nullptr;
  // token choice per slot (s2s_qwen3tts_set_sampling); reset to greedy by every prefill
  std::vector<SampSlot> tsamp, psamp;   // [max_sessions] talker, code predictor
  SampSlot* samp_d = nullptr;           // [2][TTS_MAX_B] the call's packed talker | predictor parameters
};

namespace {

int tts_max_batch(const s2s_qwen3tts* m) {
  return std::min(TTS_MAX_B, std::min(llama_max_decode_batch_of(m->talker), llama_max_decode_batch_of(m->pred)));
}

int linear_f32(const float* x, int T, int K, const float* w, const float* b, int N, int act, float* y, cudaStream_t st) {
  ConvArgs a{};
  a.x = x; a.ldx = K; a.T_in = T; a.x_row0 = 0; a.w = w; a.k = 1; a.dil = 1; a.C_in = K; a.N = N; a.bias = b; a.bias_mod = N;
  a.act = act; a.y = y; a.ldy = N; a.T_out = T; a.batch = 1;
  return conv1d_f32_launch(a, st);
}

}  // namespace

extern "C" {

// source != nullptr: talker, code predictor, codec and text side read source's weights (s2s_qwen3tts_create_shared)
static int create(s2s_ctx* ctx, const s2s_qwen3tts_config* cfg, s2s_qwen3tts* source, s2s_qwen3tts** out) {
  S2S_REQUIRE(ctx && cfg && out, "qwen3tts_create: null argument");
  S2S_REQUIRE(cfg->n_groups >= 3 && cfg->n_groups <= 32, "qwen3tts: n_groups in [3,32]");
  S2S_REQUIRE(cfg->max_sessions >= 1 && cfg->max_text >= 1 && cfg->max_positions >= 64, "qwen3tts: bad capacity");
  S2S_REQUIRE(cfg->text_vocab > 0 && cfg->text_hidden > 0, "qwen3tts: bad text geometry");
  for (int id : {cfg->tts_bos, cfg->tts_eos, cfg->tts_pad, cfg->im_start, cfg->assistant, cfg->newline})
    S2S_REQUIRE(id >= 0 && id < cfg->text_vocab, "qwen3tts: text-side special id %d outside the text vocabulary", id);
  for (int id : {cfg->codec_eos, cfg->codec_nothink, cfg->codec_think_bos, cfg->codec_think_eos, cfg->codec_pad, cfg->codec_bos})
    S2S_REQUIRE(id >= 0 && id < cfg->vocab, "qwen3tts: codec special id %d outside the codec vocabulary", id);
  S2S_REQUIRE(cfg->vocab > 1024, "qwen3tts: the codec vocabulary must exceed the 1024 reserved special ids");
  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  s2s_qwen3tts* m = new s2s_qwen3tts();
  m->ctx = ctx;
  m->cfg = *cfg;
  const auto& c = m->cfg;
  int r = S2S_OK;
  {
    s2s_llama_config t{};
    t.d_model = c.d_model; t.layers = c.layers; t.heads = c.heads; t.kv_heads = c.kv_heads; t.head_dim = c.head_dim; t.ffn = c.ffn;
    t.vocab = c.vocab; t.rope_theta = c.rope_theta; t.rms_eps = c.rms_eps; t.compute_dtype = c.compute_dtype;
    t.max_sessions = c.max_sessions; t.max_positions = c.max_positions; t.max_prefill = PROMPT_ROWS; t.qk_norm = 1; t.n_tables = 1;
    r = source ? s2s_llama_create_shared(ctx, source->talker, &t, &m->talker) : s2s_llama_create(ctx, &t, &m->talker);
  }
  if (r == S2S_OK) {
    s2s_llama_config p{};
    p.d_model = c.d_model; p.layers = c.cp_layers; p.heads = c.cp_heads; p.kv_heads = c.cp_kv_heads; p.head_dim = c.cp_head_dim;
    p.ffn = c.cp_ffn; p.vocab = c.cp_vocab; p.rope_theta = c.rope_theta; p.rms_eps = c.rms_eps; p.compute_dtype = c.compute_dtype;
    p.max_sessions = TTS_MAX_B; p.max_positions = 64; p.max_prefill = 1; p.qk_norm = 1; p.n_tables = c.n_groups - 1;
    r = source ? s2s_llama_create_shared(ctx, source->pred, &p, &m->pred) : s2s_llama_create(ctx, &p, &m->pred);
  }
  if (r == S2S_OK) r = source ? codec_create_shared(ctx, source->codec, &c.codec, &m->codec) : codec_create(ctx, &c.codec, &m->codec);
  if (r == S2S_OK && c.codec.quantizers != c.n_groups) { s2s_set_error("qwen3tts: codec quantizers %d != n_groups %d", c.codec.quantizers, c.n_groups); r = S2S_ERR_INVALID; }
  auto alloc_all = [&]() -> int {
    const int d = c.d_model, rows = c.max_text + 6;
    WeightArena& A = m->arena;
    if (source) A.borrow(source->arena);
    S2S_CHECK(A.alloc_weights(&m->text_embed, (size_t)c.text_vocab * c.text_hidden * 2));
    S2S_CHECK(A.alloc_weights(&m->fc1_w, (size_t)c.text_hidden * c.ffn * 4));
    S2S_CHECK(A.alloc_weights(&m->fc1_b, (size_t)c.ffn * 4));
    S2S_CHECK(A.alloc_weights(&m->fc2_w, (size_t)c.ffn * d * 4));
    S2S_CHECK(A.alloc_weights(&m->fc2_b, (size_t)d * 4));
    // init_random: fixed seeds (seed ^ 1 .. 5) and scales of their own
    A.add("text_embedding.weight", m->text_embed, true, (int64_t)c.text_vocab * c.text_hidden, 1.0f).seed = 1;
    A.add("text_projection.linear_fc1.weight", m->fc1_w, false, (int64_t)c.ffn * c.text_hidden, 1.0f / sqrtf((float)c.text_hidden))
        .as(W_LINEAR, c.ffn, c.text_hidden).seed = 2;
    A.add("text_projection.linear_fc1.bias", m->fc1_b, false, c.ffn, 0.05f).seed = 3;
    A.add("text_projection.linear_fc2.weight", m->fc2_w, false, (int64_t)d * c.ffn, 0.7f / sqrtf((float)c.ffn)).as(W_LINEAR, d, c.ffn).seed = 4;
    A.add("text_projection.linear_fc2.bias", m->fc2_b, false, d, 0.05f).seed = 5;
    m->sess.assign(c.max_sessions, s2s_qwen3tts::Sess());
    m->trailing_stride = (long long)c.max_text * d;
    m->history_stride = (long long)c.max_positions * c.n_groups;
    S2S_CHECK(A.alloc(&m->trailing, (size_t)c.max_sessions * m->trailing_stride * 4));
    S2S_CHECK(A.alloc(&m->pad_embed, (size_t)c.max_sessions * d * 4));
    S2S_CHECK(A.alloc(&m->xnext, (size_t)c.max_sessions * d * 4));
    S2S_CHECK(A.alloc(&m->history, (size_t)c.max_sessions * m->history_stride * 4));
    S2S_CHECK(A.alloc(&m->ids_d, (size_t)rows * 4));
    S2S_CHECK(A.alloc(&m->emb_rows, (size_t)rows * c.text_hidden * 4));
    S2S_CHECK(A.alloc(&m->proj_mid, (size_t)rows * c.ffn * 4));
    S2S_CHECK(A.alloc(&m->proj_out, (size_t)rows * d * 4));
    S2S_CHECK(A.alloc(&m->x_in_t, (size_t)TTS_MAX_B * d * 4));
    S2S_CHECK(A.alloc(&m->hidden, (size_t)TTS_MAX_B * d * 4));
    S2S_CHECK(A.alloc(&m->x_in_p, (size_t)TTS_MAX_B * d * 4));
    S2S_CHECK(A.alloc(&m->tslot_d, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->tpos_d, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->pslot_d, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->ppos_d, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->code0, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->pcodes, (size_t)TTS_MAX_B * c.n_groups * 4));
    S2S_CHECK(A.alloc(&m->tlen, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->plen, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->code0_feed, TTS_MAX_B * 4));
    S2S_CHECK(A.alloc(&m->forced_frame, (size_t)TTS_MAX_B * c.n_groups * 4));
    S2S_CHECK(A.alloc(&m->suppress, (size_t)c.vocab));
    m->tsamp.assign(c.max_sessions, samp_greedy());
    m->psamp.assign(c.max_sessions, samp_greedy());
    S2S_CHECK(A.alloc(&m->samp_d, 2 * TTS_MAX_B * sizeof(SampSlot)));
    // transformers generate(): the last 1024 ids of the codec vocabulary except codec_eos are never predicted (TF:3954-3962)
    std::vector<unsigned char> mask((size_t)c.vocab, 0);
    for (int i = c.vocab - 1024; i < c.vocab; ++i) if (i != c.codec_eos) mask[(size_t)i] = 1;
    S2S_CHECK_CUDA(cudaMemcpy(m->suppress, mask.data(), mask.size(), cudaMemcpyHostToDevice));
    return S2S_OK;
  };
  if (r == S2S_OK) r = alloc_all();
  if (r != S2S_OK) { s2s_qwen3tts_destroy(m); return r; }
  m->finalized = source != nullptr;
  *out = m;
  return S2S_OK;
}

int s2s_qwen3tts_create(s2s_ctx* ctx, const s2s_qwen3tts_config* cfg, s2s_qwen3tts** out) { return create(ctx, cfg, nullptr, out); }

int s2s_qwen3tts_create_shared(s2s_ctx* ctx, s2s_qwen3tts* source, const s2s_qwen3tts_config* cfg, s2s_qwen3tts** out) {
  const char* who = "qwen3tts create_shared";
  S2S_REQUIRE(ctx && source && cfg && out, "%s: null argument", who);
  S2S_REQUIRE(source->finalized, "%s: the source is not finalized", who);
  S2S_REQUIRE(source->ctx->device == ctx->device, "%s: the source is on device %d, the context on device %d", who,
              source->ctx->device, ctx->device);
  const s2s_qwen3tts_config& s = source->cfg;
#define S2S_SAME(f) S2S_REQUIRE_SAME(*cfg, s, f, who)
  S2S_SAME(d_model); S2S_SAME(layers); S2S_SAME(heads); S2S_SAME(kv_heads); S2S_SAME(head_dim); S2S_SAME(ffn); S2S_SAME(vocab);
  S2S_SAME(cp_layers); S2S_SAME(cp_heads); S2S_SAME(cp_kv_heads); S2S_SAME(cp_head_dim); S2S_SAME(cp_ffn); S2S_SAME(cp_vocab);
  S2S_SAME(n_groups); S2S_SAME(text_vocab); S2S_SAME(text_hidden); S2S_SAME(rope_theta); S2S_SAME(rms_eps); S2S_SAME(compute_dtype);
  S2S_SAME(codec_eos); S2S_SAME(codec_nothink); S2S_SAME(codec_think_bos); S2S_SAME(codec_think_eos); S2S_SAME(codec_pad);
  S2S_SAME(codec_bos); S2S_SAME(tts_bos); S2S_SAME(tts_eos); S2S_SAME(tts_pad); S2S_SAME(im_start); S2S_SAME(assistant);
  S2S_SAME(newline);
#undef S2S_SAME
  // the codec's own fields (codec.precision included) are checked by codec_create_shared
  return create(ctx, cfg, source, out);
}

int s2s_qwen3tts_device_bytes(s2s_qwen3tts* m, int64_t* weights, int64_t* total) {
  S2S_REQUIRE(m && weights && total, "qwen3tts device_bytes: null argument");
  int64_t w[3], t[3];
  S2S_CHECK(s2s_llama_device_bytes(m->talker, &w[0], &t[0]));
  S2S_CHECK(s2s_llama_device_bytes(m->pred, &w[1], &t[1]));
  S2S_CHECK(codec_device_bytes(m->codec, &w[2], &t[2]));
  *weights = w[0] + w[1] + w[2] + (int64_t)m->arena.weight_bytes();
  *total = t[0] + t[1] + t[2] + (int64_t)m->arena.bytes();
  return S2S_OK;
}

int s2s_qwen3tts_destroy(s2s_qwen3tts* m) {
  if (!m) return S2S_OK;
  if (m->talker) s2s_llama_destroy(m->talker);
  if (m->pred) s2s_llama_destroy(m->pred);
  if (m->codec) codec_destroy(m->codec);
  delete m;
  return S2S_OK;
}

int s2s_qwen3tts_bind_tensor(s2s_qwen3tts* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                             int32_t dtype) {
  S2S_REQUIRE(m && name && data_h && shape, "qwen3tts bind_tensor: null argument");
  S2S_CHECK(m->arena.check_writable("qwen3tts bind_tensor"));   // the talker, predictor and codec are shared with it
  const std::string n(name);
  auto starts = [&](const char* p) { return n.rfind(p, 0) == 0; };
  if (starts("code2wav.")) return codec_bind_tensor(m->codec, name + 9, data_h, shape, ndim, dtype);
  if (starts("code_predictor.model.codec_embedding.")) {
    const std::string rest = n.substr(strlen("code_predictor.model.codec_embedding."));   // "<i>.weight"
    return s2s_llama_bind_tensor(m->pred, ("model.embed_tokens." + rest).c_str(), data_h, shape, ndim, dtype);
  }
  if (starts("code_predictor.")) return s2s_llama_bind_tensor(m->pred, name + strlen("code_predictor."), data_h, shape, ndim, dtype);
  if (n == "model.codec_embedding.weight") return s2s_llama_bind_tensor(m->talker, "model.embed_tokens.weight", data_h, shape, ndim, dtype);
  if (n == "codec_head.weight") return s2s_llama_bind_tensor(m->talker, "lm_head.weight", data_h, shape, ndim, dtype);
  if (starts("model.")) return s2s_llama_bind_tensor(m->talker, name, data_h, shape, ndim, dtype);
  if (starts("hidden_projection.")) return S2S_OK;   // multimodal path of the cousin: unused by a text-only TTS turn
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  return m->arena.bind("qwen3tts", name, data_h, shape, ndim, dtype, m->cfg.compute_dtype);
}

int s2s_qwen3tts_init_random(s2s_qwen3tts* m, uint64_t seed) {
  S2S_REQUIRE(m, "qwen3tts init_random: null model");
  S2S_CHECK(m->arena.check_writable("qwen3tts init_random"));
  S2S_CHECK(s2s_llama_init_random(m->talker, seed ^ 0x7a11ull));
  S2S_CHECK(s2s_llama_init_random(m->pred, seed ^ 0x9ed1ull));
  S2S_CHECK(codec_init_random(m->codec, seed ^ 0xc0decull));
  return m->arena.init_random(seed, m->cfg.compute_dtype);
}

int s2s_qwen3tts_finalize(s2s_qwen3tts* m) {
  S2S_REQUIRE(m, "qwen3tts finalize: null model");
  S2S_CHECK(m->arena.check_writable("qwen3tts finalize"));
  S2S_CHECK(m->arena.check_all_bound("qwen3tts"));
  S2S_CHECK(s2s_llama_finalize(m->talker));
  S2S_CHECK(s2s_llama_finalize(m->pred));
  S2S_CHECK(codec_finalize(m->codec));
  m->finalized = true;
  return S2S_OK;
}

int s2s_qwen3tts_prefill(s2s_qwen3tts* m, int32_t slot, const int32_t* text_ids_h, int32_t n_text, int32_t speaker_id,
                         void* stream) {
  S2S_REQUIRE(m && m->finalized && text_ids_h, "qwen3tts prefill: null argument / not finalized");
  const auto& c = m->cfg;
  S2S_REQUIRE(slot >= 0 && slot < c.max_sessions, "qwen3tts prefill: bad slot %d", slot);
  S2S_REQUIRE(n_text >= 1 && n_text <= c.max_text, "qwen3tts prefill: %d text tokens outside [1,%d]", n_text, c.max_text);
  S2S_REQUIRE(speaker_id >= 0 && speaker_id < c.vocab, "qwen3tts prefill: speaker id %d outside the codec vocabulary", speaker_id);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  const int d = c.d_model, rows = n_text + 6;
  std::vector<int> ids;
  ids.reserve(rows);
  ids.push_back(c.im_start); ids.push_back(c.assistant); ids.push_back(c.newline);
  for (int i = 0; i < n_text; ++i) {
    S2S_REQUIRE(text_ids_h[i] >= 0 && text_ids_h[i] < c.text_vocab, "qwen3tts prefill: text token %d out of range", text_ids_h[i]);
    ids.push_back(text_ids_h[i]);
  }
  ids.push_back(c.tts_bos); ids.push_back(c.tts_eos); ids.push_back(c.tts_pad);
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->ids_d, ids.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));   // ids is a stack-lifetime host buffer
  const bool bf = c.compute_dtype == S2S_BF16;
  if (bf) gather_rows_f32_kernel<__nv_bfloat16><<<rows, 256, 0, st>>>(m->ids_d, (const __nv_bfloat16*)m->text_embed, c.text_hidden, m->emb_rows);
  else gather_rows_f32_kernel<__half><<<rows, 256, 0, st>>>(m->ids_d, (const __half*)m->text_embed, c.text_hidden, m->emb_rows);
  S2S_LAUNCH_CHECK();
  // Qwen3OmniMoeTalkerResizeMLP: fc2(silu(fc1 x))
  S2S_CHECK(linear_f32(m->emb_rows, rows, c.text_hidden, m->fc1_w, m->fc1_b, c.ffn, 2, m->proj_mid, st));
  S2S_CHECK(linear_f32(m->proj_mid, rows, c.ffn, m->fc2_w, m->fc2_b, d, 0, m->proj_out, st));
  float* trailing = m->trailing + (long long)slot * m->trailing_stride;
  if (bf) build_prompt_kernel<__nv_bfloat16><<<PROMPT_ROWS + n_text, 256, 0, st>>>(
        m->proj_out, n_text, (const __nv_bfloat16*)m->talker->embed, d, c.codec_nothink, c.codec_think_bos, c.codec_think_eos,
        speaker_id, c.codec_pad, c.codec_bos, m->talker->x, m->xnext + (long long)slot * d, trailing);
  else build_prompt_kernel<__half><<<PROMPT_ROWS + n_text, 256, 0, st>>>(
        m->proj_out, n_text, (const __half*)m->talker->embed, d, c.codec_nothink, c.codec_think_bos, c.codec_think_eos, speaker_id,
        c.codec_pad, c.codec_bos, m->talker->x, m->xnext + (long long)slot * d, trailing);
  S2S_LAUNCH_CHECK();
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->pad_embed + (long long)slot * d, m->proj_out + (long long)(n_text + 5) * d, (size_t)d * 4,
                                 cudaMemcpyDeviceToDevice, st));
  m->talker->len[slot] = 0;
  // a new utterance: greedy until s2s_qwen3tts_set_sampling, and no first code seen yet (the prompt's codec ids are not
  // penalised: the cousin's talker.generate gets no input_ids)
  m->tsamp[slot] = samp_greedy();
  m->psamp[slot] = samp_greedy();
  S2S_CHECK_CUDA(cudaMemsetAsync(m->talker->seen + (long long)slot * m->talker->seen_words, 0, (size_t)m->talker->seen_words * 4, st));
  S2S_CHECK(llama_prefill_rows(m->talker, slot, PROMPT_ROWS - 1, nullptr, nullptr, nullptr, st));
  auto& s = m->sess[slot];
  s.n_trailing = n_text; s.frames = 0; s.pos = PROMPT_ROWS - 1; s.active = true;
  return S2S_OK;
}

int s2s_qwen3tts_set_sampling(s2s_qwen3tts* m, int32_t slot, const s2s_sampling* talker, const s2s_sampling* predictor) {
  S2S_REQUIRE(m && slot >= 0 && slot < m->cfg.max_sessions, "qwen3tts set_sampling: bad slot %d", slot);
  for (const s2s_sampling* s : {talker, predictor})
    S2S_REQUIRE(!s || s->min_new_tokens == 0, "qwen3tts set_sampling: min_new_tokens must be 0 (codec_eos is the only stop)");
  S2S_REQUIRE(!predictor || predictor->repetition_penalty == 1.f,
              "qwen3tts set_sampling: the code predictor has no repetition penalty (got %g)", (double)predictor->repetition_penalty);
  SampSlot t, p;
  S2S_CHECK(samp_from_abi(talker, m->cfg.vocab, "qwen3tts set_sampling (talker)", &t));
  S2S_CHECK(samp_from_abi(predictor, m->cfg.cp_vocab, "qwen3tts set_sampling (predictor)", &p));
  t.n_eos = 0; p.n_eos = 0;
  m->tsamp[slot] = t;
  m->psamp[slot] = p;
  return S2S_OK;
}

int s2s_qwen3tts_decode_frames(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_frames, int32_t* codes_out_d,
                               const int32_t* forced_codes_d, void* stream) {
  return s2s_qwen3tts_decode_frames_logits(m, slots_h, B, n_frames, codes_out_d, forced_codes_d, nullptr, nullptr, stream);
}

int s2s_qwen3tts_decode_frames_logits(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_frames, int32_t* codes_out_d,
                                      const int32_t* forced_codes_d, float* talker_logits_out_d, float* pred_logits_out_d,
                                      void* stream) {
  S2S_REQUIRE(m && m->finalized && slots_h && codes_out_d, "qwen3tts decode_frames: null argument / not finalized");
  const auto& c = m->cfg;
  const int max_b = tts_max_batch(m);
  S2S_REQUIRE(B >= 1 && B <= max_b, "qwen3tts decode_frames: B=%d outside [1,%d]", B, max_b);
  S2S_REQUIRE(n_frames >= 1, "qwen3tts decode_frames: n_frames must be >= 1");
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  TtsBatch tb{};
  int max_pos = 0;
  for (int b = 0; b < B; ++b) {
    const int s = slots_h[b];
    S2S_REQUIRE(s >= 0 && s < c.max_sessions && m->sess[s].active, "qwen3tts decode_frames: slot %d has no utterance (prefill first)", s);
    for (int b2 = 0; b2 < b; ++b2) S2S_REQUIRE(slots_h[b2] != s, "qwen3tts decode_frames: slot %d listed twice", s);
    S2S_REQUIRE(m->sess[s].pos + n_frames <= c.max_positions, "qwen3tts decode_frames: slot %d would exceed max_positions %d", s, c.max_positions);
    tb.slot[b] = s; tb.pos0[b] = m->sess[s].pos; tb.frames0[b] = m->sess[s].frames; tb.n_trailing[b] = m->sess[s].n_trailing;
    max_pos = std::max(max_pos, tb.pos0[b]);
  }
  const int d = c.d_model, G = c.n_groups;
  const bool bf = c.compute_dtype == S2S_BF16;
  // the batch's token-choice tables, one H2D copy per call and only when a session is not greedy (the copy is staged from
  // this pageable buffer before cudaMemcpyAsync returns)
  SampSlot samp_h[2 * TTS_MAX_B];
  bool t_any = false, p_any = false;
  for (int b = 0; b < B; ++b) {
    samp_h[b] = m->tsamp[slots_h[b]];
    samp_h[TTS_MAX_B + b] = m->psamp[slots_h[b]];
    t_any |= samp_h[b].active != 0;
    p_any |= samp_h[TTS_MAX_B + b].active != 0;
  }
  if (t_any || p_any) S2S_CHECK_CUDA(cudaMemcpyAsync(m->samp_d, samp_h, sizeof(samp_h), cudaMemcpyHostToDevice, st));
  SampSlot* tsamp_d = t_any ? m->samp_d : nullptr;
  SampSlot* psamp_d = p_any ? m->samp_d + TTS_MAX_B : nullptr;
  for (int f = 0; f < n_frames; ++f) {
    frame_prepare_kernel<<<B, 256, 0, st>>>(tb, f, m->xnext, d, m->x_in_t, m->tslot_d, m->tpos_d);
    S2S_LAUNCH_CHECK();
    {   // talker: one step from x_in -> first code of the frame (special ids suppressed) + the pre-norm hidden state
      LlamaDecParams p{};
      llama_fill_dec_params(m->talker, p);
      p.B = B; p.slot = m->tslot_d; p.pos = m->tpos_d; p.max_len = max_pos + f + 1;
      p.x_in = m->x_in_t; p.first_ids = m->code0; p.n_steps = 1; p.eos = -1; p.out_ids = m->code0; p.out_len = m->tlen;
      p.hidden_out = m->hidden; p.suppress = m->suppress;
      p.samp = tsamp_d; p.seen_fixed = 1;
      p.logits_out = talker_logits_out_d ? talker_logits_out_d + (long long)f * B * c.vocab : nullptr;
      S2S_CHECK(llama_decode_launch(m->ctx, p, c.compute_dtype, m->talker->weight_format, m->talker->debug_phases, st));
    }
    frame_mid_kernel<<<B, 256, 0, st>>>(m->hidden, m->talker->norm_f, c.rms_eps, d, m->x_in_p, m->pslot_d, m->ppos_d, m->code0,
                                        forced_codes_d, f, n_frames, G, m->code0_feed, m->forced_frame, psamp_d, tb);
    S2S_LAUNCH_CHECK();
    {   // code predictor: [hidden, embed(code0)] then one step per residual codebook, each with its own table / head
      LlamaDecParams p{};
      llama_fill_dec_params(m->pred, p);
      p.B = B; p.slot = m->pslot_d; p.pos = m->ppos_d; p.max_len = 1;
      p.x_in = m->x_in_p; p.first_ids = m->code0_feed; p.n_steps = G; p.eos = -1; p.out_ids = m->pcodes; p.out_len = m->plen;
      p.forced = forced_codes_d ? m->forced_frame : nullptr;
      p.embed0 = m->talker->embed; p.embed_stride = (long long)m->pred->embed_table_elems; p.head_stride = (long long)m->pred->head_t_table_elems;
      p.samp = psamp_d;
      p.logits_out = pred_logits_out_d ? pred_logits_out_d + (long long)f * G * B * c.cp_vocab : nullptr;
      S2S_CHECK(llama_decode_launch(m->ctx, p, c.compute_dtype, m->pred->weight_format, m->pred->debug_phases, st));
    }
    const int* ff = forced_codes_d ? m->forced_frame : nullptr;
    if (bf) frame_finish_kernel<__nv_bfloat16><<<B, 256, 0, st>>>(tb, f, n_frames, G, m->pcodes, m->code0, ff, (const __nv_bfloat16*)m->talker->embed,
          (const __nv_bfloat16*)m->pred->embed, (long long)m->pred->embed_table_elems, d, m->trailing, m->trailing_stride, m->pad_embed,
          m->xnext, codes_out_d, m->history, m->history_stride, m->talker->seen, m->talker->seen_words);
    else frame_finish_kernel<__half><<<B, 256, 0, st>>>(tb, f, n_frames, G, m->pcodes, m->code0, ff, (const __half*)m->talker->embed,
          (const __half*)m->pred->embed, (long long)m->pred->embed_table_elems, d, m->trailing, m->trailing_stride, m->pad_embed,
          m->xnext, codes_out_d, m->history, m->history_stride, m->talker->seen, m->talker->seen_words);
    S2S_LAUNCH_CHECK();
  }
  for (int b = 0; b < B; ++b) {
    auto& s = m->sess[slots_h[b]];
    s.pos += n_frames; s.frames += n_frames;
    m->talker->len[slots_h[b]] = s.pos;
  }
  return S2S_OK;
}

int s2s_qwen3tts_decode_audio(s2s_qwen3tts* m, int32_t slot, int32_t n_new, int32_t left_context, float* wav_out_d,
                              int32_t* n_out_h, void* stream) {
  S2S_REQUIRE(m && m->finalized && wav_out_d, "qwen3tts decode_audio: null argument / not finalized");
  const auto& c = m->cfg;
  S2S_REQUIRE(slot >= 0 && slot < c.max_sessions && m->sess[slot].active, "qwen3tts decode_audio: bad slot %d", slot);
  const int frames = m->sess[slot].frames;
  S2S_REQUIRE(n_new >= 1 && n_new <= frames, "qwen3tts decode_audio: n_new=%d but the slot holds %d frames", n_new, frames);
  S2S_REQUIRE(left_context >= 0, "qwen3tts decode_audio: negative context");
  const int start = frames - n_new;
  const int ctx = (start - left_context > 0) ? left_context : start;   // Qwen3OmniMoeCode2Wav.chunked_decode (:3786)
  const int* codes = m->history + (long long)slot * m->history_stride + (long long)(start - ctx) * c.n_groups;
  return codec_decode(m->codec, codes, ctx + n_new, ctx, wav_out_d, n_out_h, nullptr, (cudaStream_t)stream);
}

int s2s_qwen3tts_decode_audio_batch(s2s_qwen3tts* m, const int32_t* slots_h, int32_t B, int32_t n_new, int32_t left_context,
                                    float* wav_out_d, int64_t wav_stride, int32_t* n_out_h, void* stream) {
  S2S_REQUIRE(m && m->finalized && slots_h && wav_out_d, "qwen3tts decode_audio_batch: null argument / not finalized");
  const auto& c = m->cfg;
  S2S_REQUIRE(B >= 1 && B <= TTS_MAX_B, "qwen3tts decode_audio_batch: B=%d outside [1,%d]", B, TTS_MAX_B);
  const int32_t* ptrs[TTS_MAX_B];
  int ctx0 = -1;
  for (int b = 0; b < B; ++b) {
    const int slot = slots_h[b];
    S2S_REQUIRE(slot >= 0 && slot < c.max_sessions && m->sess[slot].active, "qwen3tts decode_audio_batch: bad slot %d", slot);
    const int frames = m->sess[slot].frames;
    S2S_REQUIRE(n_new >= 1 && n_new <= frames, "qwen3tts decode_audio_batch: n_new=%d but slot %d holds %d frames", n_new, slot, frames);
    const int start = frames - n_new;
    const int ctx = (start - left_context > 0) ? left_context : start;   // Qwen3OmniMoeCode2Wav.chunked_decode (:3786)
    if (ctx0 < 0) ctx0 = ctx;
    S2S_REQUIRE(ctx == ctx0, "qwen3tts decode_audio_batch: slot %d has %d frames of history, the batch %d (group equal shapes)", slot, ctx, ctx0);
    ptrs[b] = m->history + (long long)slot * m->history_stride + (long long)(start - ctx) * c.n_groups;
  }
  return codec_decode_batch(m->codec, ptrs, B, ctx0 + n_new, ctx0, wav_out_d, wav_stride, n_out_h, nullptr, (cudaStream_t)stream);
}

int s2s_qwen3tts_set_frames(s2s_qwen3tts* m, int32_t slot, int32_t n_frames) {
  S2S_REQUIRE(m && slot >= 0 && slot < m->cfg.max_sessions, "qwen3tts set_frames: bad slot");
  S2S_REQUIRE(n_frames >= 0 && n_frames <= m->sess[slot].frames, "qwen3tts set_frames: %d outside [0,%d]", n_frames, m->sess[slot].frames);
  m->sess[slot].frames = n_frames;
  return S2S_OK;
}
int32_t s2s_qwen3tts_frames(s2s_qwen3tts* m, int32_t slot) {
  if (!m || slot < 0 || slot >= m->cfg.max_sessions) return -1;
  return m->sess[slot].frames;
}
int32_t s2s_qwen3tts_max_batch(s2s_qwen3tts* m) { return m ? tts_max_batch(m) : 0; }
int s2s_qwen3tts_set_trace(s2s_qwen3tts* m, int32_t which, uint64_t* trace_d, int32_t capacity) {
  S2S_REQUIRE(m && (which == 0 || which == 1), "qwen3tts set_trace: which = 0 (talker) or 1 (code predictor)");
  s2s_llama* t = which == 0 ? m->talker : m->pred;
  t->trace = reinterpret_cast<unsigned long long*>(trace_d);
  t->trace_cap = trace_d ? capacity : 0;
  return S2S_OK;
}
s2s_codec* s2s_qwen3tts_codec(s2s_qwen3tts* m) { return m ? m->codec : nullptr; }

}  // extern "C"
