// whisper.cu -- Whisper STT model object behind the C ABI: weight arena (transformers state-dict names ->
// kernel layouts), workspaces, and the launch sequences for log-mel, encoder and greedy decode.
// Replaces the device work of WhisperSTTHandler.process (reference S/STT/whisper_stt_handler.py:225-282):
//   prepare_model_inputs (:83-87) -> s2s_whisper_logmel ;  model.generate (:243) -> encode + decode ;
//   _detect_language (:166-197) -> s2s_whisper_detect_language.
#include <math.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "weight_arena.cuh"
#include "whisper_decode.cuh"

namespace {

constexpr int N_FRAMES = 3000;
constexpr int N_SAMPLES = 480000;

struct EncLayer {
  void *w_qkv, *w_o, *w_fc1, *w_fc2;
  float *b_qkv, *b_o, *b_fc1, *b_fc2, *ln1_w, *ln1_b, *ln2_w, *ln2_b;
};

}  // namespace

struct s2s_whisper {
  s2s_ctx* ctx = nullptr;
  s2s_whisper_config cfg{};
  int esz = 2;
  bool finalized = false;
  WeightArena arena;

  // weights
  void *conv1_w = nullptr, *conv2_w = nullptr, *embed = nullptr, *ckv_w = nullptr;
  float *conv1_b = nullptr, *conv2_b = nullptr, *enc_pos = nullptr, *dec_pos = nullptr, *ckv_b = nullptr;
  float *enc_lnf_w = nullptr, *enc_lnf_b = nullptr, *dec_lnf_w = nullptr, *dec_lnf_b = nullptr;
  std::vector<EncLayer> enc;
  WhisperDecLayer* dec_d = nullptr;      // [dec_layers] device table of the decoder layers
  // tables
  float *hann = nullptr, *twiddle = nullptr, *fb = nullptr;
  int2* fb_range = nullptr;
  // workspace
  float *pcm = nullptr, *mel_f32 = nullptr, *mel_max = nullptr, *x = nullptr;
  int* n_samples_d = nullptr;
  void* vt = nullptr;
  size_t vt_elems = 0;
  void *mel_t = nullptr, *h1 = nullptr, *xn = nullptr, *qkv = nullptr, *attn = nullptr, *hbuf = nullptr,
       *enc_out = nullptr, *cross_kv = nullptr;
  // decoder state
  float *dx = nullptr, *dq = nullptr, *dh = nullptr, *part = nullptr, *cand_val = nullptr;
  float *dx_alt = nullptr, *part_x0 = nullptr, *part_x1 = nullptr;  // cluster decode kernel (1-2 sessions)
  int cluster_decode = 1;
  void* attn16 = nullptr;
  unsigned int* attn_cnt = nullptr;
  void* self_kv = nullptr;
  int *tokens = nullptr, *out_ids = nullptr, *out_len = nullptr, *done = nullptr, *n_done = nullptr, *cand_idx = nullptr;
  unsigned char *suppress = nullptr, *suppress_lang = nullptr;
  std::vector<int> suppress_key[2];        // the id lists the device masks were built from (masks are static per options)
  int* tok_stage = nullptr;                // pinned host staging of the prompt tokens
  cudaEvent_t tok_event = nullptr;         // recorded after the staging buffer's last H2D copy
  unsigned int* sync_counter = nullptr;
  int s_max = 0;
  int last_B = 0;
  int debug_phases = 0;
  unsigned long long* trace = nullptr;
  int trace_cap = 0;
};

namespace {

inline char* off(void* base, int64_t elems, int esz) { return reinterpret_cast<char*>(base) + elems * esz; }

int build_tables(s2s_whisper* m) {
  const int n_mels = m->cfg.n_mels;
  std::vector<float> hann(400), tw(800);
  for (int i = 0; i < 400; ++i) {
    hann[i] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / 400.0));
    tw[i] = (float)cos(2.0 * M_PI * i / 400.0);
    tw[400 + i] = (float)sin(2.0 * M_PI * i / 400.0);
  }
  // slaney mel filter bank (transformers audio_utils.mel_filter_bank, norm="slaney", mel_scale="slaney")
  auto hz_to_mel = [](double f) { return f >= 1000.0 ? 15.0 + log(f / 1000.0) * (27.0 / log(6.4)) : 3.0 * f / 200.0; };
  auto mel_to_hz = [](double mm) { return mm >= 15.0 ? 1000.0 * exp((log(6.4) / 27.0) * (mm - 15.0)) : 200.0 * mm / 3.0; };
  std::vector<double> filt(n_mels + 2);
  const double m_lo = hz_to_mel(0.0), m_hi = hz_to_mel(8000.0);
  for (int i = 0; i < n_mels + 2; ++i) filt[i] = mel_to_hz(m_lo + (m_hi - m_lo) * i / (n_mels + 1));
  std::vector<float> fb((size_t)n_mels * 201, 0.f);
  std::vector<int2> rg(n_mels);
  for (int j = 0; j < n_mels; ++j) {
    int lo = 201, hi = 0;
    const double enorm = 2.0 / (filt[j + 2] - filt[j]);
    for (int k = 0; k < 201; ++k) {
      const double f = 8000.0 * k / 200.0;
      const double down = (f - filt[j]) / (filt[j + 1] - filt[j]);
      const double up = (filt[j + 2] - f) / (filt[j + 2] - filt[j + 1]);
      const double v = fmax(0.0, fmin(down, up)) * enorm;
      fb[(size_t)j * 201 + k] = (float)v;
      if (v > 0.0) { lo = k < lo ? k : lo; hi = k + 1 > hi ? k + 1 : hi; }
    }
    if (lo > hi) { lo = 0; hi = 0; }
    rg[j] = make_int2(lo, hi);
  }
  S2S_CHECK(m->arena.alloc(&m->hann, 400 * 4));
  S2S_CHECK(m->arena.alloc(&m->twiddle, 800 * 4));
  S2S_CHECK(m->arena.alloc(&m->fb, fb.size() * 4));
  S2S_CHECK(m->arena.alloc(&m->fb_range, rg.size() * sizeof(int2)));
  S2S_CHECK_CUDA(cudaMemcpy(m->hann, hann.data(), 400 * 4, cudaMemcpyHostToDevice));
  S2S_CHECK_CUDA(cudaMemcpy(m->twiddle, tw.data(), 800 * 4, cudaMemcpyHostToDevice));
  S2S_CHECK_CUDA(cudaMemcpy(m->fb, fb.data(), fb.size() * 4, cudaMemcpyHostToDevice));
  S2S_CHECK_CUDA(cudaMemcpy(m->fb_range, rg.data(), rg.size() * sizeof(int2), cudaMemcpyHostToDevice));
  return S2S_OK;
}

int alloc_weights(s2s_whisper* m) {
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, esz = m->esz;
  const float qscale = 1.0f / sqrtf((float)(d / c.heads));
  WeightArena& A = m->arena;
  const float s_qk = 1.6f / sqrtf((float)d), s_v = 0.8f / sqrtf((float)d), s_o = 1.2f / sqrtf((float)d);
  const float s_fc1 = 1.0f / sqrtf((float)d), s_fc2 = 0.5f / sqrtf((float)f);
  auto wbytes = [&](int64_t n) { return (size_t)n * esz; };

  S2S_CHECK(m->arena.alloc_weights(&m->conv1_w, wbytes((int64_t)d * 3 * c.n_mels)));
  S2S_CHECK(m->arena.alloc_weights(&m->conv1_b, d * 4));
  S2S_CHECK(m->arena.alloc_weights(&m->conv2_w, wbytes((int64_t)d * 3 * d)));
  S2S_CHECK(m->arena.alloc_weights(&m->conv2_b, d * 4));
  S2S_CHECK(m->arena.alloc_weights(&m->enc_pos, (size_t)c.max_source_positions * d * 4));
  A.add("model.encoder.conv1.weight", m->conv1_w, true, (int64_t)d * c.n_mels * 3, 0.05f).as(W_CONV_ROWS, d, c.n_mels, 3);
  A.add("model.encoder.conv2.weight", m->conv2_w, true, (int64_t)d * d * 3, 0.03f).as(W_CONV_ROWS, d, d, 3);
  A.add("model.encoder.conv1.bias", m->conv1_b, false, d);
  A.add("model.encoder.conv2.bias", m->conv2_b, false, d);
  A.add("model.encoder.embed_positions.weight", m->enc_pos, false, (int64_t)c.max_source_positions * d, 0.5f);

  auto add_ln = [&](const std::string& nm, float** w, float** b) -> int {
    S2S_CHECK(m->arena.alloc_weights(w, d * 4));
    S2S_CHECK(m->arena.alloc_weights(b, d * 4));
    A.add(nm + ".weight", *w, false, d, 0.1f, 1.0f);
    A.add(nm + ".bias", *b, false, d, 0.05f);
    return S2S_OK;
  };

  m->enc.resize(c.enc_layers);
  for (int i = 0; i < c.enc_layers; ++i) {
    EncLayer& L = m->enc[i];
    const std::string p = "model.encoder.layers." + std::to_string(i) + ".";
    S2S_CHECK(m->arena.alloc_weights(&L.w_qkv, wbytes((int64_t)3 * d * d)));
    S2S_CHECK(m->arena.alloc_weights(&L.b_qkv, 3 * d * 4));
    S2S_CHECK(m->arena.alloc_weights(&L.w_o, wbytes((int64_t)d * d)));
    S2S_CHECK(m->arena.alloc_weights(&L.b_o, d * 4));
    S2S_CHECK(m->arena.alloc_weights(&L.w_fc1, wbytes((int64_t)f * d)));
    S2S_CHECK(m->arena.alloc_weights(&L.b_fc1, f * 4));
    S2S_CHECK(m->arena.alloc_weights(&L.w_fc2, wbytes((int64_t)d * f)));
    S2S_CHECK(m->arena.alloc_weights(&L.b_fc2, d * 4));
    A.add(p + "self_attn.q_proj.weight", L.w_qkv, true, (int64_t)d * d, s_qk).scale = qscale;
    A.add(p + "self_attn.q_proj.bias", L.b_qkv, false, d).scale = qscale;
    A.add(p + "self_attn.k_proj.weight", off(L.w_qkv, (int64_t)d * d, esz), true, (int64_t)d * d, s_qk);
    A.add(p + "self_attn.v_proj.weight", off(L.w_qkv, (int64_t)2 * d * d, esz), true, (int64_t)d * d, s_v);
    A.add(p + "self_attn.v_proj.bias", L.b_qkv + 2 * d, false, d);
    A.add(p + "self_attn.out_proj.weight", L.w_o, true, (int64_t)d * d, s_o);
    A.add(p + "self_attn.out_proj.bias", L.b_o, false, d);
    A.add(p + "fc1.weight", L.w_fc1, true, (int64_t)f * d, s_fc1);
    A.add(p + "fc1.bias", L.b_fc1, false, f);
    A.add(p + "fc2.weight", L.w_fc2, true, (int64_t)d * f, s_fc2);
    A.add(p + "fc2.bias", L.b_fc2, false, d);
    S2S_CHECK(add_ln(p + "self_attn_layer_norm", &L.ln1_w, &L.ln1_b));
    S2S_CHECK(add_ln(p + "final_layer_norm", &L.ln2_w, &L.ln2_b));
  }
  S2S_CHECK(add_ln("model.encoder.layer_norm", &m->enc_lnf_w, &m->enc_lnf_b));

  // decoder.  The matrices the decode kernel streams and the token embedding (looked up, and the tied output projection)
  // are stored once, in the tiled layout (weight_tiles.cu): bind and init_random tile each tensor's rows into place.  The
  // cross-attention K/V projections are read by the encoder-side GEMM and stay row-major.
  auto alloc_tiled = [&](void** w, int N, int K) { return m->arena.alloc_weights(w, tiled_weight_elems(N, K) * 2); };
  S2S_CHECK(alloc_tiled(&m->embed, c.vocab, d));
  S2S_CHECK(m->arena.alloc_weights(&m->dec_pos, (size_t)c.max_target_positions * d * 4));
  A.add("model.decoder.embed_tokens.weight", m->embed, true, (int64_t)c.vocab * d).tiled(c.vocab, d);
  A.add("model.decoder.embed_positions.weight", m->dec_pos, false, (int64_t)c.max_target_positions * d);
  S2S_CHECK(m->arena.alloc_weights(&m->ckv_w, wbytes((int64_t)c.dec_layers * 2 * d * d)));
  S2S_CHECK(m->arena.alloc_weights(&m->ckv_b, (size_t)c.dec_layers * 2 * d * 4));
  std::vector<WhisperDecLayer> dec(c.dec_layers);
  for (int i = 0; i < c.dec_layers; ++i) {
    WhisperDecLayer& L = dec[i];
    const std::string p = "model.decoder.layers." + std::to_string(i) + ".";
    void *w_qkv, *w_o, *w_cq, *w_co, *w_fc1, *w_fc2;
    float *b_qkv, *b_o, *b_cq, *b_co, *b_fc1, *b_fc2, *l1w, *l1b, *l2w, *l2b, *l3w, *l3b;
    S2S_CHECK(alloc_tiled(&w_qkv, 3 * d, d));
    S2S_CHECK(m->arena.alloc_weights(&b_qkv, 3 * d * 4));
    S2S_CHECK(alloc_tiled(&w_o, d, d));
    S2S_CHECK(m->arena.alloc_weights(&b_o, d * 4));
    S2S_CHECK(alloc_tiled(&w_cq, d, d));
    S2S_CHECK(m->arena.alloc_weights(&b_cq, d * 4));
    S2S_CHECK(alloc_tiled(&w_co, d, d));
    S2S_CHECK(m->arena.alloc_weights(&b_co, d * 4));
    S2S_CHECK(alloc_tiled(&w_fc1, f, d));
    S2S_CHECK(m->arena.alloc_weights(&b_fc1, f * 4));
    S2S_CHECK(alloc_tiled(&w_fc2, d, f));
    S2S_CHECK(m->arena.alloc_weights(&b_fc2, d * 4));
    A.add(p + "self_attn.q_proj.weight", w_qkv, true, (int64_t)d * d, s_qk).tiled(3 * d, d, 0).scale = qscale;
    A.add(p + "self_attn.q_proj.bias", b_qkv, false, d).scale = qscale;
    A.add(p + "self_attn.k_proj.weight", w_qkv, true, (int64_t)d * d, s_qk).tiled(3 * d, d, d);
    A.add(p + "self_attn.v_proj.weight", w_qkv, true, (int64_t)d * d, s_v).tiled(3 * d, d, 2 * d);
    A.add(p + "self_attn.v_proj.bias", b_qkv + 2 * d, false, d);
    A.add(p + "self_attn.out_proj.weight", w_o, true, (int64_t)d * d, s_o).tiled(d, d);
    A.add(p + "self_attn.out_proj.bias", b_o, false, d);
    A.add(p + "encoder_attn.q_proj.weight", w_cq, true, (int64_t)d * d, s_qk).tiled(d, d).scale = qscale;
    A.add(p + "encoder_attn.q_proj.bias", b_cq, false, d).scale = qscale;
    A.add(p + "encoder_attn.k_proj.weight", off(m->ckv_w, (int64_t)i * 2 * d * d, esz), true, (int64_t)d * d, s_qk);
    A.add(p + "encoder_attn.v_proj.weight", off(m->ckv_w, (int64_t)(i * 2 + 1) * d * d, esz), true, (int64_t)d * d, s_v);
    A.add(p + "encoder_attn.v_proj.bias", m->ckv_b + (int64_t)(i * 2 + 1) * d, false, d);
    A.add(p + "encoder_attn.out_proj.weight", w_co, true, (int64_t)d * d, s_o).tiled(d, d);
    A.add(p + "encoder_attn.out_proj.bias", b_co, false, d);
    A.add(p + "fc1.weight", w_fc1, true, (int64_t)f * d, s_fc1).tiled(f, d);
    A.add(p + "fc1.bias", b_fc1, false, f);
    A.add(p + "fc2.weight", w_fc2, true, (int64_t)d * f, s_fc2).tiled(d, f);
    A.add(p + "fc2.bias", b_fc2, false, d);
    S2S_CHECK(add_ln(p + "self_attn_layer_norm", &l1w, &l1b));
    S2S_CHECK(add_ln(p + "encoder_attn_layer_norm", &l2w, &l2b));
    S2S_CHECK(add_ln(p + "final_layer_norm", &l3w, &l3b));
    L.w_qkv = w_qkv; L.b_qkv = b_qkv; L.w_o = w_o; L.b_o = b_o; L.w_cq = w_cq; L.b_cq = b_cq; L.w_co = w_co; L.b_co = b_co;
    L.w_fc1 = w_fc1; L.b_fc1 = b_fc1; L.w_fc2 = w_fc2; L.b_fc2 = b_fc2;
    L.ln1_w = l1w; L.ln1_b = l1b; L.ln2_w = l2w; L.ln2_b = l2b; L.ln3_w = l3w; L.ln3_b = l3b;
  }
  S2S_CHECK(add_ln("model.decoder.layer_norm", &m->dec_lnf_w, &m->dec_lnf_b));
  // the device layer table is the object's own (an object sharing the weights uploads the same pointers to its own copy)
  S2S_CHECK(m->arena.alloc(&m->dec_d, sizeof(WhisperDecLayer) * c.dec_layers));
  S2S_CHECK_CUDA(cudaMemcpy(m->dec_d, dec.data(), sizeof(WhisperDecLayer) * c.dec_layers, cudaMemcpyHostToDevice));
  return S2S_OK;
}

int alloc_workspace(s2s_whisper* m) {
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, B = c.max_batch, esz = m->esz;
  const int64_t rows = (int64_t)B * c.max_source_positions;
  S2S_CHECK(m->arena.alloc(&m->pcm, (size_t)B * N_SAMPLES * 4, false));
  S2S_CHECK(m->arena.alloc(&m->n_samples_d, B * 4));
  S2S_CHECK(m->arena.alloc(&m->mel_f32, (size_t)B * c.n_mels * N_FRAMES * 4));
  S2S_CHECK(m->arena.alloc(&m->mel_max, B * 4));
  S2S_CHECK(m->arena.alloc(&m->mel_t, (size_t)B * (N_FRAMES + 2) * c.n_mels * esz));
  S2S_CHECK(m->arena.alloc(&m->h1, (size_t)B * (N_FRAMES + 2) * d * esz));
  S2S_CHECK(m->arena.alloc(&m->x, (size_t)rows * d * 4));
  S2S_CHECK(m->arena.alloc(&m->xn, (size_t)rows * d * esz));
  S2S_CHECK(m->arena.alloc(&m->qkv, (size_t)rows * 3 * d * esz));
  S2S_CHECK(m->arena.alloc(&m->attn, (size_t)rows * d * esz));
  S2S_CHECK(m->arena.alloc(&m->hbuf, (size_t)rows * f * esz));
  S2S_CHECK(m->arena.alloc(&m->enc_out, (size_t)rows * d * esz));
  S2S_CHECK(m->arena.alloc(&m->cross_kv, (size_t)rows * c.dec_layers * 2 * d * esz));
  m->vt_elems = attention_tc_scratch_elems(B, c.max_source_positions, c.heads, 64);
  S2S_CHECK(m->arena.alloc(&m->vt, m->vt_elems * esz));
  // decoder
  m->s_max = (c.max_source_positions + ATT_CHUNK_KEYS - 1) / ATT_CHUNK_KEYS;
  const int grid = m->ctx->num_sms;
  S2S_CHECK(m->arena.alloc(&m->dx, (size_t)B * d * 4));
  S2S_CHECK(m->arena.alloc(&m->dq, (size_t)B * d * 4));
  S2S_CHECK(m->arena.alloc(&m->dh, (size_t)B * f * 4));
  S2S_CHECK(m->arena.alloc(&m->part, (size_t)B * c.heads * m->s_max * 68 * 4));
  S2S_CHECK(m->arena.alloc(&m->attn16, (size_t)B * d * esz));
  S2S_CHECK(m->arena.alloc(&m->dx_alt, (size_t)2 * d * 4));
  S2S_CHECK(m->arena.alloc(&m->part_x0, (size_t)c.heads * 2 * d * 4));
  S2S_CHECK(m->arena.alloc(&m->part_x1, (size_t)c.heads * 2 * d * 4));
  S2S_CHECK(m->arena.alloc(&m->attn_cnt, (size_t)B * c.heads * 4));
  S2S_CHECK(m->arena.alloc(&m->self_kv, (size_t)B * c.dec_layers * 2 * c.max_target_positions * d * esz));
  S2S_CHECK(m->arena.alloc(&m->tokens, (size_t)B * c.max_target_positions * 4));
  S2S_CHECK(m->arena.alloc(&m->out_ids, (size_t)B * c.max_target_positions * 4));
  S2S_CHECK(m->arena.alloc(&m->out_len, B * 4));
  S2S_CHECK(m->arena.alloc(&m->done, B * 4));
  S2S_CHECK(m->arena.alloc(&m->n_done, 16));
  S2S_CHECK(m->arena.alloc(&m->cand_val, (size_t)B * grid * 4));
  S2S_CHECK(m->arena.alloc(&m->cand_idx, (size_t)B * grid * 4));
  S2S_CHECK(m->arena.alloc(&m->suppress, c.vocab));
  S2S_CHECK(m->arena.alloc(&m->suppress_lang, c.vocab));
  S2S_CHECK(m->arena.alloc(&m->sync_counter, 16));
  return S2S_OK;
}

int gemm(s2s_whisper* m, GemmProblem& p, cudaStream_t st) { return gemm_tc_launch(m->ctx, p, m->cfg.compute_dtype, st); }

GemmProblem plain_gemm(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t M, int N, int K) {
  GemmProblem p{};
  p.a = a; p.a_row_stride = lda; p.a_batch_stride = lda * M; p.w = w; p.ldw = ldw;
  p.M = (int32_t)M; p.N = N; p.K = K; p.batch = 1;
  p.out_batch_rows = 0; p.out_row_offset = 0;
  return p;
}

}  // namespace

extern "C" {

// source != nullptr: the new object reads source's weights (s2s_whisper_create_shared) and comes back finalized
static int create(s2s_ctx* ctx, const s2s_whisper_config* cfg, s2s_whisper* source, s2s_whisper** out) {
  S2S_REQUIRE(ctx && cfg && out, "whisper_create: null argument");
  S2S_REQUIRE(cfg->d_model % 64 == 0 && cfg->d_model / cfg->heads == 64, "whisper: head_dim must be 64 (d=%d heads=%d)",
              cfg->d_model, cfg->heads);
  S2S_REQUIRE(cfg->ffn % 64 == 0 && cfg->n_mels % 8 == 0, "whisper: ffn %% 64 and n_mels %% 8 required");
  S2S_REQUIRE(cfg->max_source_positions == 1500, "whisper: max_source_positions must be 1500");
  S2S_REQUIRE(cfg->compute_dtype == S2S_F16 || cfg->compute_dtype == S2S_BF16, "whisper: compute_dtype must be f16/bf16");
  S2S_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= 256, "whisper: max_batch in [1,256]");
  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  s2s_whisper* m = new s2s_whisper();
  m->ctx = ctx;
  m->cfg = *cfg;
  if (source) m->arena.borrow(source->arena);
  int r = build_tables(m);
  if (r == S2S_OK) r = alloc_weights(m);
  if (r == S2S_OK) r = alloc_workspace(m);
  if (r != S2S_OK) { s2s_whisper_destroy(m); return r; }
  m->finalized = source != nullptr;
  const char* dbg = getenv("S2S_DEBUG_PHASES");
  m->debug_phases = (dbg && dbg[0] == '1') ? 1 : 0;
  const char* cl = getenv("S2S_WHISPER_CLUSTER");  // "0": always use the 8-phase kernel (A/B comparisons)
  m->cluster_decode = (cl && cl[0] == '0') ? 0 : 1;
  *out = m;
  return S2S_OK;
}

int s2s_whisper_create(s2s_ctx* ctx, const s2s_whisper_config* cfg, s2s_whisper** out) { return create(ctx, cfg, nullptr, out); }

int s2s_whisper_create_shared(s2s_ctx* ctx, s2s_whisper* source, const s2s_whisper_config* cfg, s2s_whisper** out) {
  const char* who = "whisper create_shared";
  S2S_REQUIRE(ctx && source && cfg && out, "%s: null argument", who);
  S2S_REQUIRE(source->finalized, "%s: the source is not finalized", who);
  S2S_REQUIRE(source->ctx->device == ctx->device, "%s: the source is on device %d, the context on device %d", who,
              source->ctx->device, ctx->device);
  const s2s_whisper_config& s = source->cfg;
  S2S_REQUIRE_SAME(*cfg, s, d_model, who);
  S2S_REQUIRE_SAME(*cfg, s, heads, who);
  S2S_REQUIRE_SAME(*cfg, s, enc_layers, who);
  S2S_REQUIRE_SAME(*cfg, s, dec_layers, who);
  S2S_REQUIRE_SAME(*cfg, s, ffn, who);
  S2S_REQUIRE_SAME(*cfg, s, n_mels, who);
  S2S_REQUIRE_SAME(*cfg, s, vocab, who);
  S2S_REQUIRE_SAME(*cfg, s, max_source_positions, who);
  S2S_REQUIRE_SAME(*cfg, s, max_target_positions, who);
  S2S_REQUIRE_SAME(*cfg, s, compute_dtype, who);
  return create(ctx, cfg, source, out);
}

int s2s_whisper_device_bytes(s2s_whisper* m, int64_t* weights, int64_t* total) {
  S2S_REQUIRE(m && weights && total, "whisper device_bytes: null argument");
  *weights = (int64_t)m->arena.weight_bytes();
  *total = (int64_t)m->arena.bytes();
  return S2S_OK;
}

int s2s_whisper_destroy(s2s_whisper* m) {
  if (!m) return S2S_OK;
  if (m->tok_stage) cudaFreeHost(m->tok_stage);
  if (m->tok_event) cudaEventDestroy(m->tok_event);
  delete m;
  return S2S_OK;
}

int s2s_whisper_bind_tensor(s2s_whisper* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                            int32_t dtype) {
  S2S_REQUIRE(m && name && data_h && shape, "whisper bind_tensor: null argument");
  S2S_CHECK(m->arena.check_writable("whisper bind_tensor"));
  if (strcmp(name, "proj_out.weight") == 0) return S2S_OK;  // tied to embed_tokens
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  return m->arena.bind("whisper", name, data_h, shape, ndim, dtype, m->cfg.compute_dtype);
}

int s2s_whisper_init_random(s2s_whisper* m, uint64_t seed) {
  S2S_REQUIRE(m, "whisper init_random: null model");
  S2S_CHECK(m->arena.check_writable("whisper init_random"));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  return m->arena.init_random(seed, m->cfg.compute_dtype);
}

int s2s_whisper_finalize(s2s_whisper* m) {
  S2S_REQUIRE(m, "whisper finalize: null model");
  S2S_CHECK(m->arena.check_writable("whisper finalize"));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(m->arena.check_all_bound("whisper"));
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  m->arena.release_staging();
  m->finalized = true;
  return S2S_OK;
}

int s2s_whisper_logmel(s2s_whisper* m, const float* pcm_d, int64_t pcm_stride, const int32_t* n_samples_h, int32_t B,
                       float* mel_out_d, void* stream) {
  S2S_REQUIRE(m && pcm_d && n_samples_h, "logmel: null argument");
  S2S_REQUIRE(B >= 1 && B <= m->cfg.max_batch, "logmel: B=%d outside [1,%d]", B, m->cfg.max_batch);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  for (int b = 0; b < B; ++b)
    S2S_REQUIRE(n_samples_h[b] >= 0 && ((n_samples_h[b] < N_SAMPLES ? n_samples_h[b] : N_SAMPLES) <= pcm_stride),
                "logmel: n_samples[%d]=%d exceeds stride", b, n_samples_h[b]);
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->n_samples_d, n_samples_h, B * sizeof(int), cudaMemcpyHostToDevice, st));
  LogmelTables tb{m->hann, m->twiddle, m->fb, m->fb_range};
  S2S_CHECK(logmel_launch(tb, pcm_d, pcm_stride, m->n_samples_d, B, m->cfg.n_mels, m->mel_f32, m->mel_max, m->mel_t,
                          m->cfg.compute_dtype, st));
  if (mel_out_d)
    S2S_CHECK_CUDA(cudaMemcpyAsync(mel_out_d, m->mel_f32, (size_t)B * m->cfg.n_mels * N_FRAMES * 4, cudaMemcpyDeviceToDevice, st));
  return S2S_OK;
}

int s2s_whisper_encode(s2s_whisper* m, const float* mel_in_d, int32_t B, float* enc_out_d, void* stream) {
  S2S_REQUIRE(m && m->finalized, "encode: model not finalized");
  S2S_REQUIRE(B >= 1 && B <= m->cfg.max_batch, "encode: B=%d outside [1,%d]", B, m->cfg.max_batch);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, T = c.max_source_positions, dt = c.compute_dtype, esz = m->esz;
  const int64_t rows = (int64_t)B * T;
  if (mel_in_d)
    S2S_CHECK(logmel_finalize_launch(mel_in_d, m->mel_max, 0, B, c.n_mels, nullptr, m->mel_t, dt, st));

  // conv1 (k=3, s=1, pad=1) + GELU as a strided-window GEMM over the padded, transposed mel: K = 3 * n_mels
  {
    GemmProblem p{};
    p.a = m->mel_t; p.a_row_stride = c.n_mels; p.a_batch_stride = (int64_t)(N_FRAMES + 2) * c.n_mels;
    p.w = m->conv1_w; p.ldw = 3 * c.n_mels; p.M = N_FRAMES; p.N = d; p.K = 3 * c.n_mels; p.batch = B;
    p.bias = m->conv1_b; p.act = 1; p.out_h = m->h1; p.ldo_h = d;
    p.out_batch_rows = N_FRAMES + 2; p.out_row_offset = 1;
    S2S_CHECK(gemm(m, p, st));
  }
  // conv2 (k=3, s=2, pad=1) + GELU + positional embedding -> fp32 residual stream x [B*1500, d]
  {
    GemmProblem p{};
    p.a = m->h1; p.a_row_stride = 2 * d; p.a_batch_stride = (int64_t)(N_FRAMES + 2) * d;
    p.w = m->conv2_w; p.ldw = 3 * d; p.M = T; p.N = d; p.K = 3 * d; p.batch = B;
    p.bias = m->conv2_b; p.act = 1; p.out_f = m->x; p.ldo_f = d;
    p.resid = m->enc_pos; p.ld_resid = d; p.resid_mode = 2;
    p.out_batch_rows = T; p.out_row_offset = 0;
    S2S_CHECK(gemm(m, p, st));
  }
  for (int i = 0; i < c.enc_layers; ++i) {
    const EncLayer& L = m->enc[i];
    S2S_CHECK(norm_rows_launch(m->x, L.ln1_w, L.ln1_b, 1e-5f, rows, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = plain_gemm(m->xn, d, L.w_qkv, d, rows, 3 * d, d);
      p.bias = L.b_qkv; p.out_h = m->qkv; p.ldo_h = 3 * d;
      S2S_CHECK(gemm(m, p, st));
    }
    S2S_CHECK(attention_tc_launch(m->ctx, m->qkv, off(m->qkv, d, esz), off(m->qkv, 2 * d, esz), m->attn, B, T, T, c.heads,
                                   c.heads, 64, 3 * d, 3 * d, 3 * d, d, 1.0f, 0, dt, m->vt, m->vt_elems, st));
    {
      GemmProblem p = plain_gemm(m->attn, d, L.w_o, d, rows, d, d);
      p.bias = L.b_o; p.out_f = m->x; p.ldo_f = d; p.resid = m->x; p.ld_resid = d; p.resid_mode = 1;
      S2S_CHECK(gemm(m, p, st));
    }
    S2S_CHECK(norm_rows_launch(m->x, L.ln2_w, L.ln2_b, 1e-5f, rows, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = plain_gemm(m->xn, d, L.w_fc1, d, rows, f, d);
      p.bias = L.b_fc1; p.act = 1; p.out_h = m->hbuf; p.ldo_h = f;
      S2S_CHECK(gemm(m, p, st));
    }
    {
      GemmProblem p = plain_gemm(m->hbuf, f, L.w_fc2, f, rows, d, f);
      p.bias = L.b_fc2; p.out_f = m->x; p.ldo_f = d; p.resid = m->x; p.ld_resid = d; p.resid_mode = 1;
      S2S_CHECK(gemm(m, p, st));
    }
  }
  S2S_CHECK(norm_rows_launch(m->x, m->enc_lnf_w, m->enc_lnf_b, 1e-5f, rows, d, m->enc_out, enc_out_d, dt, st));
  // cross-attention K/V for every decoder layer in one GEMM: [rows, Ld*2*d]
  {
    GemmProblem p = plain_gemm(m->enc_out, d, m->ckv_w, d, rows, c.dec_layers * 2 * d, d);
    p.bias = m->ckv_b; p.out_h = m->cross_kv; p.ldo_h = (int64_t)c.dec_layers * 2 * d;
    p.head_major_rows = T;  // [b][layer][k|v][head][t][64]: a head's keys are contiguous for the decoder
    S2S_CHECK(gemm(m, p, st));
  }
  m->last_B = B;
  return S2S_OK;
}

static int decode_impl(s2s_whisper* m, const int32_t* prefix_h, const int32_t* prefix_rows_h, int n_prefix, int max_new, int eos,
                       const unsigned char* suppress_d, int32_t B, int32_t* ids_out_d, int32_t* len_out_d,
                       const int32_t* forced_d, float* logits_out_d, cudaStream_t st) {
  const auto& c = m->cfg;
  const int d = c.d_model, esz = m->esz;
  S2S_REQUIRE(B >= 1 && B <= m->last_B, "decode: B=%d but %d utterances are encoded", B, m->last_B);
  S2S_REQUIRE(n_prefix >= 1 && max_new >= 1 && n_prefix + max_new <= c.max_target_positions,
              "decode: n_prefix %d + max_new %d > %d", n_prefix, max_new, c.max_target_positions);
  // prompt tokens for every row, through a pinned staging buffer owned by the model: no stream synchronisation per call
  // (the event only waits for the PREVIOUS call's copy, long finished in steady state)
  if (!m->tok_stage) {
    S2S_CHECK_CUDA(cudaHostAlloc(&m->tok_stage, (size_t)c.max_batch * c.max_target_positions * 4, cudaHostAllocDefault));
    S2S_CHECK_CUDA(cudaEventCreateWithFlags(&m->tok_event, cudaEventDisableTiming));
  } else {
    S2S_CHECK_CUDA(cudaEventSynchronize(m->tok_event));
  }
  for (int b = 0; b < B; ++b) {
    const int32_t* row = prefix_rows_h ? prefix_rows_h + (size_t)b * n_prefix : prefix_h;
    for (int i = 0; i < n_prefix; ++i) {
      S2S_REQUIRE(row[i] >= 0 && row[i] < c.vocab, "decode: prefix token %d out of range", row[i]);
      m->tok_stage[(size_t)b * c.max_target_positions + i] = row[i];
    }
  }
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->tokens, m->tok_stage, (size_t)B * c.max_target_positions * 4, cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaEventRecord(m->tok_event, st));
  const int group = whisper_decode_max_batch(d, c.ffn);  // sessions per persistent launch (<= 16)
  for (int b0 = 0; b0 < B; b0 += group) {
    const int nb = (B - b0) < group ? (B - b0) : group;
    WhisperDecParams p{};
    p.d = d; p.heads = c.heads; p.layers = c.dec_layers; p.ffn = c.ffn; p.vocab = c.vocab; p.B = nb;
    p.max_pos = c.max_target_positions; p.n_ctx = c.max_source_positions;
    p.lw = m->dec_d; p.embed = m->embed; p.pos = m->dec_pos; p.lnf_w = m->dec_lnf_w; p.lnf_b = m->dec_lnf_b;
    p.x = m->dx + (size_t)b0 * d; p.q = m->dq + (size_t)b0 * d; p.h = off(m->dh, (int64_t)b0 * c.ffn, esz);
    p.self_kv = off(m->self_kv, (int64_t)b0 * c.dec_layers * 2 * c.max_target_positions * d, esz);
    p.cross_kv = off(m->cross_kv, (int64_t)b0 * c.max_source_positions * c.dec_layers * 2 * d, esz);  // head-major
    p.part = m->part + (size_t)b0 * c.heads * m->s_max * 68; p.s_max = m->s_max;
    p.attn16 = off(m->attn16, (int64_t)b0 * d, esz); p.attn_cnt = m->attn_cnt + (size_t)b0 * c.heads;
    // 1-2 sessions: the cluster kernel (4 grid-wide phases per layer); its buffers hold one group at a time
    p.x_alt = m->dx_alt; p.part_x0 = m->part_x0; p.part_x1 = m->part_x1; p.cluster_size = m->cluster_decode ? 8 : 0;
    p.tokens = m->tokens + (size_t)b0 * c.max_target_positions;
    p.n_prefix = n_prefix; p.max_new = max_new; p.eos = eos; p.suppress = suppress_d;
    p.out_ids = ids_out_d + (size_t)b0 * max_new; p.out_len = len_out_d + b0;
    p.forced = forced_d ? forced_d + (size_t)b0 * max_new : nullptr;
    p.logits_out = nullptr;
    if (logits_out_d) {
      S2S_REQUIRE(B <= group, "decode: logits_out requires B <= %d", group);
      p.logits_out = logits_out_d;
    }
    p.done = m->done + b0; p.n_done = m->n_done; p.cand_val = m->cand_val + (size_t)b0 * m->ctx->num_sms;
    p.cand_idx = m->cand_idx + (size_t)b0 * m->ctx->num_sms; p.sync_counter = m->sync_counter;
    p.trace = m->trace; p.trace_cap = m->trace_cap;
    S2S_CHECK(whisper_decode_launch(m->ctx, p, c.compute_dtype, m->debug_phases, st));
  }
  return S2S_OK;
}

static int upload_suppress(s2s_whisper* m, unsigned char* dst, const int32_t* always, int n_always, const int32_t* begin,
                           int n_begin, bool invert_always, cudaStream_t st) {
  // the mask is a pure function of the id lists: rebuilt and uploaded only when they change (once per handler in practice)
  std::vector<int>& key = m->suppress_key[dst == m->suppress ? 0 : 1];
  std::vector<int> now;
  now.reserve((size_t)n_always + n_begin + 2);
  now.push_back(n_always); now.push_back(invert_always ? 1 : 0);
  now.insert(now.end(), always, always + n_always);
  now.insert(now.end(), begin, begin + n_begin);
  if (now == key) return S2S_OK;
  std::vector<unsigned char> mask((size_t)m->cfg.vocab, invert_always ? 1 : 0);
  for (int i = 0; i < n_always; ++i) {
    S2S_REQUIRE(always[i] >= 0 && always[i] < m->cfg.vocab, "suppress id %d out of range", always[i]);
    if (invert_always) mask[(size_t)always[i]] = 0; else mask[(size_t)always[i]] |= 1;
  }
  for (int i = 0; i < n_begin; ++i) {
    S2S_REQUIRE(begin[i] >= 0 && begin[i] < m->cfg.vocab, "begin-suppress id %d out of range", begin[i]);
    mask[(size_t)begin[i]] |= 2;
  }
  S2S_CHECK_CUDA(cudaMemcpyAsync(dst, mask.data(), mask.size(), cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));
  key.swap(now);
  return S2S_OK;
}

int s2s_whisper_decode(s2s_whisper* m, const s2s_whisper_decode_opts* o, int32_t B, int32_t* ids_out_d,
                       int32_t* len_out_d, const int32_t* forced_d, float* logits_out_d, void* stream) {
  S2S_REQUIRE(m && m->finalized && o && ids_out_d && len_out_d, "decode: null argument / model not finalized");
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(upload_suppress(m, m->suppress, o->suppress_h, o->n_suppress, o->begin_suppress_h, o->n_begin_suppress, false, st));
  return decode_impl(m, o->prefix_h, o->prefix_rows_h, o->n_prefix, o->max_new_tokens, o->eos_id, m->suppress, B, ids_out_d, len_out_d,
                     forced_d, logits_out_d, st);
}

int32_t s2s_whisper_max_decode_batch(s2s_whisper* m) {
  if (!m) return 0;
  return whisper_decode_max_batch(m->cfg.d_model, m->cfg.ffn);
}

int s2s_whisper_set_trace(s2s_whisper* m, uint64_t* trace_d, int32_t capacity) {
  S2S_REQUIRE(m, "set_trace: null model");
  m->trace = reinterpret_cast<unsigned long long*>(trace_d);
  m->trace_cap = trace_d ? capacity : 0;
  return S2S_OK;
}

int s2s_whisper_detect_language(s2s_whisper* m, int32_t sot_id, const int32_t* lang_ids_h, int32_t n_lang, int32_t B,
                                int32_t* lang_out_d, void* stream) {
  S2S_REQUIRE(m && m->finalized && lang_ids_h && lang_out_d && n_lang > 0, "detect_language: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(upload_suppress(m, m->suppress_lang, lang_ids_h, n_lang, nullptr, 0, true, st));
  // eos = -1: never matches, so the single generated id is returned as is
  return decode_impl(m, &sot_id, nullptr, 1, 1, -1, m->suppress_lang, B, lang_out_d, m->out_len, nullptr, nullptr, st);
}

int s2s_whisper_transcribe(s2s_whisper* m, const s2s_whisper_decode_opts* o, const float* pcm_h, int64_t pcm_stride,
                           const int32_t* n_samples_h, int32_t B, int32_t* ids_out_h, int32_t* len_out_h, void* stream) {
  S2S_REQUIRE(m && m->finalized && o && pcm_h && n_samples_h && ids_out_h && len_out_h, "transcribe: null argument");
  S2S_REQUIRE(B >= 1 && B <= m->cfg.max_batch, "transcribe: B=%d outside [1,%d]", B, m->cfg.max_batch);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  for (int b = 0; b < B; ++b) {
    const int n = n_samples_h[b] < N_SAMPLES ? n_samples_h[b] : N_SAMPLES;
    S2S_REQUIRE(n >= 0 && n <= pcm_stride, "transcribe: n_samples[%d] invalid", b);
    S2S_CHECK_CUDA(cudaMemcpyAsync(m->pcm + (size_t)b * N_SAMPLES, pcm_h + (size_t)b * pcm_stride, (size_t)n * 4,
                                   cudaMemcpyHostToDevice, st));
  }
  S2S_CHECK(s2s_whisper_logmel(m, m->pcm, N_SAMPLES, n_samples_h, B, nullptr, stream));
  S2S_CHECK(s2s_whisper_encode(m, nullptr, B, nullptr, stream));
  S2S_CHECK(s2s_whisper_decode(m, o, B, m->out_ids, m->out_len, nullptr, nullptr, stream));
  S2S_CHECK_CUDA(cudaMemcpyAsync(ids_out_h, m->out_ids, (size_t)B * o->max_new_tokens * 4, cudaMemcpyDeviceToHost, st));
  S2S_CHECK_CUDA(cudaMemcpyAsync(len_out_h, m->out_len, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));
  return S2S_OK;
}

}  // extern "C"
