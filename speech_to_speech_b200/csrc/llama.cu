// llama.cu -- Llama-family LLM model object behind the C ABI: weight arena (transformers state-dict names ->
// kernel layouts), per-session KV cache, prefill launch sequence (wgmma GEMMs + causal GQA attention) and
// the persistent greedy decode.  Replaces the device work of LanguageModelHandler._generate
// (reference S/LLM/language_model.py:832-892: tokenizer -> pipeline("text-generation") -> streamer).
//
// Layout choices:
//   * q_proj / k_proj rows are permuted so that the rotate_half partners (j, j + hd/2) of every head are stored
//     adjacently (2j, 2j+1): RoPE becomes a 2-element rotation inside one thread both in the decode GEMV epilogue
//     and in the prefill RoPE kernel; q.k dot products are invariant under the common permutation.
//   * gate_proj / up_proj rows are interleaved (gate_i, up_i): SwiGLU is fused into the producing GEMM / GEMV epilogue.
#include <math.h>
#include <algorithm>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "llama_decode.cuh"
#include "llama_model.cuh"

namespace {

template <typename T>
__global__ void embed_gather_kernel(const int* __restrict__ ids, const T* __restrict__ embed, float* __restrict__ x, int d) {
  const int t = blockIdx.x;
  const T* e = embed + (long long)ids[t] * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) x[(long long)t * d + i] = DT<T>::to_f(e[i]);
}

// qkv [n, qd + 2*kvd] (q,k pair-adjacent layout): rotate q in place, rotate k -> cache, copy v -> cache.
template <typename T>
__global__ void rope_prefill_kernel(T* __restrict__ qkv, int n, int qd, int kvd, int hd, int past,
                                    const float2* __restrict__ rope, T* __restrict__ kcache, T* __restrict__ vcache) {
  const int t = blockIdx.x;
  const int ld = qd + 2 * kvd;
  T* row = qkv + (long long)t * ld;
  const float2* cs = rope + (long long)(past + t) * (hd >> 1);
  for (int i = threadIdx.x * 2; i < ld; i += blockDim.x * 2) {
    uint32_t u = *reinterpret_cast<uint32_t*>(row + i);
    if (i < qd + kvd) {
      const float2 v = DT<T>::to_f2(u);
      const float2 c = cs[(i % hd) >> 1];
      u = DT<T>::pack2(v.x * c.x - v.y * c.y, v.y * c.x + v.x * c.y);
    }
    if (i < qd) *reinterpret_cast<uint32_t*>(row + i) = u;
    else if (i < qd + kvd) *reinterpret_cast<uint32_t*>(kcache + (long long)(past + t) * kvd + (i - qd)) = u;
    else *reinterpret_cast<uint32_t*>(vcache + (long long)(past + t) * kvd + (i - qd - kvd)) = u;
  }
}

// Qwen3 (qk_norm): per (token, head) RMSNorm over head_dim (fp32 statistics, Qwen3RMSNorm) then RoPE; q in place,
// k -> cache, v -> cache.  One CTA per token, a warp per head; rows and norm weights are stored pair-adjacent.
template <typename T, int HD>
__global__ void qknorm_rope_prefill_kernel(T* __restrict__ qkv, int H, int KV, int past, const float2* __restrict__ rope,
                                           const float* __restrict__ qn, const float* __restrict__ kn, float eps,
                                           T* __restrict__ kcache, T* __restrict__ vcache) {
  constexpr int PER = HD / 32;
  const int t = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int qd = H * HD, kvd = KV * HD, ld = qd + 2 * kvd;
  T* row = qkv + (long long)t * ld;
  const float2* cs = rope + (long long)(past + t) * (HD >> 1);
  for (int h = warp; h < H + KV; h += nw) {
    T* src = row + h * HD + lane * PER;
    const float* g = (h < H ? qn : kn) + lane * PER;
    float v[PER];
#pragma unroll
    for (int i = 0; i < PER; i += 2) { const float2 f = DT<T>::to_f2(*reinterpret_cast<const uint32_t*>(src + i)); v[i] = f.x; v[i + 1] = f.y; }
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < PER; ++i) ss = fmaf(v[i], v[i], ss);
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss * (1.0f / (float)HD) + eps);
    T* dst = h < H ? src : kcache + (long long)(past + t) * kvd + (h - H) * HD + lane * PER;
#pragma unroll
    for (int i = 0; i < PER; i += 2) {
      const float2 c = cs[(lane * PER + i) >> 1];
      const float a0 = v[i] * rstd * g[i], a1 = v[i + 1] * rstd * g[i + 1];
      *reinterpret_cast<uint32_t*>(dst + i) = DT<T>::pack2(a0 * c.x - a1 * c.y, a1 * c.x + a0 * c.y);
    }
  }
  for (int i = threadIdx.x * 2; i < kvd; i += blockDim.x * 2)
    *reinterpret_cast<uint32_t*>(vcache + (long long)(past + t) * kvd + i) = *reinterpret_cast<const uint32_t*>(row + qd + kvd + i);
}

// the lowest id among the maxima; NaN never compares greater, so it counts as -inf: starting from (-inf, id 0) makes a row with
// nothing above -inf (all -inf and / or NaN) give id 0, a valid id, instead of the start value
__global__ void argmax_row_kernel(const float* __restrict__ logits, int n, int* __restrict__ out) {
  __shared__ float sv[32];
  __shared__ int si[32];
  float bv = -INFINITY; int bi = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = logits[i];
    if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (sv[w] > bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
    *out = bi;
  }
}

// sampling.cuh's choice for one row (prefill).  The chosen id joins the seen set only when it is fed (the decode launch):
// the choice after an intermediate chunk of a long prompt is discarded.
__global__ void __launch_bounds__(1024) sample_row_kernel(const float* __restrict__ row, int n, const SampSlot s,
                                                          const unsigned int* seen, int pred_pos, int* __restrict__ out) {
  __shared__ SampShared sh;
  const int tok = sample_row(row, n, s, seen, pred_pos, sh);
  if (threadIdx.x == 0) *out = tok;
}

__global__ void seen_set_kernel(const int* __restrict__ ids, int n, unsigned int* seen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicOr(seen + (ids[i] >> 5), 1u << (ids[i] & 31));
}

constexpr int MAX_DEC_B = LLAMA_MAX_DEC_B;

int build(s2s_llama* m) {
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, hd = c.head_dim, qd = c.heads * hd, kvd = c.kv_heads * hd;
  const int esz = 2;
  auto off = [&](void* base, int64_t elems) { return reinterpret_cast<char*>(base) + elems * esz; };
  m->n_tables = c.n_tables > 1 ? c.n_tables : 1;
  m->embed_table_elems = (size_t)c.vocab * d;
  S2S_CHECK(m->arena.alloc_weights(&m->embed, m->n_tables * m->embed_table_elems * esz));
  S2S_CHECK(m->arena.alloc_weights(&m->norm_f, d * 4));
  WeightArena& A = m->arena;
  if (m->n_tables == 1) {
    A.add("model.embed_tokens.weight", m->embed, true, (int64_t)c.vocab * d);
  } else {  // code predictor: one table / head per codebook (Qwen3OmniMoeTalkerCodePredictorModel.codec_embedding, .lm_head)
    for (int t = 0; t < m->n_tables; ++t)
      A.add("model.embed_tokens." + std::to_string(t) + ".weight", off(m->embed, (int64_t)t * m->embed_table_elems), true, (int64_t)c.vocab * d);
  }
  A.add("model.norm.weight", m->norm_f, false, d, 0.1f, 1.0f);
  m->layers_h.resize(c.layers);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "model.layers." + std::to_string(i) + ".";
    float *n1, *n2, *qn = nullptr, *kn = nullptr;
    S2S_CHECK(A.alloc_weights(&n1, d * 4));
    S2S_CHECK(A.alloc_weights(&n2, d * 4));
    A.add(p + "input_layernorm.weight", n1, false, d, 0.1f, 1.0f);
    A.add(p + "post_attention_layernorm.weight", n2, false, d, 0.1f, 1.0f);
    if (c.qk_norm) {  // Qwen3Attention.q_norm / k_norm: RMSNorm(head_dim), permuted like the q/k rows
      S2S_CHECK(A.alloc_weights(&qn, hd * 4));
      S2S_CHECK(A.alloc_weights(&kn, hd * 4));
      A.add(p + "self_attn.q_norm.weight", qn, false, hd, 0.1f, 1.0f).as(W_ROPE_PERM, hd, 1, 0, hd);
      A.add(p + "self_attn.k_norm.weight", kn, false, hd, 0.1f, 1.0f).as(W_ROPE_PERM, hd, 1, 0, hd);
    }
    LlamaDecLayer& L = m->layers_h[i];
    L.norm1 = n1; L.norm2 = n2; L.q_norm = qn; L.k_norm = kn;
  }
  S2S_CHECK(m->arena.alloc(&m->layers_d, sizeof(LlamaDecLayer) * c.layers));

  // RoPE table, float32 arithmetic like LlamaRotaryEmbedding (modeling_llama.py:73-137)
  {
    std::vector<float2> tab((size_t)c.max_positions * (hd / 2));
    for (int j = 0; j < hd / 2; ++j) {
      const float inv = 1.0f / powf(c.rope_theta, (float)(2 * j) / (float)hd);
      for (int p = 0; p < c.max_positions; ++p) {
        const float ang = (float)p * inv;
        tab[(size_t)p * (hd / 2) + j] = make_float2(cosf(ang), sinf(ang));
      }
    }
    S2S_CHECK(m->arena.alloc(&m->rope, tab.size() * sizeof(float2)));
    S2S_CHECK_CUDA(cudaMemcpy(m->rope, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  // KV cache [slot][layer][2][max_pos][kvd]
  m->kv_which_stride = (long long)c.max_positions * kvd;
  m->kv_layer_stride = 2 * m->kv_which_stride;
  m->kv_slot_stride = (long long)c.layers * m->kv_layer_stride;
  S2S_CHECK(m->arena.alloc(&m->kv, (size_t)c.max_sessions * m->kv_slot_stride * esz));
  m->len.assign(c.max_sessions, 0);
  // prefill workspace
  const int P = c.max_prefill;
  S2S_CHECK(m->arena.alloc(&m->ids_d, (size_t)P * 4));
  S2S_CHECK(m->arena.alloc(&m->x, (size_t)P * d * 4));
  S2S_CHECK(m->arena.alloc(&m->xn, (size_t)P * d * esz));
  S2S_CHECK(m->arena.alloc(&m->qkv, (size_t)P * (qd + 2 * kvd) * esz));
  S2S_CHECK(m->arena.alloc(&m->attn, (size_t)P * qd * esz));
  S2S_CHECK(m->arena.alloc(&m->hbuf, (size_t)P * f * esz));
  S2S_CHECK(m->arena.alloc(&m->last_logits, (size_t)c.vocab * 4));
  S2S_CHECK(m->arena.alloc(&m->batch_logits, (size_t)MAX_DEC_B * c.vocab * 4));
  m->vt_elems = attention_tc_scratch_elems(1, c.max_positions, c.kv_heads, hd);
  S2S_CHECK(m->arena.alloc(&m->vt, m->vt_elems * esz));
  // decode state
  m->s_max = (c.max_positions + 63) / 64;
  const int grid = m->ctx->num_sms;
  S2S_CHECK(m->arena.alloc(&m->dx, (size_t)MAX_DEC_B * d * 4));
  S2S_CHECK(m->arena.alloc(&m->dq, (size_t)MAX_DEC_B * qd * 4));
  S2S_CHECK(m->arena.alloc(&m->dh, (size_t)MAX_DEC_B * f * 4));
  S2S_CHECK(m->arena.alloc(&m->part, (size_t)MAX_DEC_B * c.heads * m->s_max * (hd + 4) * 4));
  S2S_CHECK(m->arena.alloc(&m->attn16, (size_t)MAX_DEC_B * qd * 2));
  S2S_CHECK(m->arena.alloc(&m->attn_cnt, (size_t)MAX_DEC_B * c.heads * 4));
  S2S_CHECK(m->arena.alloc(&m->slot_d, MAX_DEC_B * 4));
  S2S_CHECK(m->arena.alloc(&m->pos_d, MAX_DEC_B * 4));
  S2S_CHECK(m->arena.alloc(&m->done, MAX_DEC_B * 4));
  S2S_CHECK(m->arena.alloc(&m->n_done, 16));
  S2S_CHECK(m->arena.alloc(&m->cand_val, (size_t)MAX_DEC_B * grid * 4));
  S2S_CHECK(m->arena.alloc(&m->cand_idx, (size_t)MAX_DEC_B * grid * 4));
  S2S_CHECK(m->arena.alloc(&m->out_ids, (size_t)MAX_DEC_B * c.max_positions * 4));
  S2S_CHECK(m->arena.alloc(&m->out_len, MAX_DEC_B * 4));
  S2S_CHECK(m->arena.alloc(&m->next_id, 16));
  S2S_CHECK(m->arena.alloc(&m->sync_counter, 16));
  S2S_CHECK(m->arena.alloc(&m->kraw, (size_t)MAX_DEC_B * kvd * 4));
  S2S_CHECK(m->arena.alloc(&m->qn, (size_t)MAX_DEC_B * qd * 4));
  m->samp.assign(c.max_sessions, samp_greedy());
  m->seen_words = (c.vocab + 31) / 32;
  m->seen_stale.assign(c.max_sessions, 0);
  S2S_CHECK(m->arena.alloc(&m->samp_d, MAX_DEC_B * sizeof(SampSlot)));
  S2S_CHECK(m->arena.alloc(&m->samp_rows, (size_t)MAX_DEC_B * c.vocab * 4));
  S2S_CHECK(m->arena.alloc(&m->seen, (size_t)c.max_sessions * m->seen_words * 4));
  return S2S_OK;
}

// The projections and lm_head, stored once in the tiled layout that the decode kernel streams and the prefill GEMMs read
// (16-bit tiles, or FP8 codes + row scales).  Allocated at the first bind / init_random / finalize, which fixes the weight
// format; bind and init_random write each tensor's rows straight into place.
int alloc_matrices(s2s_llama* m) {
  if (m->matrices) return S2S_OK;
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, hd = c.head_dim, qd = c.heads * hd, kvd = c.kv_heads * hd, nqkv = qd + 2 * kvd;
  const bool f8 = m->weight_format == S2S_FP8_E4M3;
  auto tbytes = [f8](int N, int K) { return f8 ? tiled_fp8_weight_bytes(N, K) : tiled_weight_elems(N, K) * 2; };
  WeightArena& A = m->arena;
  A.tiled_format = m->weight_format;
  const float sd = 1.0f / sqrtf((float)d);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "model.layers." + std::to_string(i) + ".";
    void *w_qkv, *w_o, *w_gu, *w_down;
    S2S_CHECK(A.alloc_weights(&w_qkv, tbytes(nqkv, d)));
    S2S_CHECK(A.alloc_weights(&w_o, tbytes(d, qd)));
    S2S_CHECK(A.alloc_weights(&w_gu, tbytes(2 * f, d)));
    S2S_CHECK(A.alloc_weights(&w_down, tbytes(d, f)));
    A.add(p + "self_attn.q_proj.weight", w_qkv, true, (int64_t)qd * d, 2.0f * sd).as(W_ROPE_PERM, qd, d, 0, hd).tiled(nqkv, d, 0);
    A.add(p + "self_attn.k_proj.weight", w_qkv, true, (int64_t)kvd * d, 2.0f * sd).as(W_ROPE_PERM, kvd, d, 0, hd).tiled(nqkv, d, qd);
    A.add(p + "self_attn.v_proj.weight", w_qkv, true, (int64_t)kvd * d, 0.8f * sd).tiled(nqkv, d, qd + kvd);
    A.add(p + "self_attn.o_proj.weight", w_o, true, (int64_t)d * qd, 1.0f * sd).tiled(d, qd);
    A.add(p + "mlp.gate_proj.weight", w_gu, true, (int64_t)f * d, 1.0f * sd).as(W_INTERLEAVE, f, d, 0, 0).tiled(2 * f, d, 0, 2);
    A.add(p + "mlp.up_proj.weight", w_gu, true, (int64_t)f * d, 1.0f * sd).as(W_INTERLEAVE, f, d, 0, 1).tiled(2 * f, d, 1, 2);
    A.add(p + "mlp.down_proj.weight", w_down, true, (int64_t)d * f, 0.7f / sqrtf((float)f)).tiled(d, f);
    LlamaDecLayer& L = m->layers_h[i];
    L.w_qkv = w_qkv; L.w_o = w_o; L.w_gu = w_gu; L.w_down = w_down;
  }
  m->head_t_table_elems = tiled_weight_elems(c.vocab, d);
  S2S_CHECK(A.alloc_weights(&m->lm_head_t, f8 ? tbytes(c.vocab, d) : m->n_tables * m->head_t_table_elems * 2));
  if (m->n_tables == 1) {
    A.add("lm_head.weight", m->lm_head_t, true, (int64_t)c.vocab * d).tiled(c.vocab, d);
  } else {
    for (int t = 0; t < m->n_tables; ++t)
      A.add("lm_head." + std::to_string(t) + ".weight", reinterpret_cast<char*>(m->lm_head_t) + (size_t)t * m->head_t_table_elems * 2,
            true, (int64_t)c.vocab * d).tiled(c.vocab, d);
  }
  S2S_CHECK_CUDA(cudaMemcpy(m->layers_d, m->layers_h.data(), sizeof(LlamaDecLayer) * c.layers, cudaMemcpyHostToDevice));
  m->matrices = true;
  return S2S_OK;
}

// a prefill GEMM over one of the model's tiled matrices
GemmProblem lgemm(const s2s_llama* m, const void* a, int64_t lda, const void* w, int64_t M, int N, int K) {
  GemmProblem p{};
  p.a = a; p.a_row_stride = lda; p.a_batch_stride = lda * M; p.w = w;
  p.M = (int32_t)M; p.N = N; p.K = K; p.batch = 1;
  p.w_layout = m->weight_format == S2S_FP8_E4M3 ? GEMM_W_TILED_FP8 : GEMM_W_TILED16;
  return p;
}

}  // namespace

int llama_max_decode_batch_of(const s2s_llama* m) {
  return std::min(MAX_DEC_B, llama_decode_max_batch(m->ctx->device, m->cfg.compute_dtype, m->weight_format, m->cfg.d_model, m->cfg.ffn,
                                                    m->cfg.heads * m->cfg.head_dim, dec_grid(m->ctx)));
}

void llama_fill_dec_params(s2s_llama* m, LlamaDecParams& p) {
  const auto& c = m->cfg;
  p.d = c.d_model; p.heads = c.heads; p.kv_heads = c.kv_heads; p.hd = c.head_dim; p.layers = c.layers; p.ffn = c.ffn;
  p.vocab = c.vocab; p.max_pos = c.max_positions; p.eps = c.rms_eps;
  p.lw = m->layers_d; p.embed = m->embed; p.lm_head = m->lm_head_t; p.norm_f = m->norm_f; p.rope = m->rope;
  p.x = m->dx; p.q = m->dq; p.h = m->dh; p.kv = m->kv;
  p.kv_slot_stride = m->kv_slot_stride; p.kv_layer_stride = m->kv_layer_stride; p.kv_which_stride = m->kv_which_stride;
  p.part = m->part; p.s_max = m->s_max; p.attn16 = m->attn16; p.attn_cnt = m->attn_cnt;
  p.done = m->done; p.n_done = m->n_done; p.cand_val = m->cand_val; p.cand_idx = m->cand_idx; p.sync_counter = m->sync_counter;
  p.trace = m->trace; p.trace_cap = m->trace_cap;
  p.qk_norm = c.qk_norm ? 1 : 0; p.kraw = m->kraw; p.qn = m->qn;
  p.samp_rows = m->samp_rows; p.seen = m->seen; p.seen_words = m->seen_words;
}

int samp_from_abi(const s2s_sampling* s, int vocab, const char* who, SampSlot* out) {
  SampSlot t = samp_greedy();
  if (s) {
    S2S_REQUIRE(!s->do_sample || s->temperature > 0.f, "%s: do_sample needs temperature > 0 (got %g)", who, (double)s->temperature);
    S2S_REQUIRE(s->top_p > 0.f && s->top_p <= 1.f, "%s: top_p %g outside (0, 1]", who, (double)s->top_p);
    S2S_REQUIRE(s->top_k >= 0, "%s: top_k %d < 0", who, s->top_k);
    S2S_REQUIRE(s->repetition_penalty > 0.f, "%s: repetition_penalty %g <= 0", who, (double)s->repetition_penalty);
    S2S_REQUIRE(s->min_new_tokens >= 0, "%s: min_new_tokens %d < 0", who, s->min_new_tokens);
    S2S_REQUIRE(s->n_eos >= 0 && s->n_eos <= 8, "%s: %d EOS ids (at most 8)", who, s->n_eos);
    for (int e = 0; e < s->n_eos; ++e)
      S2S_REQUIRE(s->eos_ids[e] >= 0 && s->eos_ids[e] < vocab, "%s: EOS id %d outside the vocabulary", who, s->eos_ids[e]);
    t.do_sample = s->do_sample ? 1 : 0;
    t.temperature = s->do_sample ? s->temperature : 1.f;
    t.top_k = s->top_k; t.top_p = s->top_p; t.penalty = s->repetition_penalty;
    t.min_new = s->min_new_tokens; t.n_eos = s->n_eos;
    for (int e = 0; e < s->n_eos; ++e) t.eos[e] = s->eos_ids[e];
    t.seed = s->seed;
    t.active = t.do_sample || t.penalty != 1.f || (t.min_new > 0 && t.n_eos > 0);
  }
  *out = t;
  return S2S_OK;
}

// The seen set of a slot that was reset is emptied on the stream of the slot's next launch (session_reset takes no stream).
static int seen_clear_if_reset(s2s_llama* m, int slot, cudaStream_t st) {
  if (!m->seen_stale[slot]) return S2S_OK;
  S2S_CHECK_CUDA(cudaMemsetAsync(m->seen + (size_t)slot * m->seen_words, 0, (size_t)m->seen_words * 4, st));
  m->seen_stale[slot] = 0;
  return S2S_OK;
}

// Repetition penalty: the n prompt ids (device) of a prefill join the slot's seen set, whatever its current settings, so
// that a penalty set later in the response still sees the whole prompt.
static int seen_add(s2s_llama* m, int slot, const int* ids_d, int n, cudaStream_t st) {
  S2S_CHECK(seen_clear_if_reset(m, slot, st));
  seen_set_kernel<<<(n + 255) / 256, 256, 0, st>>>(ids_d, n, m->seen + (size_t)slot * m->seen_words);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

// The token predicted from the logits row that follows a prefill of `slot`, at position pred_pos: argmax for a greedy slot,
// sampling.cuh's choice otherwise.  The slot's new-token count restarts here.
static int prefill_choose(s2s_llama* m, int slot, const float* row, int pred_pos, int32_t* out_d, cudaStream_t st) {
  SampSlot& s = m->samp[slot];
  s.base = pred_pos;
  if (!s.active) argmax_row_kernel<<<1, 1024, 0, st>>>(row, m->cfg.vocab, out_d);
  else sample_row_kernel<<<1, 1024, 0, st>>>(row, m->cfg.vocab, s, m->seen + (size_t)slot * m->seen_words, pred_pos, out_d);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

// RoPE / Qwen3 q/k norm + RoPE and the K/V append of one prefill segment: n rows of qkv at positions [past, past + n).
// q_norm == nullptr: Llama (rope_prefill_kernel), else Qwen3 (qknorm_rope_prefill_kernel).  prefill_layers and
// s2s_prefill_rope both launch through here.
static int prefill_rope_launch(void* qkv, int n, int heads, int kv_heads, int hd, int past, const float2* rope, const float* q_norm,
                               const float* k_norm, float eps, void* kc, void* vc, int dt, cudaStream_t st) {
  const bool bf = dt == S2S_BF16;
  if (q_norm) {
#define S2S_QKN(T, HD) qknorm_rope_prefill_kernel<T, HD><<<n, 256, 0, st>>>((T*)qkv, heads, kv_heads, past, rope, q_norm, k_norm, \
                                                                             eps, (T*)kc, (T*)vc)
    if (bf) { if (hd == 128) S2S_QKN(__nv_bfloat16, 128); else S2S_QKN(__nv_bfloat16, 64); }
    else { if (hd == 128) S2S_QKN(__half, 128); else S2S_QKN(__half, 64); }
#undef S2S_QKN
  } else {
    const int qd = heads * hd, kvd = kv_heads * hd;
    if (bf) rope_prefill_kernel<__nv_bfloat16><<<n, 256, 0, st>>>((__nv_bfloat16*)qkv, n, qd, kvd, hd, past, rope, (__nv_bfloat16*)kc,
                                                                  (__nv_bfloat16*)vc);
    else rope_prefill_kernel<__half><<<n, 256, 0, st>>>((__half*)qkv, n, qd, kvd, hd, past, rope, (__half*)kc, (__half*)vc);
  }
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

// One pass of all decoder layers over R = sum of the segments' rows, already embedded in m->x.  A segment is the new rows of
// one session (rows [off, off + n) of the buffers, positions [past, past + n) of its KV slot): the projections and the MLP
// run over all R rows at once -- ONE pass over the weights for every session of a batched prefill -- while RoPE / cache
// append and the causal attention run per segment against that session's cache.
struct PrefillSeg { int slot, off, n, past; };

static int prefill_layers(s2s_llama* m, const PrefillSeg* segs, int nseg, int R, cudaStream_t st) {
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, hd = c.head_dim, qd = c.heads * hd, kvd = c.kv_heads * hd, dt = c.compute_dtype;
  const int ldq = qd + 2 * kvd;
  const size_t esz = 2;
  for (int i = 0; i < c.layers; ++i) {
    const LlamaDecLayer& L = m->layers_h[i];
    S2S_CHECK(norm_rows_launch(m->x, L.norm1, nullptr, c.rms_eps, R, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = lgemm(m, m->xn, d, L.w_qkv, R, ldq, d);
      p.out_h = m->qkv; p.ldo_h = ldq;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    for (int sgi = 0; sgi < nseg; ++sgi) {
      const PrefillSeg& sg = segs[sgi];
      char* kc = reinterpret_cast<char*>(m->kv) + ((size_t)sg.slot * m->kv_slot_stride + (size_t)i * m->kv_layer_stride) * esz;
      char* vc = kc + (size_t)m->kv_which_stride * esz;
      char* qrow = reinterpret_cast<char*>(m->qkv) + (size_t)sg.off * ldq * esz;
      const int n = sg.n, past = sg.past;
      S2S_CHECK(prefill_rope_launch(qrow, n, c.heads, c.kv_heads, hd, past, m->rope, c.qk_norm ? L.q_norm : nullptr,
                                    c.qk_norm ? L.k_norm : nullptr, c.rms_eps, kc, vc, dt, st));
      S2S_CHECK(attention_tc_launch(m->ctx, qrow, kc, vc, reinterpret_cast<char*>(m->attn) + (size_t)sg.off * qd * esz, 1, n, past + n,
                                     c.heads, c.kv_heads, hd, ldq, kvd, kvd, qd, 1.0f / sqrtf((float)hd), 1, dt, m->vt, m->vt_elems, st));
    }
    {
      GemmProblem p = lgemm(m, m->attn, qd, L.w_o, R, d, qd);
      p.out_f = m->x; p.ldo_f = d; p.resid = m->x; p.ld_resid = d; p.resid_mode = 1;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    S2S_CHECK(norm_rows_launch(m->x, L.norm2, nullptr, c.rms_eps, R, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = lgemm(m, m->xn, d, L.w_gu, R, 2 * f, d);
      p.act = 2; p.out_h = m->hbuf; p.ldo_h = f;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    {
      GemmProblem p = lgemm(m, m->hbuf, f, L.w_down, R, d, f);
      p.out_f = m->x; p.ldo_f = d; p.resid = m->x; p.ld_resid = d; p.resid_mode = 1;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
  }
  return S2S_OK;
}

int llama_prefill_rows(s2s_llama* m, int slot, int n, float* logits_out_d, int32_t* next_id_d, float* hidden_out_d,
                       cudaStream_t st) {
  const auto& c = m->cfg;
  S2S_REQUIRE(n >= 1 && n <= c.max_prefill, "llama prefill: n=%d outside [1,%d]", n, c.max_prefill);
  const int past = m->len[slot];
  S2S_REQUIRE(past + n <= c.max_positions, "llama prefill: %d + %d tokens exceed max_positions %d", past, n, c.max_positions);
  const int d = c.d_model, dt = c.compute_dtype;
  const PrefillSeg seg{slot, 0, n, past};
  S2S_CHECK(prefill_layers(m, &seg, 1, n, st));
  if (hidden_out_d)
    S2S_CHECK_CUDA(cudaMemcpyAsync(hidden_out_d, m->x + (size_t)(n - 1) * d, (size_t)d * 4, cudaMemcpyDeviceToDevice, st));
  S2S_CHECK(norm_rows_launch(m->x, m->norm_f, nullptr, c.rms_eps, n, d, m->xn, nullptr, dt, st));
  if (logits_out_d) {
    GemmProblem p = lgemm(m, m->xn, d, m->lm_head_t, n, c.vocab, d);
    p.out_f = logits_out_d; p.ldo_f = c.vocab;
    S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
  }
  if (next_id_d) {
    const float* last = nullptr;
    if (logits_out_d) {
      last = logits_out_d + (size_t)(n - 1) * c.vocab;
    } else {
      GemmProblem p = lgemm(m, reinterpret_cast<char*>(m->xn) + (size_t)(n - 1) * d * 2, d, m->lm_head_t, 1, c.vocab, d);
      p.out_f = m->last_logits; p.ldo_f = c.vocab;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
      last = m->last_logits;
    }
    S2S_CHECK(prefill_choose(m, slot, last, past + n, next_id_d, st));
  }
  m->len[slot] = past + n;
  return S2S_OK;
}

// last row of every segment -> consecutive 16-bit rows (input of the one lm_head GEMM of a batched prefill)
template <typename T>
__global__ void gather_last_rows_kernel(const T* __restrict__ xn, const int* __restrict__ last_row, int d, T* __restrict__ out) {
  const T* src = xn + (long long)last_row[blockIdx.x] * d;
  T* dst = out + (long long)blockIdx.x * d;
  for (int i = threadIdx.x; i < d; i += blockDim.x) dst[i] = src[i];
}

int llama_prefill_batch(s2s_llama* m, const int32_t* slots_h, int B, const int32_t* n_h, int32_t* next_ids_d, cudaStream_t st) {
  const auto& c = m->cfg;
  PrefillSeg segs[MAX_DEC_B];
  int last_h[MAX_DEC_B], R = 0;
  for (int b = 0; b < B; ++b) {
    const int s = slots_h[b];
    S2S_REQUIRE(m->len[s] + n_h[b] <= c.max_positions, "llama prefill_batch: slot %d: %d + %d tokens exceed max_positions %d", s, m->len[s],
                n_h[b], c.max_positions);
    segs[b] = PrefillSeg{s, R, n_h[b], m->len[s]};
    R += n_h[b];
    last_h[b] = R - 1;
  }
  const int d = c.d_model, dt = c.compute_dtype;
  S2S_REQUIRE((size_t)c.max_prefill * c.heads * c.head_dim >= (size_t)B * d, "llama prefill_batch: scratch too small for %d sessions", B);
  S2S_CHECK(prefill_layers(m, segs, B, R, st));
  S2S_CHECK(norm_rows_launch(m->x, m->norm_f, nullptr, c.rms_eps, R, d, m->xn, nullptr, dt, st));
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->slot_d, last_h, (size_t)B * 4, cudaMemcpyHostToDevice, st));   // slot_d: free outside a decode launch
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));                                                        // last_h lives on this stack
  if (dt == S2S_BF16) gather_last_rows_kernel<__nv_bfloat16><<<B, 256, 0, st>>>((const __nv_bfloat16*)m->xn, m->slot_d, d, (__nv_bfloat16*)m->attn);
  else gather_last_rows_kernel<__half><<<B, 256, 0, st>>>((const __half*)m->xn, m->slot_d, d, (__half*)m->attn);
  S2S_LAUNCH_CHECK();
  {
    GemmProblem p = lgemm(m, m->attn, d, m->lm_head_t, B, c.vocab, d);
    p.out_f = m->batch_logits; p.ldo_f = c.vocab;
    S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
  }
  for (int b = 0; b < B; ++b) {
    S2S_CHECK(seen_add(m, slots_h[b], m->ids_d + segs[b].off, n_h[b], st));
    S2S_CHECK(prefill_choose(m, slots_h[b], m->batch_logits + (size_t)b * c.vocab, segs[b].past + n_h[b], next_ids_d + b, st));
  }
  for (int b = 0; b < B; ++b) m->len[slots_h[b]] += n_h[b];
  return S2S_OK;
}

extern "C" {

// source != nullptr: the new object reads source's weights (s2s_llama_create_shared) and comes back finalized
static int create(s2s_ctx* ctx, const s2s_llama_config* cfg, s2s_llama* source, s2s_llama** out) {
  S2S_REQUIRE(ctx && cfg && out, "llama_create: null argument");
  S2S_REQUIRE(cfg->head_dim == 64 || cfg->head_dim == 128, "llama: head_dim must be 64 or 128");
  S2S_REQUIRE(cfg->heads % cfg->kv_heads == 0, "llama: heads %% kv_heads != 0");
  S2S_REQUIRE(cfg->d_model % 64 == 0 && cfg->ffn % 64 == 0 && cfg->vocab % 64 == 0, "llama: d_model, ffn, vocab must be multiples of 64");
  S2S_REQUIRE(cfg->compute_dtype == S2S_BF16 || cfg->compute_dtype == S2S_F16, "llama: compute_dtype must be bf16/f16");
  S2S_REQUIRE(cfg->max_sessions >= 1 && cfg->max_positions >= 64 && cfg->max_prefill >= 1, "llama: bad capacity");
  S2S_REQUIRE(cfg->layers >= 1 && cfg->layers <= 64, "llama: layers in [1,64]");
  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  s2s_llama* m = new s2s_llama();
  m->ctx = ctx;
  m->cfg = *cfg;
  m->weight_format = source ? source->weight_format : cfg->compute_dtype;
  if (source) m->arena.borrow(source->arena);
  int r = build(m);
  if (r == S2S_OK && source) {
    r = alloc_matrices(m);
    m->lm_head_bound = true;
    m->finalized = r == S2S_OK;
  }
  if (r != S2S_OK) { s2s_llama_destroy(m); return r; }
  const char* dbg = getenv("S2S_DEBUG_PHASES");
  m->debug_phases = (dbg && dbg[0] == '1') ? 1 : 0;
  *out = m;
  return S2S_OK;
}

int s2s_llama_create(s2s_ctx* ctx, const s2s_llama_config* cfg, s2s_llama** out) { return create(ctx, cfg, nullptr, out); }

int s2s_llama_create_shared(s2s_ctx* ctx, s2s_llama* source, const s2s_llama_config* cfg, s2s_llama** out) {
  const char* who = "llama create_shared";
  S2S_REQUIRE(ctx && source && cfg && out, "%s: null argument", who);
  S2S_REQUIRE(source->finalized, "%s: the source is not finalized", who);
  S2S_REQUIRE(source->ctx->device == ctx->device, "%s: the source is on device %d, the context on device %d", who,
              source->ctx->device, ctx->device);
  const s2s_llama_config& s = source->cfg;
  S2S_REQUIRE_SAME(*cfg, s, d_model, who);
  S2S_REQUIRE_SAME(*cfg, s, layers, who);
  S2S_REQUIRE_SAME(*cfg, s, heads, who);
  S2S_REQUIRE_SAME(*cfg, s, kv_heads, who);
  S2S_REQUIRE_SAME(*cfg, s, head_dim, who);
  S2S_REQUIRE_SAME(*cfg, s, ffn, who);
  S2S_REQUIRE_SAME(*cfg, s, vocab, who);
  S2S_REQUIRE_SAME(*cfg, s, rope_theta, who);
  S2S_REQUIRE_SAME(*cfg, s, rms_eps, who);
  S2S_REQUIRE_SAME(*cfg, s, compute_dtype, who);
  S2S_REQUIRE_SAME(*cfg, s, qk_norm, who);
  S2S_REQUIRE_SAME(*cfg, s, n_tables, who);
  return create(ctx, cfg, source, out);
}

int s2s_llama_destroy(s2s_llama* m) {
  if (!m) return S2S_OK;
  delete m;
  return S2S_OK;
}

int s2s_llama_bind_tensor(s2s_llama* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                          int32_t dtype) {
  S2S_REQUIRE(m && name && data_h && shape, "llama bind_tensor: null argument");
  S2S_CHECK(m->arena.check_writable("llama bind_tensor"));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(alloc_matrices(m));
  S2S_CHECK(m->arena.bind("llama", name, data_h, shape, ndim, dtype, m->cfg.compute_dtype));
  if (strncmp(name, "lm_head.", 8) == 0) m->lm_head_bound = true;
  return S2S_OK;
}

int s2s_llama_init_random(s2s_llama* m, uint64_t seed) {
  S2S_REQUIRE(m, "llama init_random: null model");
  S2S_CHECK(m->arena.check_writable("llama init_random"));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(alloc_matrices(m));
  S2S_CHECK(m->arena.init_random(seed, m->cfg.compute_dtype));
  m->lm_head_bound = true;
  return S2S_OK;
}

int s2s_llama_set_weight_format(s2s_llama* m, int32_t format) {
  S2S_REQUIRE(m, "llama set_weight_format: null model");
  S2S_CHECK(m->arena.check_writable("llama set_weight_format"));
  S2S_REQUIRE(!m->matrices, "llama set_weight_format: the weight format is fixed by the first bind, init_random or finalize");
  if (format != m->cfg.compute_dtype) {
    if (format != S2S_FP8_E4M3 || m->cfg.compute_dtype != S2S_BF16 || m->n_tables != 1) {
      // the dequantised weights are exact in bf16, not in f16; multi-table models (TTS code predictor) stay 16-bit
      s2s_set_error("llama set_weight_format: format %d needs a single-table model with bf16 compute, or must equal compute_dtype", format);
      return S2S_ERR_UNSUPPORTED;
    }
  }
  m->weight_format = format;
  return S2S_OK;
}

int32_t s2s_llama_weight_format(s2s_llama* m) { return m ? m->weight_format : S2S_ERR_INVALID; }

int s2s_llama_finalize(s2s_llama* m) {
  S2S_REQUIRE(m, "llama finalize: null model");
  S2S_CHECK(m->arena.check_writable("llama finalize"));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK(alloc_matrices(m));
  if (m->n_tables == 1 && !m->lm_head_bound && m->arena.find("model.embed_tokens.weight")->bound) {
    // tied embeddings (tie_word_embeddings=True): lm_head is tiled (or quantised) straight from embed_tokens
    S2S_CHECK(tile_rows_launch(m->embed, m->cfg.vocab, m->cfg.d_model, m->lm_head_t, m->cfg.vocab, 0, 1,
                               m->weight_format == S2S_FP8_E4M3, 0));
    m->arena.find("lm_head.weight")->bound = true;
  }
  S2S_CHECK(m->arena.check_all_bound("llama"));
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  m->arena.release_staging();
  m->finalized = true;
  return S2S_OK;
}

int s2s_llama_device_bytes(s2s_llama* m, int64_t* weights, int64_t* total) {
  S2S_REQUIRE(m && weights && total, "llama device_bytes: null argument");
  *weights = (int64_t)m->arena.weight_bytes();
  *total = (int64_t)m->arena.bytes();
  return S2S_OK;
}

int s2s_llama_session_reset(s2s_llama* m, int32_t slot) {
  S2S_REQUIRE(m && slot >= 0 && slot < m->cfg.max_sessions, "llama session_reset: bad slot %d", slot);
  m->len[slot] = 0;
  m->seen_stale[slot] = 1;
  return S2S_OK;
}

int s2s_llama_set_sampling(s2s_llama* m, int32_t slot, const s2s_sampling* s) {
  S2S_REQUIRE(m && slot >= 0 && slot < m->cfg.max_sessions, "llama set_sampling: bad slot %d", slot);
  SampSlot t;
  S2S_CHECK(samp_from_abi(s, m->cfg.vocab, "llama set_sampling", &t));
  t.base = m->samp[slot].base;
  m->samp[slot] = t;
  return S2S_OK;
}

int s2s_llama_prefill(s2s_llama* m, int32_t slot, const int32_t* ids_h, int32_t n, float* logits_out_d,
                      int32_t* next_id_d, void* stream) {
  S2S_REQUIRE(m && m->finalized && ids_h, "llama prefill: null argument / not finalized");
  const auto& c = m->cfg;
  S2S_REQUIRE(slot >= 0 && slot < c.max_sessions, "llama prefill: bad slot %d", slot);
  S2S_REQUIRE(n >= 1 && n <= c.max_prefill, "llama prefill: n=%d outside [1,%d]", n, c.max_prefill);
  for (int i = 0; i < n; ++i) S2S_REQUIRE(ids_h[i] >= 0 && ids_h[i] < c.vocab, "llama prefill: token %d out of range", ids_h[i]);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->ids_d, ids_h, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));  // ids_h may be a temporary of the caller
  if (c.compute_dtype == S2S_BF16) embed_gather_kernel<__nv_bfloat16><<<n, 256, 0, st>>>(m->ids_d, (const __nv_bfloat16*)m->embed, m->x, c.d_model);
  else embed_gather_kernel<__half><<<n, 256, 0, st>>>(m->ids_d, (const __half*)m->embed, m->x, c.d_model);
  S2S_LAUNCH_CHECK();
  S2S_CHECK(seen_add(m, slot, m->ids_d, n, st));
  return llama_prefill_rows(m, slot, n, logits_out_d, next_id_d, nullptr, st);
}

int s2s_llama_prefill_batch(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* ids_h, const int32_t* n_h,
                            int32_t* next_ids_d, void* stream) {
  S2S_REQUIRE(m && m->finalized && slots_h && ids_h && n_h && next_ids_d, "llama prefill_batch: null argument / not finalized");
  const auto& c = m->cfg;
  S2S_REQUIRE(B >= 1 && B <= MAX_DEC_B, "llama prefill_batch: B=%d outside [1,%d]", B, MAX_DEC_B);
  S2S_REQUIRE(m->n_tables == 1, "llama prefill_batch: multi-table models are driven by the TTS entry points");
  int R = 0;
  for (int b = 0; b < B; ++b) {
    S2S_REQUIRE(slots_h[b] >= 0 && slots_h[b] < c.max_sessions, "llama prefill_batch: bad slot %d", slots_h[b]);
    for (int b2 = 0; b2 < b; ++b2) S2S_REQUIRE(slots_h[b2] != slots_h[b], "llama prefill_batch: slot %d listed twice", slots_h[b]);
    S2S_REQUIRE(n_h[b] >= 1, "llama prefill_batch: session %d has no rows", b);
    R += n_h[b];
  }
  S2S_REQUIRE(R <= c.max_prefill, "llama prefill_batch: %d rows in total exceed max_prefill %d", R, c.max_prefill);
  for (int i = 0; i < R; ++i) S2S_REQUIRE(ids_h[i] >= 0 && ids_h[i] < c.vocab, "llama prefill_batch: token %d out of range", ids_h[i]);
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->ids_d, ids_h, (size_t)R * 4, cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));  // ids_h may be a temporary of the caller
  if (c.compute_dtype == S2S_BF16) embed_gather_kernel<__nv_bfloat16><<<R, 256, 0, st>>>(m->ids_d, (const __nv_bfloat16*)m->embed, m->x, c.d_model);
  else embed_gather_kernel<__half><<<R, 256, 0, st>>>(m->ids_d, (const __half*)m->embed, m->x, c.d_model);
  S2S_LAUNCH_CHECK();
  return llama_prefill_batch(m, slots_h, B, n_h, next_ids_d, st);
}

int s2s_llama_decode(s2s_llama* m, const int32_t* slots_h, int32_t B, const int32_t* first_ids_d, int32_t n_steps,
                     int32_t eos_id, int32_t* ids_out_d, int32_t* len_out_d, const int32_t* forced_d,
                     float* logits_out_d, void* stream) {
  S2S_REQUIRE(m && m->finalized && slots_h && first_ids_d && ids_out_d && len_out_d, "llama decode: null argument");
  const auto& c = m->cfg;
  const int max_b = llama_max_decode_batch_of(m);
  S2S_REQUIRE(B >= 1 && B <= max_b, "llama decode: B=%d outside [1,%d] for this geometry", B, max_b);
  S2S_REQUIRE(n_steps >= 1, "llama decode: n_steps must be >= 1");
  S2S_REQUIRE(m->n_tables == 1, "llama decode: multi-table models are driven by the TTS entry points");
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  int pos_h[MAX_DEC_B], max_len = 0;
  for (int b = 0; b < B; ++b) {
    const int s = slots_h[b];
    S2S_REQUIRE(s >= 0 && s < c.max_sessions, "llama decode: bad slot %d", s);
    for (int b2 = 0; b2 < b; ++b2) S2S_REQUIRE(slots_h[b2] != s, "llama decode: slot %d listed twice", s);
    S2S_REQUIRE(m->len[s] + n_steps <= c.max_positions, "llama decode: slot %d would exceed max_positions", s);
    pos_h[b] = m->len[s];
    max_len = pos_h[b] + 1 > max_len ? pos_h[b] + 1 : max_len;
  }
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->slot_d, slots_h, B * 4, cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaMemcpyAsync(m->pos_d, pos_h, B * 4, cudaMemcpyHostToDevice, st));
  SampSlot samp_h[MAX_DEC_B];
  bool any_samp = false;
  for (int b = 0; b < B; ++b) {
    samp_h[b] = m->samp[slots_h[b]];
    any_samp |= samp_h[b].active != 0;
    S2S_CHECK(seen_clear_if_reset(m, slots_h[b], st));
  }
  if (any_samp) S2S_CHECK_CUDA(cudaMemcpyAsync(m->samp_d, samp_h, B * sizeof(SampSlot), cudaMemcpyHostToDevice, st));
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));
  LlamaDecParams p{};
  llama_fill_dec_params(m, p);
  p.B = B; p.slot = m->slot_d; p.pos = m->pos_d; p.max_len = max_len;
  p.first_ids = first_ids_d; p.n_steps = n_steps; p.eos = eos_id; p.out_ids = ids_out_d; p.out_len = len_out_d;
  p.forced = forced_d; p.logits_out = logits_out_d; p.samp = any_samp ? m->samp_d : nullptr;
  S2S_CHECK(llama_decode_launch(m->ctx, p, c.compute_dtype, m->weight_format, m->debug_phases, st));
  for (int b = 0; b < B; ++b) m->len[slots_h[b]] += n_steps;
  return S2S_OK;
}

int32_t s2s_llama_max_decode_batch(s2s_llama* m) { return m ? llama_max_decode_batch_of(m) : 0; }

int s2s_llama_set_trace(s2s_llama* m, uint64_t* trace_d, int32_t capacity) {
  S2S_REQUIRE(m, "llama set_trace: null model");
  m->trace = reinterpret_cast<unsigned long long*>(trace_d);
  m->trace_cap = trace_d ? capacity : 0;
  return S2S_OK;
}

int s2s_llama_generate(s2s_llama* m, int32_t slot, const int32_t* prompt_h, int32_t n_prompt, int32_t n_steps,
                       int32_t eos_id, int32_t* ids_out_h, int32_t* len_out_h, void* stream) {
  S2S_REQUIRE(m && prompt_h && ids_out_h && len_out_h, "llama generate: null argument");
  S2S_REQUIRE(n_steps >= 1 && n_steps <= m->cfg.max_positions, "llama generate: bad n_steps");
  cudaStream_t st = (cudaStream_t)stream;
  S2S_CHECK(s2s_llama_session_reset(m, slot));
  // chunked prefill
  for (int o = 0; o < n_prompt; o += m->cfg.max_prefill) {
    const int n = (n_prompt - o) < m->cfg.max_prefill ? (n_prompt - o) : m->cfg.max_prefill;
    const bool last = o + n >= n_prompt;
    S2S_CHECK(s2s_llama_prefill(m, slot, prompt_h + o, n, nullptr, last ? m->next_id : nullptr, stream));
  }
  // ids_out[0] = the token chosen from the prompt's last position; the decode kernel then feeds it and produces the rest
  int first = 0;
  S2S_CHECK_CUDA(cudaMemcpyAsync(&first, m->next_id, 4, cudaMemcpyDeviceToHost, st));
  int n_dec = 0;
  if (n_steps > 1) {
    S2S_CHECK(s2s_llama_decode(m, &slot, 1, m->next_id, n_steps - 1, eos_id, m->out_ids, m->out_len, nullptr, nullptr, stream));
    S2S_CHECK_CUDA(cudaMemcpyAsync(ids_out_h + 1, m->out_ids, (size_t)(n_steps - 1) * 4, cudaMemcpyDeviceToHost, st));
    S2S_CHECK_CUDA(cudaMemcpyAsync(&n_dec, m->out_len, 4, cudaMemcpyDeviceToHost, st));
  }
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));
  ids_out_h[0] = first;
  if (first == eos_id) {
    *len_out_h = 1;
    for (int i = 1; i < n_steps; ++i) ids_out_h[i] = eos_id;
  } else {
    *len_out_h = 1 + n_dec;
  }
  return S2S_OK;
}

int s2s_prefill_rope(s2s_ctx* ctx, void* qkv, int32_t n, int32_t heads, int32_t kv_heads, int32_t hd, int32_t past,
                     const float* rope, int32_t max_pos, const float* q_norm, const float* k_norm, float eps, void* kcache,
                     void* vcache, int32_t dtype, void* stream) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  S2S_REQUIRE(ctx && qkv && rope && kcache && vcache, "s2s_prefill_rope: null argument");
  S2S_REQUIRE(hd == 64 || hd == 128, "s2s_prefill_rope: hd %d (64 or 128)", hd);
  S2S_REQUIRE(heads >= 1 && kv_heads >= 1 && heads % kv_heads == 0, "s2s_prefill_rope: heads %d / kv_heads %d", heads, kv_heads);
  S2S_REQUIRE(n >= 1 && past >= 0 && (int64_t)past + n <= max_pos, "s2s_prefill_rope: rows [%d, %d + %d) outside [0, max_pos %d)",
              past, past, n, max_pos);
  S2S_REQUIRE(!q_norm == !k_norm, "s2s_prefill_rope: q_norm and k_norm go together (both: Qwen3, neither: Llama)");
  S2S_REQUIRE(dtype == S2S_F16 || dtype == S2S_BF16, "s2s_prefill_rope: dtype %d", dtype);
  S2S_REQUIRE(al(qkv) && al(rope) && al(q_norm) && al(k_norm) && al(kcache) && al(vcache), "s2s_prefill_rope: pointers must be 16-byte aligned");
  return prefill_rope_launch(qkv, n, heads, kv_heads, hd, past, reinterpret_cast<const float2*>(rope), q_norm, k_norm, eps, kcache,
                             vcache, dtype, (cudaStream_t)stream);
}

int s2s_argmax_row(s2s_ctx* ctx, const float* logits_d, int32_t n, int32_t* out_d, void* stream) {
  S2S_REQUIRE(ctx && logits_d && out_d && n >= 1, "s2s_argmax_row: null argument or n %d < 1", n);
  argmax_row_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits_d, n, out_d);   // as prefill_choose launches it
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

}  // extern "C"
