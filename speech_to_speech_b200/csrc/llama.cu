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
#include <unordered_map>
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

__global__ void argmax_row_kernel(const float* __restrict__ logits, int n, int* __restrict__ out) {
  __shared__ float sv[32];
  __shared__ int si[32];
  float bv = -INFINITY; int bi = 0x7fffffff;
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

inline uint16_t f2h(float f) { __half h = __float2half_rn(f); uint16_t u; memcpy(&u, &h, 2); return u; }
inline uint16_t f2bf(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fc0;
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float src_f32(const void* data, int64_t i, int dtype) {
  if (dtype == S2S_F32) return reinterpret_cast<const float*>(data)[i];
  uint16_t u = reinterpret_cast<const uint16_t*>(data)[i];
  if (dtype == S2S_BF16) { uint32_t w = (uint32_t)u << 16; float f; memcpy(&f, &w, 4); return f; }
  __half h; memcpy(&h, &u, 2); return __half2float(h);
}

}  // namespace

namespace {

constexpr int MAX_DEC_B = LLAMA_MAX_DEC_B;

template <typename P> int lalloc(s2s_llama* m, P** out, size_t bytes, bool zero = true) {
  void* p = nullptr;
  S2S_CHECK_CUDA(cudaMalloc(&p, bytes ? bytes : 16));
  if (zero) S2S_CHECK_CUDA(cudaMemset(p, 0, bytes ? bytes : 16));
  m->allocs.push_back(p);
  *out = reinterpret_cast<P*>(p);
  return S2S_OK;
}

void lslot(s2s_llama* m, const std::string& name, void* dst, bool half, int64_t rows, int64_t cols, float rnd_scale,
           float rnd_offset = 0.f, int kind = L_PLAIN, int hd = 0, int parity = 0) {
  LSlot s;
  s.dst = dst; s.half = half; s.rows = rows; s.cols = cols; s.kind = kind; s.hd = hd; s.parity = parity;
  s.rnd_scale = rnd_scale; s.rnd_offset = rnd_offset;
  m->slots[name] = s;
}

int build(s2s_llama* m) {
  const auto& c = m->cfg;
  const int d = c.d_model, f = c.ffn, hd = c.head_dim, qd = c.heads * hd, kvd = c.kv_heads * hd;
  const int esz = 2;
  auto off = [&](void* base, int64_t elems) { return reinterpret_cast<char*>(base) + elems * esz; };
  m->n_tables = c.n_tables > 1 ? c.n_tables : 1;
  m->embed_table_elems = (size_t)c.vocab * d;
  m->head_table_elems = (size_t)c.vocab * d;
  S2S_CHECK(lalloc(m, &m->embed, m->n_tables * m->embed_table_elems * esz));
  S2S_CHECK(lalloc(m, &m->lm_head, m->n_tables * m->head_table_elems * esz));
  S2S_CHECK(lalloc(m, &m->norm_f, d * 4));
  if (m->n_tables == 1) {
    lslot(m, "model.embed_tokens.weight", m->embed, true, c.vocab, d, 0.02f);
    lslot(m, "lm_head.weight", m->lm_head, true, c.vocab, d, 0.02f);
  } else {  // code predictor: one table / head per codebook (Qwen3OmniMoeTalkerCodePredictorModel.codec_embedding, .lm_head)
    for (int t = 0; t < m->n_tables; ++t) {
      lslot(m, "model.embed_tokens." + std::to_string(t) + ".weight", off(m->embed, (int64_t)t * m->embed_table_elems), true, c.vocab, d, 0.02f);
      lslot(m, "lm_head." + std::to_string(t) + ".weight", off(m->lm_head, (int64_t)t * m->head_table_elems), true, c.vocab, d, 0.02f);
    }
  }
  lslot(m, "model.norm.weight", m->norm_f, false, d, 1, 0.1f, 1.0f);
  m->layers_h.resize(c.layers);
  const float sd = 1.0f / sqrtf((float)d);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = "model.layers." + std::to_string(i) + ".";
    void *w_qkv, *w_o, *w_gu, *w_down;
    float *n1, *n2, *qn = nullptr, *kn = nullptr;
    S2S_CHECK(lalloc(m, &w_qkv, (size_t)(qd + 2 * kvd) * d * esz));
    S2S_CHECK(lalloc(m, &w_o, (size_t)d * qd * esz));
    S2S_CHECK(lalloc(m, &w_gu, (size_t)2 * f * d * esz));
    S2S_CHECK(lalloc(m, &w_down, (size_t)d * f * esz));
    S2S_CHECK(lalloc(m, &n1, d * 4));
    S2S_CHECK(lalloc(m, &n2, d * 4));
    lslot(m, p + "self_attn.q_proj.weight", w_qkv, true, qd, d, 2.0f * sd, 0.f, L_ROPE_PERM, hd);
    lslot(m, p + "self_attn.k_proj.weight", off(w_qkv, (int64_t)qd * d), true, kvd, d, 2.0f * sd, 0.f, L_ROPE_PERM, hd);
    lslot(m, p + "self_attn.v_proj.weight", off(w_qkv, (int64_t)(qd + kvd) * d), true, kvd, d, 0.8f * sd);
    lslot(m, p + "self_attn.o_proj.weight", w_o, true, d, qd, 1.0f * sd);
    lslot(m, p + "mlp.gate_proj.weight", w_gu, true, f, d, 1.0f * sd, 0.f, L_INTERLEAVE, 0, 0);
    lslot(m, p + "mlp.up_proj.weight", w_gu, true, f, d, 1.0f * sd, 0.f, L_INTERLEAVE, 0, 1);
    lslot(m, p + "mlp.down_proj.weight", w_down, true, d, f, 0.7f / sqrtf((float)f));
    lslot(m, p + "input_layernorm.weight", n1, false, d, 1, 0.1f, 1.0f);
    lslot(m, p + "post_attention_layernorm.weight", n2, false, d, 1, 0.1f, 1.0f);
    if (c.qk_norm) {  // Qwen3Attention.q_norm / k_norm: RMSNorm(head_dim), permuted like the q/k rows
      S2S_CHECK(lalloc(m, &qn, hd * 4));
      S2S_CHECK(lalloc(m, &kn, hd * 4));
      lslot(m, p + "self_attn.q_norm.weight", qn, false, hd, 1, 0.1f, 1.0f, L_ROPE_PERM, hd);
      lslot(m, p + "self_attn.k_norm.weight", kn, false, hd, 1, 0.1f, 1.0f, L_ROPE_PERM, hd);
    }
    LlamaDecLayer& L = m->layers_h[i];
    L.w_qkv = w_qkv; L.w_o = w_o; L.w_gu = w_gu; L.w_down = w_down; L.norm1 = n1; L.norm2 = n2; L.q_norm = qn; L.k_norm = kn;
  }
  S2S_CHECK(lalloc(m, &m->layers_d, sizeof(LlamaDecLayer) * c.layers));
  S2S_CHECK_CUDA(cudaMemcpy(m->layers_d, m->layers_h.data(), sizeof(LlamaDecLayer) * c.layers, cudaMemcpyHostToDevice));

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
    S2S_CHECK(lalloc(m, &m->rope, tab.size() * sizeof(float2)));
    S2S_CHECK_CUDA(cudaMemcpy(m->rope, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  // KV cache [slot][layer][2][max_pos][kvd]
  m->kv_which_stride = (long long)c.max_positions * kvd;
  m->kv_layer_stride = 2 * m->kv_which_stride;
  m->kv_slot_stride = (long long)c.layers * m->kv_layer_stride;
  S2S_CHECK(lalloc(m, &m->kv, (size_t)c.max_sessions * m->kv_slot_stride * esz));
  m->len.assign(c.max_sessions, 0);
  // prefill workspace
  const int P = c.max_prefill;
  S2S_CHECK(lalloc(m, &m->ids_d, (size_t)P * 4));
  S2S_CHECK(lalloc(m, &m->x, (size_t)P * d * 4));
  S2S_CHECK(lalloc(m, &m->xn, (size_t)P * d * esz));
  S2S_CHECK(lalloc(m, &m->qkv, (size_t)P * (qd + 2 * kvd) * esz));
  S2S_CHECK(lalloc(m, &m->attn, (size_t)P * qd * esz));
  S2S_CHECK(lalloc(m, &m->hbuf, (size_t)P * f * esz));
  S2S_CHECK(lalloc(m, &m->last_logits, (size_t)c.vocab * 4));
  S2S_CHECK(lalloc(m, &m->batch_logits, (size_t)MAX_DEC_B * c.vocab * 4));
  m->vt_elems = attention_tc_scratch_elems(1, c.max_positions, c.kv_heads, hd);
  S2S_CHECK(lalloc(m, &m->vt, m->vt_elems * esz));
  // decode state
  m->s_max = (c.max_positions + 63) / 64;
  const int grid = m->ctx->num_sms;
  S2S_CHECK(lalloc(m, &m->dx, (size_t)MAX_DEC_B * d * 4));
  S2S_CHECK(lalloc(m, &m->dq, (size_t)MAX_DEC_B * qd * 4));
  S2S_CHECK(lalloc(m, &m->dh, (size_t)MAX_DEC_B * f * 4));
  S2S_CHECK(lalloc(m, &m->part, (size_t)MAX_DEC_B * c.heads * m->s_max * (hd + 4) * 4));
  S2S_CHECK(lalloc(m, &m->attn16, (size_t)MAX_DEC_B * qd * 2));
  S2S_CHECK(lalloc(m, &m->attn_cnt, (size_t)MAX_DEC_B * c.heads * 4));
  S2S_CHECK(lalloc(m, &m->slot_d, MAX_DEC_B * 4));
  S2S_CHECK(lalloc(m, &m->pos_d, MAX_DEC_B * 4));
  S2S_CHECK(lalloc(m, &m->done, MAX_DEC_B * 4));
  S2S_CHECK(lalloc(m, &m->n_done, 16));
  S2S_CHECK(lalloc(m, &m->cand_val, (size_t)MAX_DEC_B * grid * 4));
  S2S_CHECK(lalloc(m, &m->cand_idx, (size_t)MAX_DEC_B * grid * 4));
  S2S_CHECK(lalloc(m, &m->out_ids, (size_t)MAX_DEC_B * c.max_positions * 4));
  S2S_CHECK(lalloc(m, &m->out_len, MAX_DEC_B * 4));
  S2S_CHECK(lalloc(m, &m->next_id, 16));
  S2S_CHECK(lalloc(m, &m->sync_counter, 16));
  S2S_CHECK(lalloc(m, &m->kraw, (size_t)MAX_DEC_B * kvd * 4));
  S2S_CHECK(lalloc(m, &m->qn, (size_t)MAX_DEC_B * qd * 4));
  return S2S_OK;
}

GemmProblem lgemm(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t M, int N, int K) {
  GemmProblem p{};
  p.a = a; p.a_row_stride = lda; p.a_batch_stride = lda * M; p.w = w; p.ldw = ldw;
  p.M = (int32_t)M; p.N = N; p.K = K; p.batch = 1;
  return p;
}

}  // namespace

int llama_max_decode_batch_of(const s2s_llama* m) {
  return std::min(MAX_DEC_B, llama_decode_max_batch(m->cfg.d_model, m->cfg.ffn, m->cfg.heads * m->cfg.head_dim, dec_grid(m->ctx)));
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
  const bool bf = dt == S2S_BF16;
  const size_t esz = 2;
  for (int i = 0; i < c.layers; ++i) {
    const LlamaDecLayer& L = m->layers_h[i];
    S2S_CHECK(norm_rows_launch(m->x, L.norm1, nullptr, c.rms_eps, R, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = lgemm(m->xn, d, L.w_qkv, d, R, ldq, d);
      p.out_h = m->qkv; p.ldo_h = ldq;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    for (int sgi = 0; sgi < nseg; ++sgi) {
      const PrefillSeg& sg = segs[sgi];
      char* kc = reinterpret_cast<char*>(m->kv) + ((size_t)sg.slot * m->kv_slot_stride + (size_t)i * m->kv_layer_stride) * esz;
      char* vc = kc + (size_t)m->kv_which_stride * esz;
      char* qrow = reinterpret_cast<char*>(m->qkv) + (size_t)sg.off * ldq * esz;
      const int n = sg.n, past = sg.past;
      if (c.qk_norm) {
#define S2S_QKN(T, HD) qknorm_rope_prefill_kernel<T, HD><<<n, 256, 0, st>>>((T*)qrow, c.heads, c.kv_heads, past, m->rope, \
                                                                             L.q_norm, L.k_norm, c.rms_eps, (T*)kc, (T*)vc)
        if (bf) { if (hd == 128) S2S_QKN(__nv_bfloat16, 128); else S2S_QKN(__nv_bfloat16, 64); }
        else { if (hd == 128) S2S_QKN(__half, 128); else S2S_QKN(__half, 64); }
#undef S2S_QKN
      } else if (bf) {
        rope_prefill_kernel<__nv_bfloat16><<<n, 256, 0, st>>>((__nv_bfloat16*)qrow, n, qd, kvd, hd, past, m->rope,
                                                              (__nv_bfloat16*)kc, (__nv_bfloat16*)vc);
      } else {
        rope_prefill_kernel<__half><<<n, 256, 0, st>>>((__half*)qrow, n, qd, kvd, hd, past, m->rope, (__half*)kc, (__half*)vc);
      }
      S2S_LAUNCH_CHECK();
      S2S_CHECK(attention_tc_launch(m->ctx, qrow, kc, vc, reinterpret_cast<char*>(m->attn) + (size_t)sg.off * qd * esz, 1, n, past + n,
                                     c.heads, c.kv_heads, hd, ldq, kvd, kvd, qd, 1.0f / sqrtf((float)hd), 1, dt, m->vt, m->vt_elems, st));
    }
    {
      GemmProblem p = lgemm(m->attn, qd, L.w_o, qd, R, d, qd);
      p.out_f = m->x; p.ldo_f = d; p.resid = m->x; p.ld_resid = d; p.resid_mode = 1;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    S2S_CHECK(norm_rows_launch(m->x, L.norm2, nullptr, c.rms_eps, R, d, m->xn, nullptr, dt, st));
    {
      GemmProblem p = lgemm(m->xn, d, L.w_gu, d, R, 2 * f, d);
      p.act = 2; p.out_h = m->hbuf; p.ldo_h = f;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
    }
    {
      GemmProblem p = lgemm(m->hbuf, f, L.w_down, f, R, d, f);
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
    GemmProblem p = lgemm(m->xn, d, m->lm_head, d, n, c.vocab, d);
    p.out_f = logits_out_d; p.ldo_f = c.vocab;
    S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
  }
  if (next_id_d) {
    const float* last = nullptr;
    if (logits_out_d) {
      last = logits_out_d + (size_t)(n - 1) * c.vocab;
    } else {
      GemmProblem p = lgemm(reinterpret_cast<char*>(m->xn) + (size_t)(n - 1) * d * 2, d, m->lm_head, d, 1, c.vocab, d);
      p.out_f = m->last_logits; p.ldo_f = c.vocab;
      S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
      last = m->last_logits;
    }
    argmax_row_kernel<<<1, 1024, 0, st>>>(last, c.vocab, next_id_d);
    S2S_LAUNCH_CHECK();
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
    GemmProblem p = lgemm(m->attn, d, m->lm_head, d, B, c.vocab, d);
    p.out_f = m->batch_logits; p.ldo_f = c.vocab;
    S2S_CHECK(gemm_tc_launch(m->ctx, p, dt, st));
  }
  for (int b = 0; b < B; ++b) {
    argmax_row_kernel<<<1, 1024, 0, st>>>(m->batch_logits + (size_t)b * c.vocab, c.vocab, next_ids_d + b);
    S2S_LAUNCH_CHECK();
  }
  for (int b = 0; b < B; ++b) m->len[slots_h[b]] += n_h[b];
  return S2S_OK;
}

extern "C" {

int s2s_llama_create(s2s_ctx* ctx, const s2s_llama_config* cfg, s2s_llama** out) {
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
  int r = build(m);
  if (r != S2S_OK) { s2s_llama_destroy(m); return r; }
  const char* dbg = getenv("S2S_DEBUG_PHASES");
  m->debug_phases = (dbg && dbg[0] == '1') ? 1 : 0;
  *out = m;
  return S2S_OK;
}

int s2s_llama_destroy(s2s_llama* m) {
  if (!m) return S2S_OK;
  for (void* p : m->allocs) cudaFree(p);
  delete m;
  return S2S_OK;
}

int s2s_llama_bind_tensor(s2s_llama* m, const char* name, const void* data_h, const int64_t* shape, int32_t ndim,
                          int32_t dtype) {
  S2S_REQUIRE(m && name && data_h && shape, "llama bind_tensor: null argument");
  auto it = m->slots.find(name);
  if (it == m->slots.end()) {
    s2s_set_error("llama bind_tensor: unknown tensor '%s'", name);
    return S2S_ERR_NOT_FOUND;
  }
  LSlot& s = it->second;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  S2S_REQUIRE(n == s.rows * s.cols, "llama bind_tensor: '%s' has %lld elements, expected %lld", name, (long long)n,
              (long long)(s.rows * s.cols));
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  const bool bf = m->cfg.compute_dtype == S2S_BF16;
  if (!s.half) {
    std::vector<float> tmp((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      int64_t di = i;
      if (s.kind == L_ROPE_PERM) { const int64_t half = s.hd / 2, j = i % s.hd; di = (i / s.hd) * s.hd + (j < half ? 2 * j : 2 * (j - half) + 1); }
      tmp[(size_t)di] = src_f32(data_h, i, dtype);
    }
    S2S_CHECK_CUDA(cudaMemcpy(s.dst, tmp.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  } else {
    // row-wise conversion + placement
    std::vector<uint16_t> rowbuf((size_t)s.cols);
    for (int64_t r = 0; r < s.rows; ++r) {
      for (int64_t c = 0; c < s.cols; ++c) {
        const float v = src_f32(data_h, r * s.cols + c, dtype);
        rowbuf[(size_t)c] = bf ? f2bf(v) : f2h(v);
      }
      int64_t dr = r;
      if (s.kind == L_ROPE_PERM) {
        const int64_t h = r / s.hd, j = r % s.hd, half = s.hd / 2;
        dr = h * s.hd + (j < half ? 2 * j : 2 * (j - half) + 1);
      } else if (s.kind == L_INTERLEAVE) {
        dr = 2 * r + s.parity;
      }
      S2S_CHECK_CUDA(cudaMemcpy(reinterpret_cast<char*>(s.dst) + dr * s.cols * 2, rowbuf.data(), (size_t)s.cols * 2,
                                cudaMemcpyHostToDevice));
    }
  }
  s.bound = true;
  if (strncmp(name, "lm_head.", 8) == 0) m->lm_head_bound = true;
  return S2S_OK;
}

int s2s_llama_init_random(s2s_llama* m, uint64_t seed) {
  S2S_REQUIRE(m, "llama init_random: null model");
  S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  for (auto& kv : m->slots) {
    LSlot& s = kv.second;
    uint64_t hsh = 1469598103934665603ull;
    for (char ch : kv.first) hsh = (hsh ^ (uint64_t)(unsigned char)ch) * 1099511628211ull;
    if (s.kind == L_INTERLEAVE) {
      if (s.parity == 1) { s.bound = true; continue; }  // gate slot fills the whole interleaved [2*ffn, d] block
      S2S_CHECK(fill_random_launch(s.dst, 2 * s.rows * s.cols, m->cfg.compute_dtype, s.rnd_scale, 0.f, seed ^ hsh, 0));
    } else {
      S2S_CHECK(fill_random_launch(s.dst, s.rows * s.cols, s.half ? m->cfg.compute_dtype : S2S_F32, s.rnd_scale,
                                   s.rnd_offset, seed ^ hsh, 0));
    }
    s.bound = true;
  }
  m->lm_head_bound = true;
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  return S2S_OK;
}

int s2s_llama_finalize(s2s_llama* m) {
  S2S_REQUIRE(m, "llama finalize: null model");
  if (m->n_tables == 1 && !m->lm_head_bound && m->slots["model.embed_tokens.weight"].bound) {
    // tied embeddings (tie_word_embeddings=True): lm_head shares embed_tokens
    S2S_CHECK_CUDA(cudaMemcpy(m->lm_head, m->embed, (size_t)m->cfg.vocab * m->cfg.d_model * 2, cudaMemcpyDeviceToDevice));
    m->slots["lm_head.weight"].bound = true;
  }
  for (auto& kv : m->slots)
    if (!kv.second.bound) {
      s2s_set_error("llama finalize: tensor '%s' was never bound", kv.first.c_str());
      return S2S_ERR_INVALID;
    }
  // decode-side weight layout: fragment-major tiles (weight_tiles.cu), built once per (re)load
  {
    const auto& c = m->cfg;
    const int d = c.d_model, qd = c.heads * c.head_dim, kvd = c.kv_heads * c.head_dim, f = c.ffn;
    S2S_CHECK_CUDA(cudaSetDevice(m->ctx->device));
    if (m->tiled_h.empty()) {
      m->tiled_h = m->layers_h;
      for (int i = 0; i < c.layers; ++i) {
        LlamaDecLayer& T = m->tiled_h[i];
        void *a, *b, *g, *dn;
        S2S_CHECK(lalloc(m, &a, tiled_weight_elems(qd + 2 * kvd, d) * 2));
        S2S_CHECK(lalloc(m, &b, tiled_weight_elems(d, qd) * 2));
        S2S_CHECK(lalloc(m, &g, tiled_weight_elems(2 * f, d) * 2));
        S2S_CHECK(lalloc(m, &dn, tiled_weight_elems(d, f) * 2));
        T.w_qkv = a; T.w_o = b; T.w_gu = g; T.w_down = dn;
      }
      m->head_t_table_elems = tiled_weight_elems(c.vocab, d);
      S2S_CHECK(lalloc(m, &m->lm_head_t, m->n_tables * m->head_t_table_elems * 2));
      S2S_CHECK_CUDA(cudaMemcpy(m->layers_d, m->tiled_h.data(), sizeof(LlamaDecLayer) * c.layers, cudaMemcpyHostToDevice));
    }
    for (int i = 0; i < c.layers; ++i) {
      const LlamaDecLayer& R = m->layers_h[i];
      const LlamaDecLayer& T = m->tiled_h[i];
      S2S_CHECK(tile_weights_launch(R.w_qkv, qd + 2 * kvd, d, const_cast<void*>(T.w_qkv), 0));
      S2S_CHECK(tile_weights_launch(R.w_o, d, qd, const_cast<void*>(T.w_o), 0));
      S2S_CHECK(tile_weights_launch(R.w_gu, 2 * f, d, const_cast<void*>(T.w_gu), 0));
      S2S_CHECK(tile_weights_launch(R.w_down, d, f, const_cast<void*>(T.w_down), 0));
    }
    for (int t = 0; t < m->n_tables; ++t)
      S2S_CHECK(tile_weights_launch(reinterpret_cast<char*>(m->lm_head) + (size_t)t * m->head_table_elems * 2, c.vocab, d,
                                    reinterpret_cast<char*>(m->lm_head_t) + (size_t)t * m->head_t_table_elems * 2, 0));
    S2S_CHECK_CUDA(cudaDeviceSynchronize());
  }
  m->finalized = true;
  return S2S_OK;
}

int s2s_llama_session_reset(s2s_llama* m, int32_t slot) {
  S2S_REQUIRE(m && slot >= 0 && slot < m->cfg.max_sessions, "llama session_reset: bad slot %d", slot);
  m->len[slot] = 0;
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
  S2S_CHECK_CUDA(cudaStreamSynchronize(st));
  LlamaDecParams p{};
  llama_fill_dec_params(m, p);
  p.B = B; p.slot = m->slot_d; p.pos = m->pos_d; p.max_len = max_len;
  p.first_ids = first_ids_d; p.n_steps = n_steps; p.eos = eos_id; p.out_ids = ids_out_d; p.out_len = len_out_d;
  p.forced = forced_d; p.logits_out = logits_out_d;
  S2S_CHECK(llama_decode_launch(m->ctx, p, c.compute_dtype, m->debug_phases, st));
  for (int b = 0; b < B; ++b) m->len[slots_h[b]] += n_steps;
  return S2S_OK;
}

int32_t s2s_llama_max_decode_batch(s2s_llama* m) {
  if (!m) return 0;
  return llama_max_decode_batch_of(m);
}

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
  // ids_out[0] = argmax of the prompt's last position; the decode kernel then feeds it and produces the rest
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

}  // extern "C"
