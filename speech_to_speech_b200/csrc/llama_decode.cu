// llama_decode.cu -- greedy decode of a Llama-family LLM as ONE persistent cooperative kernel.
//
// Reference path: LanguageModelHandler._generate -> pipeline("text-generation") -> model.generate greedy
// (S/LLM/language_model.py:832-892) over LlamaForCausalLM (transformers modeling_llama.py:292-333 layer,
// :225-289 attention, :171-184 MLP, :53-71 RMSNorm, :140-168 RoPE).  The reference streams the 16 GB of bf16
// weights once per token through ~10 library kernels per layer and synchronises with the host every token
// (TextIteratorStreamer); here a token step is 5 phases per layer inside one launch:
//   0: RMSNorm + QKV projection + RoPE + KV append   1: GQA attention items (32-key blocks, last split merges)
//   2: o_proj + residual                             3: RMSNorm + gate/up projection + SwiGLU     4: down + residual
//   then 5L: final RMSNorm + lm_head + per-CTA argmax      5L+1: global argmax, EOS bookkeeping, next embedding
// Sessions with sampling parameters (sampling.cuh) have their logits row stored in phase 5L and chosen from it by the CTA
// that owns the session in phase 5L+1: no extra phase, no extra grid barrier.
// Qwen3 family (qk_norm, transformers modeling_qwen3.py Qwen3Attention): phase 0 stores RAW q / k; the per-head
// RMSNorm(head_dim) + RoPE is folded into the attention items of phase 1 (ld_qk_prepare), so the phase count stays 5 per
// layer (a sixth phase would add one grid barrier per layer and step to the TTS frame loop).
// Projections are swap-AB tensor-core GEMVs (sessions on m) fed from per-warp bulk-copy rings of fragment-major weights
// (decode_common.cuh, weight_tiles.cu); HBM-bound: 15.0 GB / token for Llama-3-8B (SURVEY.md Appendix A).
// F8 instantiation: the same kernel over FP8 E4M3 weights with power-of-two row scales (7.5 GB / token), bf16 compute only.
// Every projection of the launch, lm_head included, is FP8, so the kernel still holds one GEMV routine.
#include <algorithm>
#include <vector>

#include "llama_decode.cuh"
#include "llama_decode_plan.cuh"

namespace {

// Qwen3: RMSNorm over head_dim of a raw q / k row (fp32 statistics, Qwen3RMSNorm), then RoPE.  One warp; rows are stored
// pair-adjacent (2j, 2j+1) = rotate_half partners (j, j + hd/2), and so are the norm weights.  y: this lane's PER elements.
template <int HD>
__device__ __forceinline__ void ld_norm_rope_head(const float* src, const float* nw, const float2* rope_pos, float eps,
                                                  float (&y)[HD / 32]) {
  constexpr int PER = HD / 32;  // 2 or 4 consecutive elements per lane = 1 or 2 rotation pairs
  const int lane = threadIdx.x & 31;
  float v[PER], g[PER];
  if (PER == 4) {
    const float4 t = __ldcg(reinterpret_cast<const float4*>(src + lane * 4));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    const float4 u = __ldg(reinterpret_cast<const float4*>(nw + lane * 4));
    g[0] = u.x; g[1] = u.y; g[2] = u.z; g[3] = u.w;
  } else {
    const float2 t = __ldcg(reinterpret_cast<const float2*>(src + lane * 2));
    v[0] = t.x; v[1] = t.y;
    const float2 u = __ldg(reinterpret_cast<const float2*>(nw + lane * 2));
    g[0] = u.x; g[1] = u.y;
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) ss = fmaf(v[i], v[i], ss);
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss * (1.0f / (float)HD) + eps);
#pragma unroll
  for (int i = 0; i < PER; i += 2) {
    const float2 cs = rope_pos[(lane * PER + i) >> 1];
    const float a0 = v[i] * rstd * g[i], a1 = v[i + 1] * rstd * g[i + 1];
    y[i] = a0 * cs.x - a1 * cs.y;
    y[i + 1] = a1 * cs.x + a0 * cs.y;
  }
}

// Qwen3 (qk_norm), executed by ONE warp at the head of an attention item (session b, q head h): the normalised, rotated and
// scaled q row goes to p.qn (the item's attend_blocks reads it from there); when the item's key range holds the step's own
// key (`own_key`), the kv head's normalised + rotated k row is appended to the cache first.  Items that share a (session,
// head) -- the key splits -- or a kv head write identical bytes, so no cross-CTA ordering is needed: every reader has
// written the value itself (same warp: __syncwarp, same CTA: __syncthreads, issued by the caller).
template <typename T, int HD>
__device__ __forceinline__ void ld_qk_prepare(const LlamaDecParams& p, int layer, int b, int h, int pos, bool own_key) {
  constexpr int PER = HD / 32;
  const int H = p.heads, KV = p.kv_heads, lane = threadIdx.x & 31, g = h / (H / KV);
  const LlamaDecLayer& w = p.lw[layer];
  const float2* rp = p.rope + (long long)pos * (HD >> 1);
  float y[PER];
  ld_norm_rope_head<HD>(p.q + (long long)b * H * HD + h * HD, w.q_norm, rp, p.eps, y);
  const float q_scale = rsqrtf((float)HD);
  float* qd = p.qn + (long long)b * H * HD + h * HD + lane * PER;
#pragma unroll
  for (int i = 0; i < PER; i += 2) *reinterpret_cast<float2*>(qd + i) = make_float2(y[i] * q_scale, y[i + 1] * q_scale);
  if (own_key) {
    ld_norm_rope_head<HD>(p.kraw + (long long)b * KV * HD + g * HD, w.k_norm, rp, p.eps, y);
    T* dst = reinterpret_cast<T*>(p.kv) + (long long)__ldg(p.slot + b) * p.kv_slot_stride + (long long)layer * p.kv_layer_stride +
             (long long)pos * (KV * HD) + g * HD + lane * PER;
#pragma unroll
    for (int i = 0; i < PER; i += 2) *reinterpret_cast<uint32_t*>(dst + i) = DT<T>::pack2(y[i], y[i + 1]);
  }
}

// GQA attention over each session's cached keys; items (session, q head, key split) per attn_plan (decode_common.cuh)
template <typename T, int HD>
__device__ __noinline__ void ld_attn(const LlamaDecParams& p, int layer, int step, float* rec_s) {
  const int H = p.heads, grp = p.heads / p.kv_heads, warp = threadIdx.x >> 5;
  const int kvd = p.kv_heads * HD;
  constexpr int REC = HD + PART_PAD;
  const int n_blocks = (p.max_len + step + ATT_BLK - 1) / ATT_BLK, BH = p.B * H;  // longest session
  // the split plan of assoc_b sessions (LlamaDecPlan): it fixes the softmax-merge association of every item
  const int plan = attn_plan(p.assoc_b * H, n_blocks, p.s_max, (int)gridDim.x);
  const int S = plan & 0x7f, bps = (n_blocks + S - 1) / S;
  const bool wl = plan & ATTN_WARP_LEVEL;
  const T* kv = reinterpret_cast<const T*>(p.kv);
  const float* qbase = p.qk_norm ? p.qn : p.q;
#pragma unroll 1
  for (int it = wl ? dec_first_item() : (int)blockIdx.x; it < BH * S; it += wl ? dec_item_stride() : (int)gridDim.x) {
    const int s = it % S, bh = it / S, h = bh % H, b = bh / H;
    const int pos = __ldcg(p.pos + b), len = pos + 1;  // this session's keys; splits past its end produce empty records
    const int nb = (len + ATT_BLK - 1) / ATT_BLK;
    const T* Kb = kv + (long long)__ldg(p.slot + b) * p.kv_slot_stride + (long long)layer * p.kv_layer_stride + (h / grp) * HD;
    float* part_bh = p.part + (long long)bh * p.s_max * REC;
    T* out16 = reinterpret_cast<T*>(p.attn16) + (long long)b * H * HD + h * HD;
    const float* q = qbase + (long long)b * H * HD + h * HD;
    const int blk0 = s * bps, blk1 = min((s + 1) * bps, nb);
    if (p.qk_norm && blk0 < blk1) {   // the split that holds the step's own key (the last block) appends it
      if (wl || warp == 0) ld_qk_prepare<T, HD>(p, layer, b, h, pos, blk1 == nb);
      if (wl) __syncwarp(); else __syncthreads();
    }
    attn_run_item<T, HD>(wl, q, Kb, Kb + p.kv_which_stride, kvd, len, blk0, blk1, rec_s, part_bh, s, S, p.attn_cnt + bh, out16);
  }
}

// s2s_decode_attention: the attention phase of layer 0, step 0 alone (no grid barrier inside a phase: a plain launch)
template <typename T, int HD>
__global__ void __launch_bounds__(DEC_THREADS, 1) ld_attn_only_kernel(const __grid_constant__ LlamaDecParams p) {
  extern __shared__ __align__(16) float rec_s[];   // DEC_WARPS records
  ld_attn<T, HD>(p, 0, 0, rec_s);
}


// phase kinds: 0 qkv, 1 attention (Qwen3: + q/k norm and RoPE), 2 o_proj, 3 gate/up, 4 down, 6 logits, 7 select
__host__ __device__ __forceinline__ int ld_nsub(const LlamaDecParams&) { return 5; }
__device__ __forceinline__ int ld_kind(const LlamaDecParams& p, int ph) {
  if (ph >= 5 * p.layers) return ph == 5 * p.layers ? 6 : 7;
  return ph % 5;
}
__device__ __forceinline__ bool ld_multi(const LlamaDecParams& p) { return p.head_stride != 0; }
// output head of `step` (multi-table mode: step 0 predicts nothing)
__device__ __forceinline__ bool ld_has_head(const LlamaDecParams& p, int step) { return !(ld_multi(p) && step == 0); }
__device__ __forceinline__ bool ld_has_gemv(const LlamaDecParams& p, int step, int ph) {
  const int k = ld_kind(p, ph);
  return k == 0 || k == 2 || k == 3 || k == 4 || (k == 6 && ld_has_head(p, step));
}

// s_samp: the tail-round reduction buffer of the projections, idle in this phase (the look-ahead issued between the
// previous barrier's arrive and wait only fills the weight ring and the norm-weight buffer)
template <typename T>
__device__ __noinline__ void ld_select(const LlamaDecParams& p, int step, float* s_aux, SampShared& s_samp) {
  const int d = p.d, B = p.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* s_feed = reinterpret_cast<int*>(s_aux);
#pragma unroll 1
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    const SampSlot* sc = p.samp ? p.samp + b : nullptr;
    const bool sampled = sc && sc->active && ld_has_head(p, step);
    int stok = 0;
    if (sampled) {   // the whole CTA selects from the step's logits row; pos[b] + 1 = position of the predicted token
      const float* row = p.logits_out ? p.logits_out + ((long long)step * B + b) * p.vocab : p.samp_rows + (long long)b * p.vocab;
      stok = sample_row(row, p.vocab, *sc, p.seen + (long long)p.slot[b] * p.seen_words, p.pos[b] + 1, s_samp);
    }
    if (warp == 0) {
      // bookkeeping operands first: their round trips overlap the candidate loads
      const int was_done = p.done[b];
      const int forced_tok = p.forced ? p.forced[b * p.n_steps + step] : 0;
      int tok;
      if (sampled) tok = stok;
      else if (ld_has_head(p, step)) tok = dec_argmax_merge(p.cand_val, p.cand_idx, b);
      else tok = p.first_ids[b];  // multi-table mode, step 0: nothing predicted, the known first id is fed
      if (lane == 0) {
        const int f = dec_record_token(p, b, step, p.n_steps, tok, was_done, forced_tok);
        *s_feed = f;
        if (sc && sc->penalty != 1.f && !p.seen_fixed) atomicOr(p.seen + (long long)p.slot[b] * p.seen_words + (f >> 5), 1u << (f & 31));
        p.pos[b] = p.pos[b] + 1;  // the fed token sits at the next position
      }
    }
    __syncthreads();
    const int feed = *s_feed;
    const T* tab = reinterpret_cast<const T*>(p.embed);
    if (ld_multi(p)) tab = step == 0 ? reinterpret_cast<const T*>(p.embed0) : tab + (long long)(step - 1) * p.embed_stride;
    const T* e = tab + (long long)feed * d;
#pragma unroll 2
    for (int i = threadIdx.x; i < d; i += DEC_THREADS) p.x[(long long)b * d + i] = DT<T>::to_f(e[i]);
  }
}

// The kernel's phases for dec_run (decode_common.cuh).  Holds a reference to the kernel's shared copy of the parameters.
template <typename T, bool F8>
struct LdModel {
  static constexpr bool stamps_barrier = true;
  static constexpr bool f8_weights = F8;
  const LlamaDecParams& p;
  int n_phases;

  __device__ __forceinline__ bool skip(int step, int ph) const {   // nothing to predict: no work, no barrier
    return ld_kind(p, ph) == 6 && !ld_has_head(p, step);
  }
  __device__ __forceinline__ bool has_gemv(int step, int ph) const { return ld_has_gemv(p, step, ph); }
  __device__ __forceinline__ bool lookahead_target(int step, int ph) const { return ld_has_gemv(p, step, ph); }
  __device__ __forceinline__ void prefetch_l2(int, int) const {}
  __device__ __forceinline__ DecNorm norm_of(int ph) const {
    const int k = ld_kind(p, ph);
    if (k == 0) return {p.lw[ph / ld_nsub(p)].norm1, nullptr};
    if (k == 3) return {p.lw[ph / ld_nsub(p)].norm2, nullptr};
    return {k == 6 ? p.norm_f : nullptr, nullptr};
  }

  __device__ __forceinline__ void gemv_args(int step, int ph, GemvArgs& a) const {
    const int d = p.d, B = p.B, qd = p.heads * p.hd, kvd = p.kv_heads * p.hd;
    gemv_args_reset(a, d, p.q);
    a.pos = p.pos; a.slot = p.slot; a.kv_slot = p.kv_slot_stride; a.kv_ld = kvd; a.rope = p.rope; a.hd = p.hd;
    a.q_rows = qd; a.k_rows = kvd; a.q_scale = rsqrtf((float)p.hd);
    const int kind = ld_kind(p, ph);
    if (kind < 6) {
      const int layer = ph / ld_nsub(p);
      const LlamaDecLayer& w = p.lw[layer];
      switch (kind) {
        case 0:
          a.W = w.w_qkv; a.N = qd + 2 * kvd; a.mode = EPI_QKV_ROPE; a.out = p.q; a.ldo = qd; a.plan_id = 0;
          a.kv0 = reinterpret_cast<T*>(p.kv) + (long long)layer * p.kv_layer_stride; a.kv_which = p.kv_which_stride;
          a.kraw = p.qk_norm ? p.kraw : nullptr;
          return;
        case 2: a.W = w.w_o; a.N = d; a.K = qd; a.mode = EPI_RESID; a.out = p.x; a.ldo = d; a.plan_id = 1; return;
        case 3: a.W = w.w_gu; a.N = 2 * p.ffn; a.mode = EPI_SWIGLU; a.out_h = p.h; a.ldh = p.ffn; a.plan_id = 2; return;
        case 4:
          a.W = w.w_down; a.N = d; a.K = p.ffn; a.mode = EPI_RESID; a.out = p.x; a.ldo = d; a.plan_id = 3;
          if (p.down_kc > 0) { a.xsrc = p.h; a.xsrc_ld = p.ffn; a.kc = p.down_kc; a.plan_id = -1; }
          return;
        default: return;
      }
    }
    if (kind == 6 && ld_has_head(p, step)) {
      a.W = ld_multi(p) ? reinterpret_cast<const T*>(p.lm_head) + (long long)(step - 1) * p.head_stride : p.lm_head;
      a.N = p.vocab; a.mode = EPI_LOGITS; a.plan_id = 4; a.suppress = p.suppress;
      // sessions that sample read their row back in the select phase: from logits_out when the caller asked for it, else from
      // the row scratch (every row of such a launch is stored, a few MB against the step's weight stream)
      a.logits_out = p.logits_out ? p.logits_out + (long long)step * B * p.vocab : p.samp ? p.samp_rows : nullptr;
      a.logits_ld = p.vocab;
    }
  }

  __device__ __forceinline__ void phase(int step, int ph, const DecViews<T>& sm, GemvRing& ring, GemvArgs* ready,
                                        GemvArgs* scratch, int wb_ready, unsigned long long*) const {
    const int d = p.d, B = p.B;
    float best_v[2] = {-INFINITY, -INFINITY};
    int best_i[2] = {0x7fffffff, 0x7fffffff};
    const int kind = ld_kind(p, ph);
    if (!ready && ld_has_gemv(p, step, ph)) {
      if (threadIdx.x == 0) gemv_args(step, ph, *scratch);  // one thread writes the shared struct
      __syncthreads();
    }
    GemvArgs& a = ready ? *ready : *scratch;
    if (kind < 6) {
      const int layer = ph / ld_nsub(p);
      const LlamaDecLayer& w = p.lw[layer];
      switch (kind) {
        case 0: stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 2, w.norm1, nullptr, p.eps, sm.s_red, sm.wb, wb_ready, p.norm_rg); break;
        case 1:
          if (p.hd == 128) ld_attn<T, 128>(p, layer, step, reinterpret_cast<float*>(sm.red));
          else ld_attn<T, 64>(p, layer, step, reinterpret_cast<float*>(sm.red));
          return;
        case 2: stage_rows_copy<T>(reinterpret_cast<const T*>(p.attn16), B, p.heads * p.hd, sm.xh); break;
        case 3: stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 2, w.norm2, nullptr, p.eps, sm.s_red, sm.wb, wb_ready, p.norm_rg); break;
        default:
          if (a.kc > 0) { gemv_mma_chunked<T, true, F8>(a, sm.xh, B, best_v, best_i, ring, sm.red); return; }
          stage_rows_copy<T>(reinterpret_cast<const T*>(p.h), B, p.ffn, sm.xh); break;
      }
      gemv_mma<T, true, F8>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      return;
    }
    if (kind == 6) {
      if (p.hidden_out && blockIdx.x == 0)  // the residual stream before the final norm (Qwen3-TTS: input of the code predictor)
        for (int i = threadIdx.x; i < B * d; i += DEC_THREADS) p.hidden_out[(long long)step * B * d + i] = __ldcg(p.x + i);
      stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 2, p.norm_f, nullptr, p.eps, sm.s_red, sm.wb, wb_ready, p.norm_rg);
      gemv_mma<T, true, F8>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      gemv_argmax_candidates(best_v, best_i, B, sm.sv, sm.si, p.cand_val, p.cand_idx);
    } else {
      static_assert(sizeof(SampShared) <= 2 * DEC_THREADS * 16, "sampling scratch must fit the tail-round buffer");
      ld_select<T>(p, step, sm.sv, *reinterpret_cast<SampShared*>(sm.red));
    }
  }
};

template <typename T, bool F8>
__global__ void __launch_bounds__(DEC_THREADS, 1)
llama_decode_kernel(const LlamaDecParams p, int step_begin, int step_end, int ph_begin, int ph_end, int coop) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ LlamaDecParams sp;
  __shared__ LlamaDecLayer s_layers[64];
  __shared__ GemvPlan s_plans[5];  // qkv | o_proj | gate/up | down | lm_head
  __shared__ GemvArgs s_args[2];   // [0] prepared for the next projection, [1] built in-phase
  __shared__ GemvRing s_rings[DEC_WARPS];
  if (threadIdx.x < 5) {
    const int i = threadIdx.x, qd = p.heads * p.hd, kvd = p.kv_heads * p.hd;
    gemv_make_plan(i == 0 ? qd + 2 * kvd : i == 2 ? 2 * p.ffn : i == 4 ? p.vocab : p.d, i == 1 ? qd : i == 3 ? p.ffn : p.d, s_plans[i]);
  }
  if (threadIdx.x == 0) { sp = p; sp.lw = s_layers; }
  for (int i = threadIdx.x; i < p.layers; i += DEC_THREADS) s_layers[i] = p.lw[i];
  __syncthreads();
  const int kmax_whole = p.down_kc > 0 ? ld_kmax(p.d, p.down_kc, p.heads * p.hd) : ld_kmax(p.d, p.ffn, p.heads * p.hd);
  const DecSmem lay = dec_smem_layout(p.B, p.d, kmax_whole, p.d, p.norm_rg);
  GemvRing& ring = s_rings[threadIdx.x >> 5];
  gemv_ring_init(ring, smem_raw + lay.ring_off, p.ring_slots, s_plans);
  const LdModel<T, F8> model{sp, ld_nsub(p) * p.layers + 2};
  dec_run<T>(p, model, dec_views<T>(smem_raw, lay), ring, s_args, step_begin, step_end, ph_begin, ph_end, coop);
}

template <typename T>
__global__ void llama_decode_init_kernel(const LlamaDecParams p) {
  const int b = blockIdx.x;
  if (p.x_in) {
    for (int i = threadIdx.x; i < p.d; i += blockDim.x) p.x[(long long)b * p.d + i] = p.x_in[(long long)b * p.d + i];
  } else {
    const int tok = p.first_ids[b];
    const T* e = reinterpret_cast<const T*>(p.embed) + (long long)tok * p.d;
    for (int i = threadIdx.x; i < p.d; i += blockDim.x) p.x[(long long)b * p.d + i] = DT<T>::to_f(e[i]);
  }
  // the first fed id is in the sequence now: it joins the seen set of a session with a repetition penalty (the select
  // phase adds the ids fed after it)
  if (threadIdx.x == 0 && p.samp && p.samp[b].active && p.samp[b].penalty != 1.f && !p.seen_fixed) {
    const int f = p.first_ids[b];
    atomicOr(p.seen + (long long)p.slot[b] * p.seen_words + (f >> 5), 1u << (f & 31));
  }
  dec_init_session(p, b, p.n_steps);
}

template <typename T, bool F8>
int launch_t(s2s_ctx* ctx, const LlamaDecParams& p, int debug_phases, cudaStream_t stream) {
  const int grid = dec_grid(ctx);  // the context's SM partition (s2s_set_sm_partition)
  auto kern = llama_decode_kernel<T, F8>;
  long long max_dyn = 0;
  S2S_CHECK_CUDA(s2s_max_dyn_smem(kern, ctx->device, &max_dyn));
  LlamaDecPlan pl;
  S2S_REQUIRE(llama_decode_plan(p.B, p.d, p.ffn, p.heads * p.hd, grid, max_dyn, &pl),
              "llama decode: batch %d does not fit shared memory for d %d, ffn %d", p.B, p.d, p.ffn);
  const DecSmem lay = dec_smem_layout(p.B, p.d, pl.kmax, p.d, pl.rg);
  LlamaDecParams pr = p;
  pr.ring_slots = pl.slots; pr.norm_rg = pl.rg; pr.down_kc = pl.kc; pr.assoc_b = pl.assoc_b;
  const size_t smem = dec_smem_bytes(lay, pl.slots);
  S2S_REQUIRE((long long)smem <= max_dyn, "llama decode: plan of batch %d needs %zu B of shared memory, %lld available", p.B, smem,
              max_dyn);
  S2S_CHECK_CUDA(s2s_opt_in_max_smem(kern, ctx->device, smem, nullptr));
  llama_decode_init_kernel<T><<<p.B, 256, 0, stream>>>(pr);
  S2S_LAUNCH_CHECK();
  return dec_launch(kern, pr, grid, 0, smem, p.n_steps, ld_nsub(p) * p.layers + 2, debug_phases, stream);
}

}  // namespace

int llama_decode_launch(s2s_ctx* ctx, const LlamaDecParams& p, int dtype, int weight_format, int debug_phases, cudaStream_t stream) {
  S2S_REQUIRE(p.hd == 64 || p.hd == 128, "llama decode: head_dim must be 64 or 128");
  S2S_REQUIRE(p.layers <= 64, "llama decode: at most 64 layers");
  S2S_REQUIRE(p.n_steps >= 1, "llama decode: n_steps must be >= 1");
  S2S_REQUIRE(p.B >= 1 && p.B <= DEC_MAX_B, "llama decode: batch %d > %d must be split by the caller", p.B, DEC_MAX_B);
  S2S_REQUIRE(p.d % 64 == 0 && p.ffn % 64 == 0 && (p.heads * p.hd) % 64 == 0, "llama decode: d, ffn, heads*hd must be multiples of 64");
  if (weight_format == S2S_FP8_E4M3) {
    if (dtype == S2S_BF16 && p.head_stride == 0) return launch_t<__nv_bfloat16, true>(ctx, p, debug_phases, stream);
  } else if (weight_format == dtype) {
    if (dtype == S2S_BF16) return launch_t<__nv_bfloat16, false>(ctx, p, debug_phases, stream);
    if (dtype == S2S_F16) return launch_t<__half, false>(ctx, p, debug_phases, stream);
  }
  s2s_set_error("llama decode: unsupported dtype %d with weight format %d", dtype, weight_format);
  return S2S_ERR_UNSUPPORTED;
}

int llama_decode_max_batch(int device, int dtype, int weight_format, int d, int ffn, int qd, int grid) {
  long long max_dyn = 0;
  const cudaError_t e = weight_format == S2S_FP8_E4M3 ? s2s_max_dyn_smem(llama_decode_kernel<__nv_bfloat16, true>, device, &max_dyn)
                        : dtype == S2S_F16            ? s2s_max_dyn_smem(llama_decode_kernel<__half, false>, device, &max_dyn)
                                                      : s2s_max_dyn_smem(llama_decode_kernel<__nv_bfloat16, false>, device, &max_dyn);
  if (e != cudaSuccess) return 0;
  return llama_decode_plan_max_batch(d, ffn, qd, grid, max_dyn);
}

extern "C" int s2s_decode_attention(s2s_ctx* ctx, const s2s_dec_attn_args* args, int32_t* plan_out_h, void* stream) {
  S2S_REQUIRE(ctx && args, "s2s_decode_attention: null argument");
  const s2s_dec_attn_args& a = *args;
  S2S_REQUIRE(a.q && a.kv && a.out && a.slots_h && a.lens_h, "s2s_decode_attention: null q / kv / out / slots_h / lens_h");
  S2S_REQUIRE(a.B >= 1 && a.B <= DEC_MAX_B, "s2s_decode_attention: B %d not in [1, %d]", a.B, DEC_MAX_B);
  S2S_REQUIRE(a.heads >= 1 && a.kv_heads >= 1 && a.heads % a.kv_heads == 0, "s2s_decode_attention: heads %d / kv_heads %d",
              a.heads, a.kv_heads);
  S2S_REQUIRE(a.hd == 64 || a.hd == 128, "s2s_decode_attention: hd %d (64 or 128)", a.hd);
  S2S_REQUIRE(a.dtype == S2S_F16 || a.dtype == S2S_BF16, "s2s_decode_attention: dtype %d", a.dtype);
  S2S_REQUIRE(a.max_pos >= 1 && a.grid >= 0 && a.assoc_b >= 0 && a.assoc_b <= DEC_MAX_B,
              "s2s_decode_attention: max_pos %d / grid %d / assoc_b %d", a.max_pos, a.grid, a.assoc_b);
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  S2S_REQUIRE(al(a.q) && al(a.kv), "s2s_decode_attention: q / kv must be 16-byte aligned");
  S2S_REQUIRE(a.qk_norm == 0 || a.qk_norm == 1, "s2s_decode_attention: qk_norm %d", a.qk_norm);
  if (a.qk_norm) {
    S2S_REQUIRE(a.kraw && a.q_norm && a.k_norm && a.rope, "s2s_decode_attention: qk_norm needs kraw / q_norm / k_norm / rope");
    S2S_REQUIRE(al(a.kraw) && al(a.q_norm) && al(a.k_norm) && al(a.rope) && al(a.qn_out),
                "s2s_decode_attention: kraw / q_norm / k_norm / rope / qn_out must be 16-byte aligned");
  }
  int host[2 * DEC_MAX_B] = {}, max_len = 0;   // slots, then positions (len - 1)
  for (int b = 0; b < a.B; ++b) {
    S2S_REQUIRE(a.slots_h[b] >= 0 && a.lens_h[b] >= 1 && a.lens_h[b] <= a.max_pos,
                "s2s_decode_attention: session %d: slot %d / len %d not in [1, %d]", b, a.slots_h[b], a.lens_h[b], a.max_pos);
    host[b] = a.slots_h[b];
    host[DEC_MAX_B + b] = a.lens_h[b] - 1;
    max_len = std::max(max_len, a.lens_h[b]);
  }
  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  const cudaStream_t st = (cudaStream_t)stream;
  const int grid = a.grid > 0 ? a.grid : dec_grid(ctx);
  const int kvd = a.kv_heads * a.hd, BH = a.B * a.heads;
  LlamaDecParams p{};
  p.heads = a.heads; p.kv_heads = a.kv_heads; p.hd = a.hd; p.B = a.B; p.max_pos = a.max_pos; p.layers = 1;
  p.q = const_cast<float*>(a.q); p.kv = a.kv; p.attn16 = a.out;
  p.kv_which_stride = (long long)a.max_pos * kvd; p.kv_layer_stride = 2 * p.kv_which_stride; p.kv_slot_stride = p.kv_layer_stride;
  p.s_max = (a.max_pos + 63) / 64;   // as llama_create sizes the records
  p.max_len = max_len; p.assoc_b = a.assoc_b > 0 ? a.assoc_b : a.B;
  if (plan_out_h) *plan_out_h = attn_plan(p.assoc_b * a.heads, (max_len + ATT_BLK - 1) / ATT_BLK, p.s_max, grid);
  // per-call scratch: split records, split counters (zeroed), slots and positions; Qwen3: the one-layer weight table and,
  // without qn_out, the normalised q
  const size_t part_bytes = (size_t)BH * p.s_max * (a.hd + PART_PAD) * 4;
  const size_t idx_off = part_bytes + (size_t)BH * 4, layer_off = (idx_off + sizeof(host) + 15) / 16 * 16;
  const size_t qn_off = layer_off + (sizeof(LlamaDecLayer) + 15) / 16 * 16;
  const size_t scratch_bytes = a.qk_norm ? qn_off + (a.qn_out ? 0 : (size_t)BH * a.hd * 4) : idx_off + sizeof(host);
  char* scratch = nullptr;
  S2S_CHECK_CUDA(cudaMalloc(&scratch, scratch_bytes));
  p.part = reinterpret_cast<float*>(scratch);
  p.attn_cnt = reinterpret_cast<unsigned int*>(scratch + part_bytes);
  int* idx_d = reinterpret_cast<int*>(scratch + idx_off);
  p.slot = idx_d; p.pos = idx_d + DEC_MAX_B;
  LlamaDecLayer layer{};
  if (a.qk_norm) {   // ld_attn's Qwen3 path reads the norm weights from layer 0 of the model's table
    layer.q_norm = a.q_norm; layer.k_norm = a.k_norm;
    p.lw = reinterpret_cast<const LlamaDecLayer*>(scratch + layer_off);
    p.qk_norm = 1; p.kraw = const_cast<float*>(a.kraw); p.rope = reinterpret_cast<const float2*>(a.rope); p.eps = a.eps;
    p.qn = a.qn_out ? a.qn_out : reinterpret_cast<float*>(scratch + qn_off);
  }
  std::vector<unsigned int> cnt((size_t)BH, 0u);
  auto run = [&]() -> int {
    S2S_CHECK_CUDA(cudaMemsetAsync(p.attn_cnt, 0, (size_t)BH * 4, st));
    S2S_CHECK_CUDA(cudaMemcpyAsync(idx_d, host, sizeof(host), cudaMemcpyHostToDevice, st));
    if (a.qk_norm) S2S_CHECK_CUDA(cudaMemcpyAsync(scratch + layer_off, &layer, sizeof(layer), cudaMemcpyHostToDevice, st));
    const size_t smem = (size_t)DEC_WARPS * (a.hd + PART_PAD) * 4;
    if (a.dtype == S2S_F16) {
      if (a.hd == 128) ld_attn_only_kernel<__half, 128><<<grid, DEC_THREADS, smem, st>>>(p);
      else ld_attn_only_kernel<__half, 64><<<grid, DEC_THREADS, smem, st>>>(p);
    } else {
      if (a.hd == 128) ld_attn_only_kernel<__nv_bfloat16, 128><<<grid, DEC_THREADS, smem, st>>>(p);
      else ld_attn_only_kernel<__nv_bfloat16, 64><<<grid, DEC_THREADS, smem, st>>>(p);
    }
    S2S_LAUNCH_CHECK();
    S2S_CHECK_CUDA(cudaMemcpyAsync(cnt.data(), p.attn_cnt, (size_t)BH * 4, cudaMemcpyDeviceToHost, st));
    S2S_CHECK_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < BH; ++i)   // the decode launch reuses the counters in its next attention phase
      S2S_REQUIRE(cnt[i] == 0u, "s2s_decode_attention: split counter of (session %d, head %d) left at %u", i / a.heads,
                  i % a.heads, cnt[i]);
    return S2S_OK;
  };
  const int rc = run();
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  return rc;
}
