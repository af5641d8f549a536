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
// Qwen3 family (qk_norm, transformers modeling_qwen3.py Qwen3Attention): phase 0 stores RAW q / k; the per-head
// RMSNorm(head_dim) + RoPE is folded into the attention items of phase 1 (ld_qk_prepare), so the phase count stays 5 per
// layer (a sixth phase would add one grid barrier per layer and step to the TTS frame loop).
// Projections are swap-AB tensor-core GEMVs (sessions on m) fed from per-warp bulk-copy rings of fragment-major weights
// (decode_common.cuh, weight_tiles.cu); HBM-bound: 15.0 GB / token for Llama-3-8B (SURVEY.md Appendix A).
#include <algorithm>

#include "llama_decode.cuh"
#include "decode_common.cuh"

namespace {

__device__ __forceinline__ unsigned long long gtimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

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
  const int plan = attn_plan(BH, n_blocks, p.s_max, (int)gridDim.x);
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
    if (wl) {
      attend_blocks<T, HD>(q, Kb, Kb + p.kv_which_stride, kvd, kvd, len, blk0, blk1, 1, rec_s + warp * REC);
      attn_finish_item<T, HD>(rec_s + warp * REC, 1, part_bh, s, S, p.attn_cnt + bh, out16);
      __syncwarp();
    } else {
      attend_blocks<T, HD>(q, Kb, Kb + p.kv_which_stride, kvd, kvd, len, blk0 + warp, blk1, DEC_WARPS, rec_s + warp * REC);
      __syncthreads();
      if (warp == 0) attn_finish_item<T, HD>(rec_s, DEC_WARPS, part_bh, s, S, p.attn_cnt + bh, out16);
      __syncthreads();
    }
  }
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

template <typename T>
__device__ __noinline__ void ld_select(const LlamaDecParams& p, int step, float* s_aux) {
  const int d = p.d, B = p.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* s_feed = reinterpret_cast<int*>(s_aux);
#pragma unroll 1
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    if (warp == 0) {
      float bv = -INFINITY; int bi = 0x7fffffff;
      if (ld_has_head(p, step)) {
#pragma unroll 1
        for (int c = lane; c < (int)gridDim.x; c += 32) {
          const float v = __ldcg(p.cand_val + b * gridDim.x + c); const int i = __ldcg(p.cand_idx + b * gridDim.x + c);
          if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
      } else {
        bi = p.first_ids[b];  // multi-table mode, step 0: nothing predicted, the known first id is fed
      }
      if (lane == 0) {
        int tok = bi;
        const bool was_done = p.done[b] != 0;
        if (was_done) tok = p.eos;
        p.out_ids[b * p.n_steps + step] = tok;
        if (!was_done && !p.forced) {
          if (tok == p.eos) { p.done[b] = 1; p.out_len[b] = step + 1; atomicAdd(p.n_done, 1); }
          else if (step == p.n_steps - 1) { p.out_len[b] = p.n_steps; }
        }
        if (p.forced && step == p.n_steps - 1) p.out_len[b] = p.n_steps;
        *s_feed = p.forced ? p.forced[b * p.n_steps + step] : tok;
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

template <typename T>
__device__ __forceinline__ bool ld_gemv_args(const LlamaDecParams& p, int step, int ph, GemvArgs& a) {
  const int d = p.d, B = p.B, qd = p.heads * p.hd, kvd = p.kv_heads * p.hd;
  a.K = d; a.mode = EPI_STORE; a.out = p.q; a.ldo = qd; a.out_h = nullptr; a.ldh = 0; a.d = d; a.kv0 = nullptr; a.kv_which = 0; a.kv_batch = 0;
  a.suppress = nullptr; a.first_step = 0; a.logits_out = nullptr; a.logits_ld = 0; a.bias = nullptr; a.W = nullptr; a.N = 0;
  a.pos = p.pos; a.slot = p.slot; a.kv_slot = p.kv_slot_stride; a.kv_ld = kvd; a.rope = p.rope; a.hd = p.hd;
  a.q_rows = qd; a.k_rows = kvd; a.q_scale = rsqrtf((float)p.hd); a.kraw = nullptr; a.plan_id = -1;
  a.xsrc = nullptr; a.xsrc_ld = 0; a.kc = 0;
  const int kind = ld_kind(p, ph);
  if (kind < 6) {
    const int layer = ph / ld_nsub(p);
    const LlamaDecLayer& w = p.lw[layer];
    switch (kind) {
      case 0:
        a.W = w.w_qkv; a.N = qd + 2 * kvd; a.mode = EPI_QKV_ROPE; a.out = p.q; a.ldo = qd; a.plan_id = 0;
        a.kv0 = reinterpret_cast<T*>(p.kv) + (long long)layer * p.kv_layer_stride; a.kv_which = p.kv_which_stride;
        a.kraw = p.qk_norm ? p.kraw : nullptr;
        return true;
      case 2: a.W = w.w_o; a.N = d; a.K = qd; a.mode = EPI_RESID; a.out = p.x; a.ldo = d; a.plan_id = 1; return true;
      case 3: a.W = w.w_gu; a.N = 2 * p.ffn; a.mode = EPI_SWIGLU; a.out_h = p.h; a.ldh = p.ffn; a.plan_id = 2; return true;
      case 4:
        a.W = w.w_down; a.N = d; a.K = p.ffn; a.mode = EPI_RESID; a.out = p.x; a.ldo = d; a.plan_id = 3;
        if (p.down_kc > 0) { a.xsrc = p.h; a.xsrc_ld = p.ffn; a.kc = p.down_kc; a.plan_id = -1; }
        return true;
      default: return false;
    }
  }
  if (kind == 6 && ld_has_head(p, step)) {
    a.W = ld_multi(p) ? reinterpret_cast<const T*>(p.lm_head) + (long long)(step - 1) * p.head_stride : p.lm_head;
    a.N = p.vocab; a.mode = EPI_LOGITS; a.plan_id = 4; a.suppress = p.suppress;
    a.logits_out = p.logits_out ? p.logits_out + (long long)step * B * p.vocab : nullptr; a.logits_ld = p.vocab;
    return true;
  }
  return false;
}

template <typename T>
struct LdSmem {
  T* xh; float* xs; float* sv; int* si; float* s_red; float* wb; float4* red;
};

__host__ __device__ inline int ld_kmax(int d, int ffn, int qd) { return (d > ffn ? d : ffn) > qd ? (d > ffn ? d : ffn) : qd; }

template <typename T>
__device__ __forceinline__ void ld_phase(const LlamaDecParams& p, int step, int ph, const LdSmem<T>& sm, GemvRing& ring,
                                         GemvArgs* ready, GemvArgs& a_scratch, int wb_ready) {
  const int d = p.d, B = p.B;
  float best_v[2] = {-INFINITY, -INFINITY};
  int best_i[2] = {0x7fffffff, 0x7fffffff};
  // argument struct and ring state live in shared memory (all threads write identical values), not on the stack
  const int kind = ld_kind(p, ph);
  if (!ready && ld_has_gemv(p, step, ph)) {
    if (threadIdx.x == 0) ld_gemv_args<T>(p, step, ph, a_scratch);  // one thread writes the shared struct
    __syncthreads();
  }
  GemvArgs& a = ready ? *ready : a_scratch;
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
        if (a.kc > 0) { gemv_mma_chunked<T, true>(a, sm.xh, B, best_v, best_i, ring, sm.red); return; }
        stage_rows_copy<T>(reinterpret_cast<const T*>(p.h), B, p.ffn, sm.xh); break;
    }
    gemv_mma<T, true>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
    return;
  }
  if (kind == 6) {
    if (p.hidden_out && blockIdx.x == 0)  // the residual stream before the final norm (Qwen3-TTS: input of the code predictor)
      for (int i = threadIdx.x; i < B * d; i += DEC_THREADS) p.hidden_out[(long long)step * B * d + i] = __ldcg(p.x + i);
    stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 2, p.norm_f, nullptr, p.eps, sm.s_red, sm.wb, wb_ready, p.norm_rg);
    gemv_mma<T, true>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
    gemv_argmax_candidates(best_v, best_i, B, sm.sv, sm.si, p.cand_val, p.cand_idx);
  } else {
    ld_select<T>(p, step, sm.sv);
  }
}

template <typename T>
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
  LdSmem<T> sm;
  sm.xh = reinterpret_cast<T*>(smem_raw);
  sm.xs = reinterpret_cast<float*>(smem_raw + lay.xs_off);
  sm.sv = reinterpret_cast<float*>(smem_raw + lay.aux_off);
  sm.si = reinterpret_cast<int*>(smem_raw + lay.si_off);
  sm.s_red = reinterpret_cast<float*>(smem_raw + lay.red_s_off);
  sm.wb = reinterpret_cast<float*>(smem_raw + lay.wb_off);
  sm.red = reinterpret_cast<float4*>(smem_raw + lay.redbuf_off);
  GemvRing& ring = s_rings[threadIdx.x >> 5];
  {
    unsigned char* rb = smem_raw + lay.ring_off;
    const int warp = threadIdx.x >> 5;
    uint64_t* bars = reinterpret_cast<uint64_t*>(rb + (size_t)DEC_WARPS * p.ring_slots * GV_SLOT_BYTES) + warp * p.ring_slots;
    if ((threadIdx.x & 31) == 0) {   // lane 0 owns the warp's ring state in shared memory
      ring.slots = p.ring_slots;
      ring.base_s = smem_u32(rb + (size_t)warp * p.ring_slots * GV_SLOT_BYTES);
      ring.bars_s = smem_u32(bars);
      ring.slot = 0;
      ring.parity = 0;
      ring.plans_s = s_plans;
      ring.pre_valid = 0; ring.pre_pj = 0; ring.pre_pu = 0; ring.pre_nvalid = 0; ring.pre_W = nullptr;
      for (int i = 0; i < p.ring_slots; ++i) mbar_init(bars + i, 1);
      fence_barrier_init();
    }
    __syncthreads();
  }
  unsigned int epoch = 0;
  int trace_i = 0;
  GemvArgs& pre_args = s_args[0];
  if (threadIdx.x == 0) pre_args.K = p.d;
  int pre_tag = -1, wb_tag = -1;
  const int n_ph = ld_nsub(p) * p.layers + 2;
  for (int step = step_begin; step < step_end; ++step) {
    const int pb = coop ? 0 : ph_begin, pe = coop ? n_ph : ph_end;
    for (int ph = pb; ph < pe; ++ph) {
      const bool tracing = sp.trace && trace_i < sp.trace_cap && threadIdx.x == 0 && blockIdx.x == 0;
      unsigned long long* tr = tracing ? sp.trace + (long long)trace_i * 3 : nullptr;
      if (tracing) tr[0] = gtimer_ns();
      const bool skip = ld_kind(sp, ph) == 6 && !ld_has_head(sp, step);  // nothing to predict: no work, no barrier
      if (!skip) ld_phase<T>(sp, step, ph, sm, ring, (pre_tag == step * n_ph + ph) ? &pre_args : nullptr, s_args[1], wb_tag == step * n_ph + ph);
      if (tracing) tr[1] = gtimer_ns();
      if (coop && !skip) {
        grid_arrive(p.sync_counter, epoch);
        // ---- between arrive and wait: prepare the next projection (arguments, first weight units, norm weights) ----
        if (!ring.pre_valid) {
          int nph = ph + 1, nstep = step;
          if (nph == n_ph) { nph = 0; nstep = step + 1; }
#pragma unroll 1
          for (int look = 0; look < 3 && nstep < step_end; ++look) {
            if (ld_has_gemv(sp, nstep, nph)) {
              if (threadIdx.x == 0) ld_gemv_args<T>(sp, nstep, nph, pre_args);  // one thread writes the shared struct
              __syncthreads();
              if (pre_args.kc == 0) gemv_prefetch<T>(pre_args, ring);   // a K-chunked projection starts its own stream
              pre_tag = nstep * n_ph + nph;
              const float* nw = nullptr;
              const int nk = ld_kind(sp, nph);
              if (nk == 0) nw = sp.lw[nph / ld_nsub(sp)].norm1; else if (nk == 3) nw = sp.lw[nph / ld_nsub(sp)].norm2;
              else if (nk == 6) nw = sp.norm_f;
              if (nw && wb_tag != pre_tag) { stage_norm_weights(nw, nullptr, sp.d, sm.wb); wb_tag = pre_tag; }
              break;
            }
            if (++nph == n_ph) { nph = 0; ++nstep; }
          }
        }
        grid_wait(p.sync_counter, epoch, p.sync_relaxed);
      }
      if (tracing) tr[2] = gtimer_ns();
      ++trace_i;
    }
    if (coop && !p.forced && *reinterpret_cast<volatile int*>(p.n_done) >= p.B) break;
  }
  gemv_drain(pre_args.K, ring);
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
  if (threadIdx.x == 0) {
    p.done[b] = 0;
    p.out_len[b] = 0;
    if (b == 0) { *p.n_done = 0; *p.sync_counter = 0; }
    for (int h = 0; h < p.heads; ++h) p.attn_cnt[b * p.heads + h] = 0u;
  }
  for (int i = threadIdx.x; i < p.n_steps; i += blockDim.x) p.out_ids[b * p.n_steps + i] = p.eos;
}

template <typename T>
int launch_t(s2s_ctx* ctx, const LlamaDecParams& p, int debug_phases, cudaStream_t stream) {
  int kmax = 0, rg = 0, kc = 0, slots = 0;
  int grid = dec_grid(ctx);                          // the context's SM partition (s2s_set_sm_partition)
  if (const char* e = getenv("S2S_DECODE_CTAS")) {   // developer knob: override for experiments (tests/dev/dev_lanes.py)
    const int v = atoi(e);
    if (v >= 8 && v < ctx->num_sms) grid = v;
  }
  S2S_REQUIRE(llama_decode_plan(p.B, p.d, p.ffn, p.heads * p.hd, grid, &kmax, &rg, &kc, &slots),
              "llama decode: batch %d does not fit shared memory for d %d, ffn %d", p.B, p.d, p.ffn);
  const DecSmem lay = dec_smem_layout(p.B, p.d, kmax, p.d, rg);
  LlamaDecParams pr = p;
  pr.sync_relaxed = dec_sync_relaxed_env();
  pr.ring_slots = slots; pr.norm_rg = rg; pr.down_kc = kc;
  const size_t smem = (size_t)lay.ring_off + (size_t)DEC_WARPS * pr.ring_slots * (GV_SLOT_BYTES + 8) + 128;
  auto kern = llama_decode_kernel<T>;
  S2S_CHECK_CUDA(s2s_opt_in_max_smem(kern, ctx->device, smem, nullptr));
  llama_decode_init_kernel<T><<<p.B, 256, 0, stream>>>(pr);
  S2S_LAUNCH_CHECK();
  const int n_ph = ld_nsub(p) * p.layers + 2;
  if (!debug_phases) {
    int sb = 0, se = p.n_steps, pb = 0, pe = n_ph, coop = 1;
    LlamaDecParams pp = pr;
    void* args[] = {&pp, &sb, &se, &pb, &pe, &coop};
    S2S_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(DEC_THREADS), args, smem, stream));
    s2s_count_launch();
  } else {
    for (int s = 0; s < p.n_steps; ++s)
      for (int ph = 0; ph < n_ph; ++ph) {
        if (ph == n_ph - 2 && pr.head_stride != 0 && s == 0) continue;  // multi-table mode: step 0 predicts nothing
        kern<<<grid, DEC_THREADS, smem, stream>>>(pr, s, s + 1, ph, ph + 1, 0);
        S2S_LAUNCH_CHECK();
      }
  }
  return S2S_OK;
}

}  // namespace

int llama_decode_launch(s2s_ctx* ctx, const LlamaDecParams& p, int dtype, int debug_phases, cudaStream_t stream) {
  S2S_REQUIRE(p.hd == 64 || p.hd == 128, "llama decode: head_dim must be 64 or 128");
  S2S_REQUIRE(p.layers <= 64, "llama decode: at most 64 layers");
  S2S_REQUIRE(p.n_steps >= 1, "llama decode: n_steps must be >= 1");
  S2S_REQUIRE(p.B >= 1 && p.B <= DEC_MAX_B, "llama decode: batch %d > %d must be split by the caller", p.B, DEC_MAX_B);
  S2S_REQUIRE(p.d % 64 == 0 && p.ffn % 64 == 0 && (p.heads * p.hd) % 64 == 0, "llama decode: d, ffn, heads*hd must be multiples of 64");
  if (dtype == S2S_BF16) return launch_t<__nv_bfloat16>(ctx, p, debug_phases, stream);
  if (dtype == S2S_F16) return launch_t<__half>(ctx, p, debug_phases, stream);
  s2s_set_error("llama decode: unsupported dtype %d", dtype);
  return S2S_ERR_UNSUPPORTED;
}

// Shared-memory plan of a batch.  Preferred: everything staged whole in one round trip (rg = B, kc = 0).  When that does not
// leave two ring slots per warp: stage the ffn-wide down-projection operand in K-chunks of max(d, qd) columns and walk the
// fp32 statistics copy in row groups (largest power of two that fits) -- Llama-3-8B: 4 sessions whole, 8 with chunks.
bool llama_decode_plan(int B, int d, int ffn, int qd, int grid, int* kmax, int* rg, int* kc, int* ring_slots) {
  {
    const int km = ld_kmax(d, ffn, qd);
    const int s = dec_ring_slots(dec_smem_layout(B, d, km, d, B));
    if (s >= 2) { *kmax = km; *rg = B; *kc = 0; *ring_slots = s; return true; }
  }
  const int lim = ((std::max(d, qd) + 255) / 256) * 256;     // chunk = the widest operand that is staged whole anyway
  if (ffn <= lim || !gemv_chunk_ok(d, ffn, lim, grid)) return false;
  const int km = ld_kmax(d, lim, qd);
  for (int g = B; g >= 2; g >>= 1) {
    int gg = 1;
    while (gg * 2 <= g) gg *= 2;
    const int s = dec_ring_slots(dec_smem_layout(B, d, km, d, gg));
    if (s >= 2) { *kmax = km; *rg = gg; *kc = lim; *ring_slots = s; return true; }
  }
  return false;
}

int llama_decode_max_batch(int d, int ffn, int qd, int grid) {
  int kmax, rg, kc, slots;
  for (int B = DEC_MAX_B; B >= 1; --B)
    if (llama_decode_plan(B, d, ffn, qd, grid, &kmax, &rg, &kc, &slots)) return B;
  return 0;
}
