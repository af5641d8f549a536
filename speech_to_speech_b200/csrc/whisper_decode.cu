// whisper_decode.cu -- the whole Whisper greedy decode loop as ONE persistent cooperative kernel.
//
// Reference path: WhisperGenerationMixin.generate short-form greedy (transformers generation_whisper.py:383-968)
// over WhisperDecoder (modeling_whisper.py:691-797, layer :449-507) with the tied proj_out (:1081),
// SuppressTokens / SuppressTokensAtBegin processors (generation_whisper.py:1774-1813) and EOS stop.  The
// reference launches ~10 tiny kernels per layer per token and syncs with the host every token for the EOS
// check; here the host launches once per utterance batch and reads the ids at the end.
//
// One CTA per SM (132 on an H100), 256 threads, 1-16 sessions per launch.  A token step is a fixed sequence of phases separated by
// a grid barrier:
//   per layer  0: LN1 + QKV projection (+ self-KV append)   1: self-attention items (32-key blocks, last split merges)
//              2: out-projection + residual                 3: LN2 + cross-q projection
//              4: cross-attention items over 1500 keys      5: out-projection + residual
//              6: LN3 + fc1 + GELU                          7: fc2 + residual
//   then       8L: final LN + tied logits projection + suppress masks + per-CTA argmax
//              8L+1: global argmax, EOS / length bookkeeping, next-token embedding
// Projections are swap-AB tensor-core GEMVs fed from per-warp bulk-copy weight rings (decode_common.cuh); the kernel is
// HBM/latency-bound (decoder weights once per step for the whole batch + per-session cross-KV; SURVEY.md Appendix A).
// A second kernel in this file (whisper_decode_cluster_kernel) serves single sessions with one thread-block cluster per
// attention head and four grid-wide phases per layer.
#include <algorithm>

#include "whisper_decode.cuh"
#include "decode_common.cuh"

// Dynamic shared memory the 8-phase kernel's plans are made against: a fixed 220 KB (below the device limit), so that the
// batch per launch -- and with it the attention split plans and the ids -- does not depend on the kernel's static size.
constexpr long long WD_SMEM_BUDGET = 220LL * 1024 - 128;

namespace {

constexpr int HD = 64;
static_assert(ATT_CHUNK == ATT_CHUNK_KEYS, "chunk size mismatch");

// L2 prefetch of what this warp will read first in the NEXT phase: its first cross-attention block (called
// between grid_arrive and grid_wait).
template <typename T>
__device__ __noinline__ void wd_prefetch(const WhisperDecParams& p, int step, int ph) {
  const int L = p.layers;
  if (ph < 8 * L && (ph & 7) == 4) {
    const int BH = p.B * p.heads, n_blocks = (p.n_ctx + ATT_BLK - 1) / ATT_BLK;
    const int S = p.cross_plan & 0x7f, bps = (n_blocks + S - 1) / S;
    const bool wl = p.cross_plan & ATTN_WARP_LEVEL;
    const int it = wl ? dec_first_item() : (int)blockIdx.x;
    if (it < BH * S) {
      const int s = it % S, bh = it / S, h = bh % p.heads, b = bh / p.heads;
      const int blk = s * bps + (wl ? 0 : (int)(threadIdx.x >> 5));
      if (blk < min((s + 1) * bps, n_blocks)) {
        const long long head_elems = (long long)p.n_ctx * HD;
        const T* Kb = reinterpret_cast<const T*>(p.cross_kv) +
                      (((long long)b * L + (ph >> 3)) * 2 * p.heads + h) * head_elems + (long long)blk * ATT_BLK * HD;
        const int n_keys = min(ATT_BLK, p.n_ctx - blk * ATT_BLK);
        prefetch_strided_l2(Kb, HD * (long long)sizeof(T), n_keys, HD * (int)sizeof(T));
        prefetch_strided_l2(Kb + p.heads * head_elems, HD * (long long)sizeof(T), n_keys, HD * (int)sizeof(T));
      }
    }
  }
}

// One attention phase over `n_keys` keys of every (session, head), cut into items by `plan` (attn_plan).
// Kbase(b, h) / the K->V offset / the row stride describe the cache; rec_s: DEC_WARPS records of shared memory.
template <typename T>
__device__ __forceinline__ void wd_attn_items(const WhisperDecParams& p, int plan, int n_keys, const T* kv0, long long b_stride,
                                              long long h_stride, long long v_off, long long ld, float* rec_s) {
  const int d = p.d, H = p.heads;
  constexpr int REC = HD + PART_PAD;
  const int n_blocks = (n_keys + ATT_BLK - 1) / ATT_BLK, BH = p.B * H;
  const int S = plan & 0x7f, bps = (n_blocks + S - 1) / S;
  const bool wl = plan & ATTN_WARP_LEVEL;
#pragma unroll 1
  for (int it = wl ? dec_first_item() : (int)blockIdx.x; it < BH * S; it += wl ? dec_item_stride() : (int)gridDim.x) {
    const int s = it % S, bh = it / S, h = bh % H, b = bh / H;
    const T* Kb = kv0 + b * b_stride + h * h_stride;
    attn_run_item<T, HD>(wl, p.q + b * d + h * HD, Kb, Kb + v_off, ld, n_keys, s * bps, min((s + 1) * bps, n_blocks), rec_s,
                         p.part + (long long)bh * p.s_max * REC, s, S, p.attn_cnt + bh, reinterpret_cast<T*>(p.attn16) + (long long)b * d + h * HD);
  }
}

// self-attention over the pos + 1 cached keys: cache [b][layer][k|v][pos][d]
template <typename T>
__device__ __noinline__ void wd_self_attn(const WhisperDecParams& p, int layer, int pos, float* rec_s) {
  const long long kvs = (long long)p.max_pos * p.d;
  const T* kv0 = reinterpret_cast<const T*>(p.self_kv) + (long long)layer * 2 * kvs;
  wd_attn_items<T>(p, p.self_plan[(pos + ATT_BLK) / ATT_BLK], pos + 1, kv0, (long long)p.layers * 2 * kvs, HD, kvs, p.d, rec_s);
}

// cross-attention over the n_ctx encoder positions: cache [b][layer][k|v][head][t][64]
template <typename T>
__device__ __noinline__ void wd_cross_attn(const WhisperDecParams& p, int layer, float* rec_s) {
  const long long head_elems = (long long)p.n_ctx * HD;
  const T* kv0 = reinterpret_cast<const T*>(p.cross_kv) + (long long)layer * 2 * p.heads * head_elems;
  wd_attn_items<T>(p, p.cross_plan, p.n_ctx, kv0, (long long)p.layers * 2 * p.heads * head_elems, head_elems,
                   p.heads * head_elems, HD, rec_s);
}

// global argmax, EOS / length bookkeeping, next-token embedding
template <typename T>
__device__ __noinline__ void wd_select(const WhisperDecParams& p, int g, int pos, float* s_aux) {
  const int d = p.d, B = p.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* s_feed = reinterpret_cast<int*>(s_aux);
#pragma unroll 1
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    if (warp == 0) {
      if (g >= 0) {
        // bookkeeping operands first: their round trips overlap the candidate loads
        const int was_done = p.done[b];
        const int forced_tok = p.forced ? p.forced[b * p.max_new + g] : 0;
        const int tok = dec_argmax_merge(p.cand_val, p.cand_idx, b);
        if (lane == 0) {
          const int feed = dec_record_token(p, b, g, p.max_new, tok, was_done, forced_tok);
          if (pos + 1 < p.max_pos) p.tokens[b * p.max_pos + pos + 1] = feed;
          *s_feed = feed;
        }
      } else if (lane == 0) {
        *s_feed = p.tokens[b * p.max_pos + pos + 1];
      }
    }
    __syncthreads();
    const int feed = *s_feed;
    if (pos + 1 < p.max_pos) {
      const T* e = reinterpret_cast<const T*>(p.embed);
      const float* pe = p.pos + (long long)(pos + 1) * d;
#pragma unroll 2
      for (int i = threadIdx.x; i < d; i += DEC_THREADS) p.x[b * d + i] = DT<T>::to_f(e[gv_tiled_elem(feed, i, d)]) + pe[i];
    }
  }
}

// The 8-phase kernel's phases for dec_run (decode_common.cuh).  Holds a reference to the kernel's shared copy of the parameters.
template <typename T>
struct WdModel {
  static constexpr bool stamps_barrier = true;
  static constexpr bool f8_weights = false;
  const WhisperDecParams& p;
  int n_phases;

  // the logits phase is skipped while the forced prompt is still being fed
  __device__ __forceinline__ bool skip(int step, int ph) const { return ph == 8 * p.layers && step < p.n_prefix - 1; }
  // pure predicate: the argument struct lives in shared memory and is written by ONE thread, so nobody may call gemv_args
  // just to find out
  __device__ __forceinline__ bool has_gemv(int step, int ph) const {
    if (ph < 8 * p.layers) return (ph & 7) != 1 && (ph & 7) != 4;
    return ph == 8 * p.layers && step >= p.n_prefix - 1;
  }
  __device__ __forceinline__ bool lookahead_target(int step, int ph) const { return has_gemv(step, ph); }
  __device__ __forceinline__ void prefetch_l2(int step, int ph) const { wd_prefetch<T>(p, step, ph); }
  __device__ __forceinline__ DecNorm norm_of(int ph) const {
    if (ph >= 8 * p.layers) return {p.lnf_w, p.lnf_b};
    const WhisperDecLayer& w = p.lw[ph >> 3];
    const int sub = ph & 7;
    if (sub == 0) return {w.ln1_w, w.ln1_b};
    if (sub == 3) return {w.ln2_w, w.ln2_b};
    if (sub == 6) return {w.ln3_w, w.ln3_b};
    return {nullptr, nullptr};
  }

  // arguments of the projection GEMV of phase `ph` (has_gemv): shared by the phase itself and by the look-ahead
  __device__ __forceinline__ void gemv_args(int step, int ph, GemvArgs& a) const {
    const int L = p.layers, pos = step, d = p.d, B = p.B;
    gemv_args_reset(a, d, p.q);
    a.plan_id = 1;
    if (ph < 8 * L) {
      const int layer = ph >> 3;
      const WhisperDecLayer& w = p.lw[layer];
      switch (ph & 7) {
        case 0: {
          const long long kvs = (long long)p.max_pos * d;
          a.W = w.w_qkv; a.N = 3 * d; a.bias = w.b_qkv; a.mode = EPI_QKV; a.out = p.q; a.plan_id = 0;
          a.kv0 = reinterpret_cast<T*>(p.self_kv) + ((long long)layer * 2) * kvs + (long long)pos * d;
          a.kv_which = kvs; a.kv_batch = (long long)L * 2 * kvs;
        } return;
        case 2: a.W = w.w_o; a.N = d; a.bias = w.b_o; a.mode = EPI_RESID; a.out = p.x; return;
        case 3: a.W = w.w_cq; a.N = d; a.bias = w.b_cq; a.mode = EPI_STORE; a.out = p.q; return;
        case 5: a.W = w.w_co; a.N = d; a.bias = w.b_co; a.mode = EPI_RESID; a.out = p.x; return;
        case 6: a.W = w.w_fc1; a.N = p.ffn; a.bias = w.b_fc1; a.mode = EPI_GELU; a.out_h = p.h; a.ldh = p.ffn; a.plan_id = 2; return;
        case 7: a.W = w.w_fc2; a.N = d; a.K = p.ffn; a.bias = w.b_fc2; a.mode = EPI_RESID; a.out = p.x; a.plan_id = 3; return;
        default: return;
      }
    }
    const int g = step - (p.n_prefix - 1);
    if (ph == 8 * L && g >= 0) {
      a.W = p.embed; a.N = p.vocab; a.mode = EPI_LOGITS; a.plan_id = 4; a.suppress = p.suppress; a.first_step = (g == 0);
      a.logits_out = p.logits_out ? p.logits_out + (long long)g * B * p.vocab : nullptr; a.logits_ld = p.vocab;
    }
  }

  // One phase = (stage inputs into shared memory) + (one shared routine).  Thin: only argument setup is inlined.
  __device__ __forceinline__ void phase(int step, int ph, const DecViews<T>& sm, GemvRing& ring, GemvArgs* ready,
                                        GemvArgs* scratch, int wb_ready, unsigned long long* tr) const {
    const int L = p.layers, pos = step, d = p.d, B = p.B;
    float best_v[2] = {-INFINITY, -INFINITY};
    int best_i[2] = {0x7fffffff, 0x7fffffff};
    // argument struct and ring state live in SHARED memory (one thread writes): per-thread copies on the stack
    // (256 x ~300 B) do not fit the small L1 left next to the weight rings and turned into L2 traffic
    if (!ready && has_gemv(step, ph)) {
      if (threadIdx.x == 0) gemv_args(step, ph, *scratch);  // one thread writes, everybody reads after the barrier
      __syncthreads();
    }
    GemvArgs& a = ready ? *ready : *scratch;
    if (ph < 8 * L) {
      const int layer = ph >> 3;
      const WhisperDecLayer& w = p.lw[layer];
      switch (ph & 7) {
        case 0: stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, w.ln1_w, w.ln1_b, 1e-5f, sm.s_red, sm.wb, wb_ready); break;
        case 1: wd_self_attn<T>(p, layer, pos, reinterpret_cast<float*>(sm.red)); return;
        case 2: stage_rows_copy<T>(reinterpret_cast<const T*>(p.attn16), B, d, sm.xh); break;
        case 3: stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, w.ln2_w, w.ln2_b, 1e-5f, sm.s_red, sm.wb, wb_ready); break;
        case 4: wd_cross_attn<T>(p, layer, reinterpret_cast<float*>(sm.red)); return;
        case 5: stage_rows_copy<T>(reinterpret_cast<const T*>(p.attn16), B, d, sm.xh); break;
        case 6: stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, w.ln3_w, w.ln3_b, 1e-5f, sm.s_red, sm.wb, wb_ready); break;
        default: stage_rows_copy<T>(reinterpret_cast<const T*>(p.h), B, p.ffn, sm.xh); break;
      }
      if (tr) tr[1] = dec_clock_ns();  // inputs staged
      gemv_mma<T, false>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      return;
    }
    if (ph == 8 * L) {
      // final LayerNorm + tied output projection + suppress masks + per-CTA argmax candidates
      stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, p.lnf_w, p.lnf_b, 1e-5f, sm.s_red, sm.wb, wb_ready);
      gemv_mma<T, false>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      gemv_argmax_candidates(best_v, best_i, B, sm.sv, sm.si, p.cand_val, p.cand_idx);
    } else {
      wd_select<T>(p, step - (p.n_prefix - 1), pos, sm.sv);
    }
  }
};

template <typename T>
__global__ void __launch_bounds__(DEC_THREADS, 1)
whisper_decode_kernel(const WhisperDecParams p, int step_begin, int step_end, int ph_begin, int ph_end, int coop) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ WhisperDecParams sp;
  __shared__ WhisperDecLayer s_layers[32];  // per-layer pointer tables: no global pointer chase inside a phase
  __shared__ GemvPlan s_plans[5];           // qkv [3d,d] | [d,d] | fc1 [ffn,d] | fc2 [d,ffn] | logits [vocab,d]
  __shared__ GemvArgs s_args[2];            // [0] prepared for the next projection, [1] built in-phase
  __shared__ GemvRing s_rings[DEC_WARPS];   // per-warp ring state
  if (threadIdx.x < 5) {
    const int i = threadIdx.x;
    gemv_make_plan(i == 0 ? 3 * p.d : i == 2 ? p.ffn : i == 4 ? p.vocab : p.d, i == 3 ? p.ffn : p.d, s_plans[i]);
  }
  if (threadIdx.x == 0) { sp = p; sp.lw = s_layers; }
  for (int i = threadIdx.x; i < p.layers; i += DEC_THREADS) s_layers[i] = p.lw[i];
  __syncthreads();
  const DecSmem lay = dec_smem_layout(p.B, p.d, max(p.d, p.ffn), 2 * p.d);
  GemvRing& ring = s_rings[threadIdx.x >> 5];
  gemv_ring_init(ring, smem_raw + lay.ring_off, p.ring_slots, s_plans);
  const WdModel<T> model{sp, 8 * p.layers + 2};
  // the loop reads the shared copy here (the kernel parameter costs this kernel ~20 registers; the other two prefer it)
  dec_run<T>(sp, model, dec_views<T>(smem_raw, lay), ring, s_args, step_begin, step_end, ph_begin, ph_end, coop);
}

// =====================================================================================================================
// Cluster variant for 1-2 sessions per launch: FOUR grid-wide phases per layer instead of eight.
//
// At batch 1 the step time is the number of grid-wide dependency hops (grid barrier + L2 round trip),
// not bytes.  Launched with thread-block clusters of CS CTAs, one cluster per attention head, the chain
//   LN + q/k/v rows of the head -> attention of the head -> the head's slice of the out-projection
// never leaves the cluster: its two internal hand-offs use barrier.cluster (hardware) + L2 instead of the
// grid barrier.  Each head leaves a PARTIAL out-projection [B, d] (its 64 columns of W_o); the next phase sums the
// H partials in fixed order while staging its input (stage_rows_norm_sum: deterministic, no atomics), and one CTA
// writes the summed residual stream back for the later phases:
//   phase 4l+0  self block : LN1(X0)                         -> qkv_h | barrier.cluster | attention_h | barrier.cluster | P0[h] = W_o[:, h] o_h
//   phase 4l+1  cross block: x1 = X0 + b_o + sum P0 -> X1, LN2 -> cq_h  | barrier.cluster | cross-attn_h | barrier.cluster | P1[h] = W_co[:, h] o_h
//   phase 4l+2  fc1        : x2 = X1 + b_co + sum P1 -> X0, LN3 -> fc1 + GELU            (whole grid)
//   phase 4l+3  fc2        : X0 += fc2(h)                                                 (whole grid)
//   then logits and select as in the 8-phase kernel.  Clusters beyond the H heads idle in the block phases.
// =====================================================================================================================
__device__ __forceinline__ unsigned int cluster_ctarank() {
  unsigned int r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned int cluster_id_x() {
  unsigned int r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned int cluster_nctaid_x() {
  unsigned int r;
  asm volatile("mov.u32 %0, %%cluster_nctaid.x;" : "=r"(r));
  return r;
}
// all threads of all CTAs of the cluster; release/acquire at cluster scope covers the global-memory hand-offs
// ONE thread publishes the CTA's writes (bar.sync + fence by thread 0: cumulative, like grid_arrive); the hardware barrier
// itself is relaxed -- barrier.cluster.arrive.release makes EVERY thread execute MEMBAR.ALL.GPU, which serialises
// with 256 threads.  Readers use L2 accesses (ld.global.cg) after the wait.
__device__ __forceinline__ void cluster_barrier() {
  __syncthreads();
  if (threadIdx.x == 0) asm volatile("fence.acq_rel.gpu;" ::: "memory");
  asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
  // acquire side, mirrored: one fencing thread, then the CTA barrier extends the order to the others
  if (threadIdx.x == 0) asm volatile("fence.acq_rel.gpu;" ::: "memory");
  __syncthreads();
}

struct WdcCtx { int cid, rank, cs; };

// the head's 64-column slice of an out-projection: partial[h][b][row] = sum_{k < 64} W[row][64 h + k] * o_h[b][k]
__device__ __forceinline__ void wdc_out_args(const WhisperDecParams& p, const WdcCtx& cx, int layer, bool cross, GemvArgs& a) {
  const WhisperDecLayer& w = p.lw[layer];
  a.K = HD; a.N = p.d; a.W = cross ? w.w_co : w.w_o; a.bias = nullptr; a.mode = EPI_STORE;
  a.out = (cross ? p.part_x1 : p.part_x0) + (long long)cx.cid * p.B * p.d; a.ldo = p.d; a.plan_id = 2;
}

// The cluster kernel's phases for dec_run (decode_common.cuh): the kernel's shared copy of the parameters and the cluster
// identity.  Stamps 2 and 3 of the trace are the block's intra-phase milestones: q/k/v rows done, cluster barrier 1 passed.
template <typename T>
struct WdcModel {
  static constexpr bool stamps_barrier = false;
  static constexpr bool f8_weights = false;
  const WhisperDecParams& p;
  WdcCtx cx;
  int n_phases;

  __device__ __forceinline__ bool skip(int step, int ph) const { return ph == 4 * p.layers && step < p.n_prefix - 1; }
  // false: select, or a cluster without a head
  __device__ __forceinline__ bool has_gemv(int step, int ph) const {
    if (ph < 4 * p.layers) return (ph & 3) >= 2 || cx.cid < p.heads;
    return ph == 4 * p.layers && step >= p.n_prefix - 1;
  }
  // every CTA stages its input, also clusters without a head: the look-ahead stages their norm weights
  __device__ __forceinline__ bool lookahead_target(int step, int ph) const { return !skip(step, ph) && ph != 4 * p.layers + 1; }
  __device__ __forceinline__ void prefetch_l2(int, int) const {}
  __device__ __forceinline__ DecNorm norm_of(int ph) const {
    if (ph >= 4 * p.layers) return {p.lnf_w, p.lnf_b};
    const WhisperDecLayer& w = p.lw[ph >> 2];
    const int sub = ph & 3;
    if (sub == 0) return {w.ln1_w, w.ln1_b};
    if (sub == 1) return {w.ln2_w, w.ln2_b};
    if (sub == 2) return {w.ln3_w, w.ln3_b};
    return {nullptr, nullptr};
  }

  // first projection of phase `ph` (4 per layer + logits; has_gemv)
  __device__ __forceinline__ void gemv_args(int step, int ph, GemvArgs& a) const {
    const int L = p.layers, pos = step, d = p.d, B = p.B;
    gemv_args_reset(a, d, p.q);
    if (ph < 4 * L) {
      const int layer = ph >> 2;
      const WhisperDecLayer& w = p.lw[layer];
      switch (ph & 3) {
        case 0: {
          const long long kvs = (long long)p.max_pos * d;
          a.W = w.w_qkv; a.N = 3 * d; a.bias = w.b_qkv; a.mode = EPI_QKV; a.out = p.q; a.plan_id = 0;
          a.kv0 = reinterpret_cast<T*>(p.self_kv) + ((long long)layer * 2) * kvs + (long long)pos * d;
          a.kv_which = kvs; a.kv_batch = (long long)L * 2 * kvs;
        } return;
        case 1: a.W = w.w_cq; a.N = d; a.bias = w.b_cq; a.mode = EPI_STORE; a.out = p.q; a.plan_id = 1; return;
        case 2: a.W = w.w_fc1; a.N = p.ffn; a.bias = w.b_fc1; a.mode = EPI_GELU; a.out_h = p.h; a.ldh = p.ffn; a.plan_id = 3; return;
        default: a.W = w.w_fc2; a.N = d; a.K = p.ffn; a.bias = w.b_fc2; a.mode = EPI_RESID; a.out = p.x; a.plan_id = 4; return;
      }
    }
    const int g = step - (p.n_prefix - 1);
    a.W = p.embed; a.N = p.vocab; a.mode = EPI_LOGITS; a.plan_id = 5; a.suppress = p.suppress; a.first_step = (g == 0);
    a.logits_out = p.logits_out ? p.logits_out + (long long)g * B * p.vocab : nullptr; a.logits_ld = p.vocab;
  }

  // self / cross attention block of one layer (see the comment above).  scratch: (heads + 1) * B * d floats.
  __device__ __forceinline__ void block(int step, int layer, bool cross, const DecViews<T>& sm, GemvRing& ring, GemvArgs* ready,
                                        GemvArgs* scratch /*[2]*/, int wb_ready, unsigned long long* tr) const {
    const WhisperDecLayer& w = p.lw[layer];
    const int d = p.d, B = p.B, H = p.heads, warp = threadIdx.x >> 5;
    constexpr int REC = HD + PART_PAD;
    float best_v[2] = {-INFINITY, -INFINITY};
    int best_i[2] = {0x7fffffff, 0x7fffffff};
    // A. input of the block
    if (!cross) {
      stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, w.ln1_w, w.ln1_b, 1e-5f, sm.s_red, sm.wb, wb_ready);
    } else {
      stage_rows_norm_sum<T>(p.x, p.part_x0, H, (long long)B * d, w.b_o, blockIdx.x == 0 ? p.x_alt : nullptr, B, d, sm.xs, sm.xh, 1,
                             w.ln2_w, w.ln2_b, 1e-5f, sm.s_red, sm.wb, wb_ready);
    }
    if (tr) tr[1] = dec_clock_ns();
    if (cx.cid >= H) return;  // no head for this cluster (nothing was prefetched for it: has_gemv)
    const int h = cx.cid;
    // B. the head's q (k, v) rows
    GemvArgs& a = ready ? *ready : scratch[0];
    GemvArgs& ao = scratch[1];
    if (threadIdx.x == 0) {  // ONE thread writes the shared argument structs; the barrier publishes them
      if (!ready) gemv_args(step, layer * 4 + (cross ? 1 : 0), scratch[0]);
      ao = a;
      wdc_out_args(p, cx, layer, cross, ao);
    }
    __syncthreads();
    gemv_mma<T, false>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
    if (tr) tr[2] = dec_clock_ns();
    // C. start streaming the head's out-projection slice
    gemv_prefetch<T>(ao, ring);
    // D. q (and the new k, v cache rows) of the head are visible to the whole cluster
    cluster_barrier();
    if (tr) tr[3] = dec_clock_ns();
    // E. attention: 32-key blocks over (CTA rank, warp); one record per CTA
    float* rec_s = reinterpret_cast<float*>(sm.red);
    {
      const int n_keys = cross ? p.n_ctx : step + 1;
      const int n_blocks = (n_keys + ATT_BLK - 1) / ATT_BLK;
      const long long kvs = (long long)p.max_pos * d, head_elems = (long long)p.n_ctx * HD;
#pragma unroll 1
      for (int b = 0; b < B; ++b) {
        const T* Kb; long long v_off, ld;
        if (cross) {
          Kb = reinterpret_cast<const T*>(p.cross_kv) + (((long long)b * p.layers + layer) * 2 * H + h) * head_elems;
          v_off = H * head_elems; ld = HD;
        } else {
          Kb = reinterpret_cast<const T*>(p.self_kv) + ((long long)b * p.layers + layer) * 2 * kvs + h * HD;
          v_off = kvs; ld = d;
        }
        attend_blocks<T, HD>(p.q + b * d + h * HD, Kb, Kb + v_off, ld, ld, n_keys, cx.rank + cx.cs * warp, n_blocks,
                             cx.cs * DEC_WARPS, rec_s + warp * REC);
        __syncthreads();
        if (warp == 0)
          // always the record path (splits >= 2): with a 1-CTA cluster (a profiler that drops the cluster shape) the single
          // record is merged below like any other, instead of attn_finish_item's splits == 1 shortcut writing a head output
          attn_finish_item<T, HD>(rec_s, DEC_WARPS, p.part + (long long)(b * H + h) * p.s_max * REC, cx.rank, max(cx.cs, 2), nullptr,
                                  static_cast<T*>(nullptr));
        __syncthreads();
      }
    }
    // F. every CTA's record of the head is visible to the cluster
    cluster_barrier();
    // G. merge the CS records (redundantly in every CTA: one L2 round trip, no further hand-off) -> o_h as x operand
    if (warp < B) attn_merge_records<T, HD>(p.part + (long long)(warp * H + h) * p.s_max * REC, cx.cs, sm.xh + warp * (HD + GV_XPAD));
    __syncthreads();
    // H. the head's slice of the out-projection -> partial residual update
    gemv_mma<T, false>(ao, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
  }

  __device__ __forceinline__ void phase(int step, int ph, const DecViews<T>& sm, GemvRing& ring, GemvArgs* ready,
                                        GemvArgs* scratch /*[2]*/, int wb_ready, unsigned long long* tr) const {
    const int L = p.layers, d = p.d, B = p.B;
    float best_v[2] = {-INFINITY, -INFINITY};
    int best_i[2] = {0x7fffffff, 0x7fffffff};
    if (ph < 4 * L) {
      const int layer = ph >> 2, sub = ph & 3;
      if (sub < 2) { block(step, layer, sub == 1, sm, ring, ready, scratch, wb_ready, tr); return; }
      const WhisperDecLayer& w = p.lw[layer];
      if (!ready) {
        if (threadIdx.x == 0) gemv_args(step, ph, scratch[0]);
        __syncthreads();
      }
      GemvArgs& a = ready ? *ready : scratch[0];
      if (sub == 2)
        stage_rows_norm_sum<T>(p.x_alt, p.part_x1, p.heads, (long long)B * d, w.b_co, blockIdx.x == 0 ? p.x : nullptr, B, d, sm.xs,
                               sm.xh, 1, w.ln3_w, w.ln3_b, 1e-5f, sm.s_red, sm.wb, wb_ready);
      else
        stage_rows_copy<T>(reinterpret_cast<const T*>(p.h), B, p.ffn, sm.xh);
      if (tr) tr[1] = dec_clock_ns();
      gemv_mma<T, false>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      return;
    }
    if (ph == 4 * L) {
      if (!ready) {
        if (threadIdx.x == 0) gemv_args(step, ph, scratch[0]);
        __syncthreads();
      }
      GemvArgs& a = ready ? *ready : scratch[0];
      stage_rows_norm<T>(p.x, B, d, sm.xs, sm.xh, 1, p.lnf_w, p.lnf_b, 1e-5f, sm.s_red, sm.wb, wb_ready);
      gemv_mma<T, false>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
      gemv_argmax_candidates(best_v, best_i, B, sm.sv, sm.si, p.cand_val, p.cand_idx);
    } else {
      wd_select<T>(p, step - (p.n_prefix - 1), step, sm.sv);
    }
  }
};

// shared-memory layout of the cluster kernel: [xh | scratch (heads + 1) * B * d fp32 | the tail of dec_smem_layout]
__host__ __device__ inline DecSmem wdc_smem_layout(int B, int d, int kmax, int heads) {
  DecSmem L;
  L.xs_off = (((unsigned)B * (unsigned)(kmax + GV_XPAD) * 2u) + 127u) & ~127u;
  dec_smem_tail(L, (L.xs_off + (unsigned)(heads + 1) * (unsigned)B * (unsigned)d * 4u + 127u) & ~127u, 2 * d);
  return L;
}

template <typename T>
__global__ void __launch_bounds__(DEC_THREADS, 1)
whisper_decode_cluster_kernel(const WhisperDecParams p, int step_begin, int step_end, int ph_begin, int ph_end, int coop) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ WhisperDecParams sp;
  __shared__ WhisperDecLayer s_layers[32];
  __shared__ GemvPlan s_plans[6];  // qkv of the head | cq of the head | out-projection slice | fc1 | fc2 | logits
  __shared__ GemvArgs s_args[3];   // [0] prepared for the next projection, [1] built in-phase, [2] out-projection slice
  __shared__ GemvRing s_rings[DEC_WARPS];
  WdcCtx cx;
  // Cluster identity comes from the hardware registers only: whatever cluster shape the launch really got (a tool that
  // intercepts the launch may drop or change the cluster attribute -- a size taken from the parameter block would then
  // give wrong ids), rank / size / id stay mutually consistent and the head -> cluster
  // assignment stays correct; a shape with fewer clusters than heads is caught below.
  cx.cid = (int)cluster_id_x(); cx.rank = (int)cluster_ctarank(); cx.cs = (int)cluster_nctaid_x();
  if ((int)(gridDim.x / cx.cs) < p.heads) __trap();
  if (threadIdx.x < 6) {
    const int i = threadIdx.x;
    const bool has_head = cx.cid < p.heads;
    GemvPlan& pl = s_plans[i];
    if (i == 0) {         // q, k, v rows of head cid
      gemv_head_plan<HD>(GEMV_PLAN_QKV_HEAD, p.d, cx.cid, cx.rank, cx.cs, has_head, pl);
    } else if (i == 1) {  // cross-attention q rows of head cid
      gemv_head_plan<HD>(GEMV_PLAN_Q_HEAD, p.d, cx.cid, cx.rank, cx.cs, has_head, pl);
    } else if (i == 2) {  // all d rows x the head's 64 columns
      gemv_head_plan<HD>(GEMV_PLAN_OUT_SLICE, p.d, cx.cid, cx.rank, cx.cs, has_head, pl);
    } else {
      gemv_make_plan(i == 3 ? p.ffn : i == 5 ? p.vocab : p.d, i == 4 ? p.ffn : p.d, pl);
    }
  }
  if (threadIdx.x == 0) { sp = p; sp.lw = s_layers; }
  for (int i = threadIdx.x; i < p.layers; i += DEC_THREADS) s_layers[i] = p.lw[i];
  __syncthreads();
  const DecSmem lay = wdc_smem_layout(p.B, p.d, max(p.d, p.ffn), p.heads);
  GemvRing& ring = s_rings[threadIdx.x >> 5];
  gemv_ring_init(ring, smem_raw + lay.ring_off, p.ring_slots, s_plans);
  const WdcModel<T> model{sp, cx, 4 * p.layers + 2};
  dec_run<T>(p, model, dec_views<T>(smem_raw, lay), ring, s_args, step_begin, step_end, ph_begin, ph_end, coop);
}

template <typename T>
__global__ void whisper_decode_init_kernel(const WhisperDecParams p) {
  // x = E[first prompt token] + pos[0]; reset flags
  const int b = blockIdx.x;
  const int tok = p.tokens[b * p.max_pos];
  const T* e = reinterpret_cast<const T*>(p.embed);
  for (int i = threadIdx.x; i < p.d; i += blockDim.x) p.x[b * p.d + i] = DT<T>::to_f(e[gv_tiled_elem(tok, i, p.d)]) + p.pos[i];
  dec_init_session(p, b, p.max_new);
}

// ---- cluster kernel launcher: returns S2S_OK and sets *used = 1 when the launch configuration exists on this device
template <typename T>
int launch_cluster_t(s2s_ctx* ctx, const WhisperDecParams& p, int debug_phases, cudaStream_t stream, int* used) {
  *used = 0;
  auto kern = whisper_decode_cluster_kernel<T>;
  const int kmax = std::max(p.d, p.ffn);
  const DecSmem lay = wdc_smem_layout(p.B, p.d, kmax, p.heads);
  const int slots = dec_ring_slots(lay, WD_SMEM_BUDGET);
  if (slots < 2) return S2S_OK;
  const size_t smem = dec_smem_bytes(lay, slots);
  S2S_CHECK_CUDA(s2s_opt_in_max_smem(kern, ctx->device, smem, nullptr));
  // every head needs its own co-resident 8-CTA cluster (queried once per configuration)
  static thread_local size_t cached_smem = 0;
  static thread_local int cached_heads = -1, cached_cs = 0, cached_n = 0, cached_grid = 0;
  const int lane_grid = dec_grid(ctx);
  int cs = 0, n_clusters = 0;
  const bool cache_hit = cached_smem == smem && cached_heads == p.heads && cached_grid == lane_grid;
  if (cache_hit) { cs = cached_cs; n_clusters = cached_n; }
  // only the 8-CTA configuration is validated on hardware (12 heads of Whisper-small on 14-15 co-resident clusters);
  // geometries whose heads do not fit (large-v3: 20 heads) use the 8-phase kernel
  for (int cand = 8; cand >= 8 && !cs && !cache_hit; cand >>= 1) {
    cudaLaunchConfig_t qc{};
    qc.gridDim = dim3((lane_grid / cand) * cand); qc.blockDim = dim3(DEC_THREADS); qc.dynamicSmemBytes = smem;
    cudaLaunchAttribute qa[1];
    qa[0].id = cudaLaunchAttributeClusterDimension; qa[0].val.clusterDim.x = cand; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = 1;
    qc.attrs = qa; qc.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &qc) != cudaSuccess) { cudaGetLastError(); continue; }
    n = std::min(n, lane_grid / cand);
    if (n >= p.heads) { cs = cand; n_clusters = n; }
  }
  cached_smem = smem; cached_heads = p.heads; cached_cs = cs; cached_n = n_clusters; cached_grid = lane_grid;
  if (!cs) return S2S_OK;
  WhisperDecParams pr = p;
  pr.ring_slots = slots;
  pr.cluster_size = cs;
  whisper_decode_init_kernel<T><<<p.B, 256, 0, stream>>>(pr);
  S2S_LAUNCH_CHECK();
  S2S_CHECK(dec_launch(kern, pr, n_clusters * cs, cs, smem, p.n_prefix - 1 + p.max_new, 4 * p.layers + 2, debug_phases, stream));
  *used = 1;
  return S2S_OK;
}

template <typename T>
int launch_t(s2s_ctx* ctx, const WhisperDecParams& p, int debug_phases, cudaStream_t stream) {
  // single sessions: the cluster kernel (fewer grid-wide hops per token); batches use the 8-phase kernel,
  // whose weight stream and attention items spread over all SMs
  if (p.cluster_size != 0 && p.B == 1 && p.x_alt && p.part_x0 && p.part_x1) {
    int used = 0;
    S2S_CHECK(launch_cluster_t<T>(ctx, p, debug_phases, stream, &used));
    if (used) return S2S_OK;
  }
  const DecSmem lay = dec_smem_layout(p.B, p.d, std::max(p.d, p.ffn), 2 * p.d);
  WhisperDecParams pr = p;
  pr.ring_slots = dec_ring_slots(lay, WD_SMEM_BUDGET);
  {
    const int BH = p.B * p.heads, grid = dec_grid(ctx);
    pr.cross_plan = attn_plan(BH, (p.n_ctx + ATT_BLK - 1) / ATT_BLK, p.s_max, grid);
    const int nb_max = (p.max_pos + ATT_BLK - 1) / ATT_BLK;
    S2S_REQUIRE(nb_max < (int)sizeof(pr.self_plan), "whisper decode: max_target_positions %d too large", p.max_pos);
    for (int nb = 1; nb <= nb_max; ++nb) pr.self_plan[nb] = (unsigned char)attn_plan(BH, nb, p.s_max, grid);
  }
  S2S_REQUIRE(pr.ring_slots >= 2, "whisper decode: batch %d leaves no shared memory for the weight ring", p.B);
  const size_t smem = dec_smem_bytes(lay, pr.ring_slots);
  auto kern = whisper_decode_kernel<T>;
  S2S_CHECK_CUDA(s2s_opt_in_max_smem(kern, ctx->device, smem, nullptr));
  whisper_decode_init_kernel<T><<<p.B, 256, 0, stream>>>(pr);
  S2S_LAUNCH_CHECK();
  return dec_launch(kern, pr, dec_grid(ctx), 0, smem, p.n_prefix - 1 + p.max_new, 8 * p.layers + 2, debug_phases, stream);
}

}  // namespace

int whisper_decode_launch(s2s_ctx* ctx, const WhisperDecParams& p, int dtype, int debug_phases, cudaStream_t stream) {
  S2S_REQUIRE(p.d / p.heads == HD, "whisper decode: head_dim must be 64");
  S2S_REQUIRE(p.layers <= 32, "whisper decode: at most 32 decoder layers");
  S2S_REQUIRE(p.B >= 1 && p.B <= DEC_MAX_B, "whisper decode: batch %d > %d must be split by the caller", p.B, DEC_MAX_B);
  S2S_REQUIRE(p.d % 64 == 0 && p.ffn % 64 == 0, "whisper decode: d and ffn must be multiples of 64");
  S2S_REQUIRE(p.n_prefix >= 1 && p.max_new >= 1 && p.n_prefix + p.max_new <= p.max_pos,
              "whisper decode: prompt %d + max_new %d exceeds max_target_positions %d", p.n_prefix, p.max_new, p.max_pos);
  if (dtype == S2S_F16) return launch_t<__half>(ctx, p, debug_phases, stream);
  if (dtype == S2S_BF16) return launch_t<__nv_bfloat16>(ctx, p, debug_phases, stream);
  s2s_set_error("whisper decode: unsupported dtype %d", dtype);
  return S2S_ERR_UNSUPPORTED;
}

int whisper_decode_max_batch(int d, int ffn) {
  for (int B = DEC_MAX_B; B >= 1; --B)
    if (dec_ring_slots(dec_smem_layout(B, d, std::max(d, ffn), 2 * d), WD_SMEM_BUDGET) >= 2) return B;
  return 1;
}
