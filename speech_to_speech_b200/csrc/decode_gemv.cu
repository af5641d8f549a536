// decode_gemv.cu -- the skinny GEMM of the persistent decode kernels by itself (s2s_decode_gemv, exposed for tests).
//
// One ordinary launch of DEC_THREADS-thread CTAs runs 1..3 projections back to back through the decode kernels' own device
// functions (decode_common.cuh): the operand is staged as a phase stages it (stage_rows_copy, stage_rows_norm incl. the
// DEC_NORM_L2 variant, stage_rows_norm_sum, or the K-chunked operand of gemv_mma_chunked), and gemv_mma /
// gemv_mma_chunked stream the tiled weights through each warp's ring and run the epilogue.  Every warp keeps ONE GemvRing
// across the projections, so ring slot and parity carry over from one projection to the next as they do between the
// phases of a decode launch; the shared-memory layout is dec_smem_layout's.  There is no grid barrier: the projections of
// one call must not read what an earlier one of the same call writes.  Both LLAMA instantiations (the epilogue sets of the
// Llama family and of Whisper) live here, so the entry point belongs to neither model's file.
#include <algorithm>
#include <vector>

#include "decode_common.cuh"

namespace {

struct DgProj {
  GemvArgs a;
  int input;                                                  // S2S_GEMV_IN_*
  const void* x16;                                            // COPY: 16-bit [B][K]
  const float* xf; int norm; const float* nw; const float* nb; float eps; int rg;   // NORM / NORM_SUM: fp32 [B][K]
  const float* parts; int n_parts; const float* add_bias; float* x_out;             // NORM_SUM
  void* staged;                                               // CTA 0's staged 16-bit operand [B][K] (null: not copied)
  float* cand_val; int* cand_idx;                             // LOGITS: per-CTA argmax candidates [B][grid]
  int* plan_out;                                              // n_tiles, main_rounds, ks_log, slice, tail_rounds (CTA 0)
  int head_plan; long long x_cluster_stride, out_cluster_stride;   // virtual clusters
};
struct DgParams {
  DgProj pr[3];
  int n_proj, B, slots, prefetch, drain;
  int cluster, heads;   // virtual clusters: CTA i = rank i % cluster of cluster i / cluster (0: whole-grid plans only)
  DecSmem lay;
};

template <typename T, bool LLAMA, bool F8>
__global__ void __launch_bounds__(DEC_THREADS, 1) decode_gemv_kernel(const __grid_constant__ DgParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ GemvPlan s_plans[3];   // the plans of the call's projections, computed once at kernel start (plan_id i)
  __shared__ GemvArgs s_args[3];
  __shared__ GemvRing s_rings[DEC_WARPS];
  const int cid = p.cluster > 0 ? (int)blockIdx.x / p.cluster : 0;
  const int cid_x = min(cid, max(p.heads - 1, 0));   // operand / output offset: clusters without a head reuse the last head's
  if (threadIdx.x < p.n_proj) {
    const DgProj& q = p.pr[threadIdx.x];
    GemvArgs& a = s_args[threadIdx.x];
    a = q.a;
    if (q.head_plan) {
      // QKV / Q rows of head cid: the model width is K; the out-projection slice: the rows (and weight row length) are N
      gemv_head_plan<64>(q.head_plan, q.head_plan == GEMV_PLAN_OUT_SLICE ? a.N : a.K, cid, (int)blockIdx.x % p.cluster, p.cluster,
                         cid < p.heads, s_plans[threadIdx.x]);
      if (a.out) a.out += cid_x * q.out_cluster_stride;
    } else {
      gemv_make_plan(a.N, a.K, s_plans[threadIdx.x]);
    }
  }
  __syncthreads();
  GemvRing& ring = s_rings[threadIdx.x >> 5];
  gemv_ring_init(ring, smem_raw + p.lay.ring_off, p.slots, s_plans);
  const DecViews<T> sm = dec_views<T>(smem_raw, p.lay);
  const int B = p.B;
#pragma unroll 1
  for (int i = 0; i < p.n_proj; ++i) {
    const DgProj& q = p.pr[i];
    const GemvArgs& a = s_args[i];
    const int K = a.K;
    __syncthreads();   // every warp is done with the previous projection's operand and reduction buffers
    if (p.drain && i == p.n_proj - 1) {   // an early exit's look-ahead: units of projection 0 issued, then waited for unused
      gemv_prefetch<T, F8>(s_args[0], ring);
      gemv_drain<F8>(s_args[0].K, ring);
    }
    if (p.prefetch && q.input != S2S_GEMV_IN_CHUNKED) gemv_prefetch<T, F8>(a, ring);   // before the input, as the look-ahead
    switch (q.input) {
      case S2S_GEMV_IN_COPY:
        stage_rows_copy<T>(reinterpret_cast<const T*>(q.x16) + (q.head_plan ? cid_x * q.x_cluster_stride : 0), B, K, sm.xh);
        break;
      case S2S_GEMV_IN_NORM: stage_rows_norm<T>(q.xf, B, K, sm.xs, sm.xh, q.norm, q.nw, q.nb, q.eps, sm.s_red, sm.wb, 0, q.rg); break;
      case S2S_GEMV_IN_NORM_SUM:
        stage_rows_norm_sum<T>(q.xf, q.parts, q.n_parts, (long long)B * K, q.add_bias, blockIdx.x == 0 ? q.x_out : nullptr, B, K,
                               sm.xs, sm.xh, q.norm, q.nw, q.nb, q.eps, sm.s_red, sm.wb, 0);
        break;
      default: break;
    }
    if (q.staged && blockIdx.x == 0 && q.input != S2S_GEMV_IN_CHUNKED) {
      const int hw = K >> 1;   // 32-bit words per row
      for (int e = threadIdx.x; e < B * hw; e += DEC_THREADS) {
        const int b = e / hw, c = e - b * hw;
        reinterpret_cast<uint32_t*>(q.staged)[e] = reinterpret_cast<const uint32_t*>(sm.xh + (long long)b * (K + GV_XPAD))[c];
      }
    }
    float best_v[2] = {-INFINITY, -INFINITY};
    int best_i[2] = {0x7fffffff, 0x7fffffff};
    if (q.input == S2S_GEMV_IN_CHUNKED) gemv_mma_chunked<T, LLAMA, F8>(a, sm.xh, B, best_v, best_i, ring, sm.red);
    else gemv_mma<T, LLAMA, F8>(a, smem_u32(sm.xh), B, best_v, best_i, ring, sm.red);
    if (a.mode == EPI_LOGITS) gemv_argmax_candidates(best_v, best_i, B, sm.sv, sm.si, q.cand_val, q.cand_idx);
    if (blockIdx.x == 0 && threadIdx.x == 0 && q.plan_out) {
      GemvPlan pl = ring.plan;   // warp 0's ring: the plan gemv_mma ran
      if (q.input == S2S_GEMV_IN_CHUNKED) gemv_make_plan(a.N, a.kc, pl);   // gemv_mma_chunked keeps its plan to itself
      q.plan_out[0] = pl.n_tiles; q.plan_out[1] = pl.main_rounds; q.plan_out[2] = pl.ks_log; q.plan_out[3] = pl.slice;
      q.plan_out[4] = pl.tail_rounds;
    }
  }
  gemv_drain<F8>(s_args[0].K, ring);   // nothing is left in flight unless a bookkeeping bug left a prefetch behind
}

// the select phase's merge of the per-CTA candidates: block (0, b) merges session b over gridDim.x = the gemv's grid
__global__ void decode_gemv_argmax_kernel(const float* cand_val, const int* cand_idx, int* out) {
  if (blockIdx.x != 0) return;
  const int id = dec_argmax_merge(cand_val, cand_idx, (int)blockIdx.y);
  if (threadIdx.x == 0) out[blockIdx.y] = id;
}

template <typename T, bool LLAMA, bool F8>
int run_t(s2s_ctx* ctx, DgParams& p, int grid, int want_slots, int (*merge)[2], int n_merge, int* argmax_out[3], int B,
          cudaStream_t st) {
  auto kern = decode_gemv_kernel<T, LLAMA, F8>;
  long long max_dyn = 0;
  S2S_CHECK_CUDA(s2s_max_dyn_smem(kern, ctx->device, &max_dyn));
  const int fit = dec_ring_slots(p.lay, max_dyn);
  S2S_REQUIRE(fit >= 1, "s2s_decode_gemv: the operand of %d sessions leaves no room for a weight ring", B);
  S2S_REQUIRE(want_slots <= fit, "s2s_decode_gemv: %d ring slots requested, %d fit", want_slots, fit);
  p.slots = want_slots > 0 ? want_slots : fit;
  const size_t smem = dec_smem_bytes(p.lay, p.slots);
  S2S_CHECK_CUDA(s2s_opt_in_max_smem(kern, ctx->device, smem, nullptr));
  kern<<<grid, DEC_THREADS, smem, st>>>(p);
  S2S_LAUNCH_CHECK();
  for (int m = 0; m < n_merge; ++m) {
    const DgProj& q = p.pr[merge[m][0]];
    // dec_argmax_merge counts the candidates by gridDim.x: x spans the gemv's grid (only x = 0 works), y the sessions
    decode_gemv_argmax_kernel<<<dim3(grid, B), 32, 0, st>>>(q.cand_val, q.cand_idx, argmax_out[merge[m][0]]);
    S2S_LAUNCH_CHECK();
  }
  return S2S_OK;
}

bool aligned(const void* ptr, int bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (uintptr_t)(bytes - 1)) == 0; }
bool aligned16(const void* ptr) { return aligned(ptr, 16); }

}  // namespace

extern "C" int s2s_decode_gemv(s2s_ctx* ctx, const s2s_dec_gemv_args* args, int32_t* plans_out_h, void* stream) {
  S2S_REQUIRE(ctx && args, "s2s_decode_gemv: null argument");
  const s2s_dec_gemv_args& g = *args;
  S2S_REQUIRE(g.n_proj >= 1 && g.n_proj <= 3, "s2s_decode_gemv: n_proj %d not in [1, 3]", g.n_proj);
  S2S_REQUIRE(g.B >= 1 && g.B <= DEC_MAX_B, "s2s_decode_gemv: B %d not in [1, %d]", g.B, DEC_MAX_B);
  S2S_REQUIRE(g.dtype == S2S_F16 || g.dtype == S2S_BF16, "s2s_decode_gemv: dtype %d", g.dtype);
  const bool f8 = g.weight_format == S2S_FP8_E4M3;
  S2S_REQUIRE(g.weight_format == g.dtype || (f8 && g.dtype == S2S_BF16 && g.llama),
              "s2s_decode_gemv: weight format %d with dtype %d (FP8 needs bf16 and the Llama family)", g.weight_format, g.dtype);
  S2S_REQUIRE(g.slots >= 0 && g.slots <= 4, "s2s_decode_gemv: slots %d not in [0, 4]", g.slots);
  S2S_REQUIRE(g.grid >= 0 && g.grid <= 4096, "s2s_decode_gemv: grid %d", g.grid);
  const int grid = g.grid > 0 ? g.grid : dec_grid(ctx);
  const int B = g.B;
  S2S_REQUIRE(g.cluster == 0 || (g.cluster > 0 && grid % g.cluster == 0 && g.heads >= 1 && grid / g.cluster >= g.heads),
              "s2s_decode_gemv: cluster %d / heads %d on %d CTAs (a whole number of clusters, at least one per head)", g.cluster,
              g.heads, grid);
  DgParams p{};
  p.n_proj = g.n_proj; p.B = B; p.prefetch = g.prefetch ? 1 : 0; p.drain = g.drain ? 1 : 0;
  p.cluster = g.cluster; p.heads = g.cluster > 0 ? g.heads : 0;
  int kmax = 32, d_norm = 0, rg_rows = 0, sum_floats = 0, n_merge = 0, merge[3][2] = {};
  size_t cand_bytes = 0;
  for (int i = 0; i < g.n_proj; ++i) {
    const s2s_dec_gemv_proj& s = g.proj[i];
    const int N = s.N, K = s.K, m = s.mode;
    S2S_REQUIRE(s.w && aligned16(s.w) && N >= 1 && K >= 32 && K % 32 == 0,
                "s2s_decode_gemv: projection %d: w / N %d / K %d (K a positive multiple of 32, w 16-byte aligned)", i, N, K);
    const bool mode_ok = g.llama ? (m == EPI_STORE || m == EPI_RESID || m == EPI_LOGITS || m == EPI_QKV_ROPE || m == EPI_SWIGLU)
                                 : (m == EPI_STORE || m == EPI_RESID || m == EPI_LOGITS || m == EPI_QKV || m == EPI_GELU);
    S2S_REQUIRE(mode_ok, "s2s_decode_gemv: projection %d: mode %d does not exist in the %s instantiation", i, m,
                g.llama ? "Llama-family" : "Whisper");
    // the pair epilogue stores two rows at a time and only checks row0 < N; the bias is read as a float2 at row0
    S2S_REQUIRE(N % 2 == 0 || m == EPI_LOGITS, "s2s_decode_gemv: projection %d: odd N %d outside LOGITS", i, N);
    S2S_REQUIRE(!s.bias || N % 2 == 0, "s2s_decode_gemv: projection %d: a bias with odd N %d", i, N);
    // the epilogue's vector accesses: float2 at out / bias / kraw / rope + an even offset, 16-bit pairs (uint32) at out_h (GELU)
    // and in the caches at even element offsets
    S2S_REQUIRE(!s.bias || aligned(s.bias, 8), "s2s_decode_gemv: projection %d: bias not 8-byte aligned", i);
    if (m == EPI_STORE || m == EPI_RESID || m == EPI_QKV || m == EPI_QKV_ROPE)
      S2S_REQUIRE(s.out && aligned(s.out, 8) && s.ldo >= 2 && s.ldo % 2 == 0 && s.out_cluster_stride % 2 == 0,
                  "s2s_decode_gemv: projection %d: out (8-byte aligned) / ldo %d / out_cluster_stride (even)", i, s.ldo);
    if (m == EPI_GELU)
      S2S_REQUIRE(s.out_h && aligned(s.out_h, 4) && s.ldh >= 2 && s.ldh % 2 == 0,
                  "s2s_decode_gemv: projection %d: out_h (4-byte aligned) / ldh %d (even)", i, s.ldh);
    if (m == EPI_SWIGLU)
      S2S_REQUIRE(s.out_h && aligned(s.out_h, 2) && s.ldh >= 1, "s2s_decode_gemv: projection %d: out_h / ldh %d", i, s.ldh);
    if (m == EPI_QKV)
      S2S_REQUIRE(s.kv0 && aligned(s.kv0, 4) && s.d >= 2 && s.d % 2 == 0 && N == 3 * s.d && s.kv_which % 2 == 0 && s.kv_batch % 2 == 0,
                  "s2s_decode_gemv: projection %d: QKV needs kv0 (4-byte aligned), N = 3 d, even d / kv_which / kv_batch", i);
    if (m == EPI_QKV_ROPE)
      S2S_REQUIRE(s.kv0 && aligned(s.kv0, 4) && s.pos && s.slot && s.rope && aligned(s.rope, 8) && s.hd >= 2 && s.hd % 2 == 0 &&
                      s.q_rows % 2 == 0 && s.k_rows % 2 == 0 && s.q_rows + s.k_rows <= N && s.kv_which % 2 == 0 &&
                      s.kv_slot % 2 == 0 && s.kv_ld % 2 == 0 && (!s.kraw || (s.k_rows > 0 && aligned(s.kraw, 8))),
                  "s2s_decode_gemv: projection %d: QKV_ROPE needs kv0, pos, slot, rope, kraw aligned and even hd / q_rows / k_rows "
                  "/ cache strides", i);
    if (m == EPI_LOGITS) {
      S2S_REQUIRE(s.argmax_out, "s2s_decode_gemv: projection %d: LOGITS needs argmax_out", i);
      S2S_REQUIRE(!s.logits_out || (aligned(s.logits_out, 4) && s.logits_ld >= N),
                  "s2s_decode_gemv: projection %d: logits_out / logits_ld %lld < N", i, (long long)s.logits_ld);
      merge[n_merge][0] = i; merge[n_merge][1] = (int)cand_bytes; ++n_merge;
      cand_bytes += (size_t)B * grid * 8;
    }
    DgProj& q = p.pr[i];
    GemvArgs& a = q.a;
    a.W = s.w; a.N = N; a.K = K; a.bias = s.bias; a.mode = m; a.out = s.out; a.ldo = s.ldo; a.out_h = s.out_h; a.ldh = s.ldh;
    a.kv0 = s.kv0; a.kv_which = s.kv_which; a.kv_batch = s.kv_batch; a.d = s.d;
    a.suppress = s.suppress; a.first_step = s.first_step; a.logits_out = s.logits_out; a.logits_ld = s.logits_ld;
    a.pos = s.pos; a.slot = s.slot; a.kv_slot = s.kv_slot; a.kv_ld = s.kv_ld; a.rope = reinterpret_cast<const float2*>(s.rope);
    a.hd = s.hd; a.q_rows = s.q_rows; a.k_rows = s.k_rows; a.q_scale = s.q_scale; a.kraw = s.kraw;
    a.plan_id = (g.use_plans || s.head_plan) ? i : -1;   // a head plan exists only in the kernel's plan table
    S2S_REQUIRE(s.head_plan >= 0 && s.head_plan <= GEMV_PLAN_OUT_SLICE, "s2s_decode_gemv: projection %d: head_plan %d", i, s.head_plan);
    if (s.head_plan) {
      const int hd_tot = 64 * g.heads;
      const bool shape_ok = s.head_plan == GEMV_PLAN_QKV_HEAD  ? (N == 3 * K && hd_tot <= K)
                            : s.head_plan == GEMV_PLAN_Q_HEAD  ? (N == K && hd_tot <= K)
                                                               : (K == 64 && N % 8 == 0 && hd_tot <= N);
      S2S_REQUIRE(g.cluster > 0 && s.input != S2S_GEMV_IN_CHUNKED && shape_ok && s.x_cluster_stride >= 0 && s.out_cluster_stride >= 0,
                  "s2s_decode_gemv: projection %d: head_plan %d needs virtual clusters, an unchunked input and a [3d, d] / [d, d] / "
                  "[d, 64 of d] shape with 64 * heads <= d", i, s.head_plan);
    }
    q.head_plan = s.head_plan; q.x_cluster_stride = s.x_cluster_stride; q.out_cluster_stride = s.out_cluster_stride;
    a.xsrc = nullptr; a.xsrc_ld = 0; a.kc = 0;
    q.input = s.input; q.staged = s.staged;
    switch (s.input) {
      case S2S_GEMV_IN_COPY:
        S2S_REQUIRE(s.x16 && aligned16(s.x16), "s2s_decode_gemv: projection %d: x16 (16-byte aligned)", i);
        q.x16 = s.x16; kmax = std::max(kmax, K);
        break;
      case S2S_GEMV_IN_NORM:
      case S2S_GEMV_IN_NORM_SUM: {
        const bool sum = s.input == S2S_GEMV_IN_NORM_SUM;
        S2S_REQUIRE(s.xf && aligned16(s.xf) && (s.norm == 1 || s.norm == 2) && s.norm_w && aligned16(s.norm_w) &&
                        (s.norm == 2 || (s.norm_b && aligned16(s.norm_b))),
                    "s2s_decode_gemv: projection %d: xf / norm %d / norm_w / norm_b (LayerNorm 1, RMSNorm 2; 16-byte aligned)", i,
                    s.norm);
        S2S_REQUIRE(sum ? s.rg == 0 : (s.rg == DEC_NORM_L2 || (s.rg >= 0 && s.rg <= DEC_MAX_B)),
                    "s2s_decode_gemv: projection %d: rg %d", i, s.rg);
        S2S_REQUIRE(s.rg != DEC_NORM_L2 || K <= NORM_L2_MAX_D, "s2s_decode_gemv: projection %d: rg -1 needs K <= %d", i, NORM_L2_MAX_D);
        if (sum) {
          S2S_REQUIRE(s.n_parts >= 0 && s.n_parts <= 64 && (s.n_parts == 0 || (s.parts && aligned16(s.parts))) && s.add_bias &&
                          aligned16(s.add_bias) && (!s.x_out || aligned16(s.x_out)),
                      "s2s_decode_gemv: projection %d: parts / n_parts %d / add_bias / x_out", i, s.n_parts);
          sum_floats = std::max(sum_floats, (s.n_parts + 1) * B * K);
        }
        q.xf = s.xf; q.norm = s.norm; q.nw = s.norm_w; q.nb = s.norm == 1 ? s.norm_b : nullptr; q.eps = s.eps; q.rg = s.rg;
        q.parts = s.parts; q.n_parts = s.n_parts; q.add_bias = s.add_bias; q.x_out = s.x_out;
        kmax = std::max(kmax, K); d_norm = std::max(d_norm, K);
        if (s.rg != DEC_NORM_L2) rg_rows = std::max(rg_rows, (s.rg <= 0 || s.rg > B) ? B : s.rg);
        break;
      }
      case S2S_GEMV_IN_CHUNKED:
        S2S_REQUIRE(s.x16 && aligned16(s.x16) && gemv_chunk_ok(N, K, s.kc, grid),
                    "s2s_decode_gemv: projection %d: kc %d does not chunk [%d, %d] on %d CTAs (gemv_chunk_ok)", i, s.kc, N, K, grid);
        S2S_REQUIRE(!s.staged, "s2s_decode_gemv: projection %d: a chunked operand is never staged whole", i);
        a.xsrc = s.x16; a.xsrc_ld = K; a.kc = s.kc;
        kmax = std::max(kmax, s.kc);
        break;
      default: S2S_REQUIRE(false, "s2s_decode_gemv: projection %d: input %d", i, s.input);
    }
  }
  // the decode kernels' layout; a norm-sum input keeps its (n_parts + 1) * B rows in the fp32 region, as the cluster kernel
  // sizes it (whisper_decode.cu wdc_smem_layout)
  DecSmem lay = dec_smem_layout(B, std::max(d_norm, 32), kmax, 2 * d_norm, rg_rows > 0 ? rg_rows : DEC_NORM_L2);
  const unsigned int sum_end = (lay.xs_off + (unsigned)sum_floats * 4u + 127u) & ~127u;
  if (sum_end > lay.aux_off) dec_smem_tail(lay, sum_end, 2 * d_norm);
  p.lay = lay;

  S2S_CHECK_CUDA(cudaSetDevice(ctx->device));
  const cudaStream_t st = (cudaStream_t)stream;
  // per-call scratch: argmax candidates of the LOGITS projections, the plans CTA 0 ran
  char* scratch = nullptr;
  const size_t plan_bytes = (size_t)g.n_proj * 5 * 4;
  S2S_CHECK_CUDA(cudaMalloc(&scratch, cand_bytes + plan_bytes));
  int* argmax_out[3] = {};
  for (int m = 0; m < n_merge; ++m) {
    DgProj& q = p.pr[merge[m][0]];
    q.cand_val = reinterpret_cast<float*>(scratch + merge[m][1]);
    q.cand_idx = reinterpret_cast<int*>(scratch + merge[m][1] + (size_t)B * grid * 4);
    argmax_out[merge[m][0]] = g.proj[merge[m][0]].argmax_out;
  }
  int* plans_d = reinterpret_cast<int*>(scratch + cand_bytes);
  for (int i = 0; i < g.n_proj; ++i) p.pr[i].plan_out = plans_d + 5 * i;
  int rc = S2S_OK;
  if (f8) rc = run_t<__nv_bfloat16, true, true>(ctx, p, grid, g.slots, merge, n_merge, argmax_out, B, st);
  else if (g.dtype == S2S_BF16) rc = g.llama ? run_t<__nv_bfloat16, true, false>(ctx, p, grid, g.slots, merge, n_merge, argmax_out, B, st)
                                             : run_t<__nv_bfloat16, false, false>(ctx, p, grid, g.slots, merge, n_merge, argmax_out, B, st);
  else rc = g.llama ? run_t<__half, true, false>(ctx, p, grid, g.slots, merge, n_merge, argmax_out, B, st)
                    : run_t<__half, false, false>(ctx, p, grid, g.slots, merge, n_merge, argmax_out, B, st);
  std::vector<int> plans((size_t)g.n_proj * 5, 0);
  if (rc == S2S_OK) {
    const cudaError_t e = cudaMemcpyAsync(plans.data(), plans_d, plan_bytes, cudaMemcpyDeviceToHost, st);
    const cudaError_t e2 = cudaStreamSynchronize(st);
    if (e != cudaSuccess || e2 != cudaSuccess) {
      s2s_set_error("s2s_decode_gemv: %s", cudaGetErrorString(e != cudaSuccess ? e : e2));
      rc = S2S_ERR_CUDA;
    }
  }
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  if (rc == S2S_OK && plans_out_h) std::copy(plans.begin(), plans.end(), plans_out_h);
  return rc;
}
