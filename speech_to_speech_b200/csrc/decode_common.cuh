// decode_common.cuh -- building blocks of the persistent single-token decode kernels
// (Whisper decoder, Llama-family decoder).
//
// A decode step at small batch is a chain of tiny matrix-vector phases; per phase every SM touches only a few
// KB, so the phase time is (HBM/L2 round trips on its critical path) + (grid barrier), not bytes / bandwidth.
// Everything here is therefore written for memory-level parallelism: all loads of a phase are independent and
// issued back to back (cp.async / cp.async.bulk into shared memory, or explicit register staging) so that each
// phase costs ONE round trip; work items are interleaved across CTAs so all SMs pull from HBM; buffers produced by
// other CTAs inside the launch are read through L2 (ld.global.cg, cp.async.cg, bulk copies) so a stale L1 line can
// never be observed.  Projections run on the tensor cores (mma.sync, sessions on the m dimension), attention and
// normalisation on the CUDA cores; accumulation is fp32.  State shared by the threads of a CTA (argument structs,
// ring bookkeeping) lives in shared memory, not on the stack: the L1 left next to ~150-220 KB of shared memory is
// too small for 256 private copies.
#pragma once
#include "common.cuh"

constexpr int DEC_THREADS = 256;
constexpr int DEC_WARPS = DEC_THREADS / 32;
constexpr int ATT_CHUNK = 64;   // record storage granularity: s_max = ceil(max keys / 64) records per (session, head)
constexpr int PART_PAD = 4;     // partial record = [o[hd], m, l, pad, pad] (16-byte aligned records)

// ---- grid barrier (all CTAs co-resident: cooperative launch) ------------------------------
// Monotonic counter: barrier #e completes when counter == e * gridDim.x.  Bounded spin -> trap.
// Split-phase: grid_arrive() publishes this CTA's results; everything that does not depend on other CTAs (argument
// setup, weight-ring issue, norm-weight loads for the NEXT phase) runs between arrive and wait, i.e. off the
// critical path; grid_wait() then blocks until every CTA has arrived.
__device__ __forceinline__ void grid_arrive(unsigned int* counter, unsigned int& epoch) {
  __syncthreads();  // CTA-scope: every thread's phase results happen-before thread 0's release below
  if (threadIdx.x == 0) {
    epoch += 1;
    // release-add at gpu scope (cumulative over the bar.sync above); no MEMBAR.SC, no L1 flush: all cross-CTA
    // data is read with ld.global.cg / .nc, never through L1.
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
  }
}
__device__ __forceinline__ unsigned int ld_relaxed_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Polling the counter costs one L2 round trip per sample; with a single load in flight the release is
// noticed on average half a round trip late.  Thread 0 therefore keeps FOUR relaxed loads in flight, issued a
// quarter round trip apart; the pipeline is self-clocking (each consumed load is re-issued at once), so the counter
// is sampled several times per round trip.  After the successful sample thread 0 executes fence.acq_rel.gpu: relaxed load + fence is
// the PTX acquire pattern, it synchronises with every producer's red.release, and the bar.sync that follows extends
// the ordering to the CTA's other threads (causality order is transitive over barriers).  `relaxed` != 0 skips the
// fence (A/B measurements only, S2S_SYNC_RELAXED=1): without it the cross-CTA reads race under the PTX memory model
// even when every one of them is an L2 access.
__device__ __forceinline__ void grid_wait(unsigned int* counter, unsigned int epoch_thread0, int relaxed = 0) {
  if (threadIdx.x == 0) {
    const unsigned int target = epoch_thread0 * gridDim.x;
    unsigned int v0 = ld_relaxed_gpu(counter), v1 = 0, v2 = 0, v3 = 0;
    if (v0 < target) {
      long long t = clock64();
      while (clock64() - t < 330) {}
      v1 = ld_relaxed_gpu(counter);
      t = clock64();
      while (clock64() - t < 330) {}
      v2 = ld_relaxed_gpu(counter);
      t = clock64();
      while (clock64() - t < 330) {}
      v3 = ld_relaxed_gpu(counter);
      unsigned int spins = 0;
      while (true) {
        if (v0 >= target) break;
        v0 = ld_relaxed_gpu(counter);
        if (v1 >= target) break;
        v1 = ld_relaxed_gpu(counter);
        if (v2 >= target) break;
        v2 = ld_relaxed_gpu(counter);
        if (v3 >= target) break;
        v3 = ld_relaxed_gpu(counter);
        if (++spins > (1u << 26)) __trap();
      }
    }
    if (!relaxed) asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncthreads();
}
__device__ __forceinline__ void grid_sync(unsigned int* counter, unsigned int& epoch) {
  grid_arrive(counter, epoch);
  grid_wait(counter, epoch);
}
// host: S2S_SYNC_RELAXED=1 selects the unfenced barrier waits (measurement aid, never the default)
inline int dec_sync_relaxed_env() {
  const char* e = getenv("S2S_SYNC_RELAXED");  // read per launch so one process can A/B
  return (e && e[0] == '1') ? 1 : 0;
}

// Warp w of CTA c takes work items  w * gridDim.x + c, then + total_warps ...: consecutive items land on
// different SMs, so a phase with few items still spreads over the whole chip.
__device__ __forceinline__ int dec_first_item() { return (threadIdx.x >> 5) * gridDim.x + blockIdx.x; }
__device__ __forceinline__ int dec_item_stride() { return gridDim.x * DEC_WARPS; }

// L2 warm-up of one attention work item: n_rows rows of `row_bytes` bytes at stride ld_bytes.
__device__ __forceinline__ void prefetch_strided_l2(const void* base, long long ld_bytes, int n_rows, int row_bytes) {
  const int lane = threadIdx.x & 31;
  const int lines_per_row = (row_bytes + 127) >> 7;
#pragma unroll 1
  for (int i = lane; i < n_rows * lines_per_row; i += 32) {
    const char* a = reinterpret_cast<const char*>(base) + (long long)(i / lines_per_row) * ld_bytes + (i % lines_per_row) * 128;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(a));
  }
}

// ---- shared-memory operand layout of the skinny GEMM --------------------------------------------------------
// The activation operand lives in shared memory as 16-bit rows xh[b][K + GV_XPAD]; the 64-byte pad puts
// consecutive rows 64 bytes apart modulo 128, so the 16-byte fragment loads of a quarter-warp (2 rows x 4 k-groups)
// touch 8 distinct 16-byte bank groups.
// The weight operand is stored in GLOBAL memory already in fragment order ("tiled", weight_tiles.cu): tile = 8 rows,
// window = 32 k; element (row 8*tile + g, k 32*w + 8*t + e) sits at ((tile * K/32 + w) * 32 + 4*g + t) * 8 + e.
// Any run of windows of a tile is one contiguous block, so a ring unit is ONE bulk copy of up to 4 KB and a warp's
// 16-byte fragment loads of a window read 512 consecutive bytes (conflict-free without padding).
constexpr int DEC_MAX_B = 16;        // sessions per launch: the m dimension of mma.m16n8k16
constexpr int GV_XPAD = 32;          // elements
constexpr int GV_ROWS = 8;           // weight rows per tile: the n dimension of mma.m16n8k16
constexpr int GV_UK = 256;           // k elements per ring unit (8 windows of 32)
constexpr int GV_WIN_BYTES = GV_ROWS * 32 * 2;           // one 32-element k window of a tile: 512 B, fragment-major
constexpr int GV_SLOT_BYTES = GV_ROWS * GV_UK * 2;       // 4096
constexpr int GV_LAT_ELEMS = 352;    // cost model: one dependent round ~ streaming 352 k-elements of a tile

// ---- dynamic shared-memory layout shared by the decode kernels (host computes the same numbers) ----------
//   [ xh : B x (kmax + GV_XPAD) 16-bit | the fp32 copy used for norm statistics aliases its tail ]
//   [ sv, si : argmax candidates | s_red | wb : norm weights | red : tail-round partial fragments ]
//   [ weight rings : DEC_WARPS x slots x GV_SLOT_BYTES | mbarriers ]
struct DecSmem {
  unsigned int xs_off;     // fp32 statistics copy (B * d floats), inside the xh region
  unsigned int aux_off;    // sv
  unsigned int si_off, red_s_off, wb_off, redbuf_off, ring_off;
};
// rg: rows of the fp32 statistics copy that are resident at a time (stage_rows_norm walks the B rows in groups of rg; rg = B
// = everything in one memory round trip, the default); kmax: widest activation operand that is staged WHOLE (a wider one is
// staged in K-chunks of kmax columns, gemv_mma_chunked).
__host__ __device__ inline DecSmem dec_smem_layout(int B, int d, int kmax, int wb_floats, int rg = 0) {
  DecSmem L;
  if (rg <= 0 || rg > B) rg = B;
  const unsigned int xh_small = (((unsigned)B * (unsigned)(d + GV_XPAD) * 2u) + 15u) & ~15u;
  unsigned int xh_bytes = (unsigned)B * (unsigned)(kmax + GV_XPAD) * 2u;
  const unsigned int with_stats = xh_small + (unsigned)rg * (unsigned)d * 4u;
  if (with_stats > xh_bytes) xh_bytes = with_stats;
  xh_bytes = (xh_bytes + 127u) & ~127u;
  L.xs_off = xh_small;
  L.aux_off = xh_bytes;
  L.si_off = L.aux_off + DEC_WARPS * DEC_MAX_B * 4;
  L.red_s_off = L.si_off + DEC_WARPS * DEC_MAX_B * 4;
  L.wb_off = L.red_s_off + 2 * DEC_WARPS * DEC_MAX_B * 4;   // s_red: [row iterations <= 16][2][DEC_WARPS]
  L.redbuf_off = (L.wb_off + (unsigned)wb_floats * 4u + 15u) & ~15u;
  L.ring_off = (L.redbuf_off + 2u * DEC_THREADS * 16u + 127u) & ~127u;
  return L;
}
// ring slots that fit next to the fixed part (at most 4 per warp)
inline int dec_ring_slots(const DecSmem& L) {
  const long long avail = 220LL * 1024 - (long long)L.ring_off - 256;  // static shared memory (parameter tables) takes ~5 KB
  long long s = avail / ((long long)DEC_WARPS * (GV_SLOT_BYTES + 8));
  return (int)(s > 4 ? 4 : s);
}

// 16-byte asynchronous global -> shared copy through L2 (no registers held while in flight)
__device__ __forceinline__ void cp_async16(uint32_t dst_s, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_s), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Norm weights of a phase (w [| bias] -> wb[d (+ d)]), asynchronous: callable between grid_arrive and grid_wait
// without putting their L2 round trip on the barrier's critical path; they are complete after the consumer's
// cp_async_wait_all() + __syncthreads() (stage_rows_norm).
static __device__ __forceinline__ void stage_norm_weights(const float* w, const float* bias, int d, float* wb) {
  const uint32_t wb_s = smem_u32(wb);
#pragma unroll 1
  for (int i = threadIdx.x * 4; i < d; i += DEC_THREADS * 4) {
    cp_async16(wb_s + (uint32_t)i * 4, w + i);
    if (bias) cp_async16(wb_s + (uint32_t)(d + i) * 4, bias + i);
  }
}

// ---- stage B rows of the fp32 residual stream (produced by other CTAs) into xh, normalised ----------------
// mode 1: LayerNorm (w, bias); 2: RMSNorm (w).  All rows land in shared memory (xs, B*d floats) through cp.async:
// every copy of the phase is in flight at once whatever B is (one L2 round trip, no registers), then one-pass
// statistics (sum, sum of squares) and the normalised row is written as 16-bit into xh[b][d + GV_XPAD].
// Ends with a __syncthreads().
// statistics + normalisation of B rows already in shared memory (xs) -> xh; ends with a __syncthreads()
template <typename T>
static __device__ __forceinline__ void norm_from_smem(const float* xs, int B, int d, T* xh, int mode, float eps, float* s_red,
                                                      const float* wb) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int wpr = DEC_WARPS;  // warps per row: largest power of two with wpr * B <= DEC_WARPS (min 1)
  while (wpr > 1 && wpr * B > DEC_WARPS) wpr >>= 1;
  const int rows_per_iter = DEC_WARPS / wpr;
  const int xstride = d + GV_XPAD;
  const float inv_d = 1.f / (float)d;
  // pass 1: every row's partial statistics (all iterations), ONE barrier; pass 2: normalise
  const int sub = warp % wpr, rsel = warp / wpr;
#pragma unroll 1
  for (int r0 = 0, it = 0; r0 < B; r0 += rows_per_iter, ++it) {
    const int row = r0 + rsel;
    float s1 = 0.f, s2 = 0.f;
    if (row < B) {
      const float* xr = xs + row * d;
#pragma unroll 2
      for (int i = (sub * 32 + lane) * 2; i < d; i += wpr * 64) {
        const float2 v = *reinterpret_cast<const float2*>(xr + i);
        s1 += v.x + v.y;
        s2 = fmaf(v.x, v.x, s2);
        s2 = fmaf(v.y, v.y, s2);
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) { s_red[it * 2 * DEC_WARPS + warp] = s1; s_red[it * 2 * DEC_WARPS + DEC_WARPS + warp] = s2; }
  }
  __syncthreads();
#pragma unroll 1
  for (int r0 = 0, it = 0; r0 < B; r0 += rows_per_iter, ++it) {
    const int row = r0 + rsel, grp = rsel * wpr;
    if (row < B) {
      float t1 = 0.f, t2 = 0.f;
      for (int k = 0; k < wpr; ++k) { t1 += s_red[it * 2 * DEC_WARPS + grp + k]; t2 += s_red[it * 2 * DEC_WARPS + DEC_WARPS + grp + k]; }
      const float mean = (mode == 1) ? t1 * inv_d : 0.f;
      // var = E[x^2] - mean^2 in fp32: accurate to ~1e-6 * (1 + mean^2/var), far below the stated tolerances
      const float var = fmaxf(t2 * inv_d - mean * mean, 0.f);
      const float rstd = rsqrtf(var + eps);
      const float* xr = xs + row * d;
      T* dst = xh + row * xstride;
#pragma unroll 2
      for (int i = (sub * 32 + lane) * 2; i < d; i += wpr * 64) {
        const float2 v = *reinterpret_cast<const float2*>(xr + i);
        const float2 g = *reinterpret_cast<const float2*>(wb + i);
        float y0 = (v.x - mean) * rstd * g.x, y1 = (v.y - mean) * rstd * g.y;
        if (mode == 1) { const float2 bb = *reinterpret_cast<const float2*>(wb + d + i); y0 += bb.x; y1 += bb.y; }
        *reinterpret_cast<uint32_t*>(dst + i) = DT<T>::pack2(y0, y1);
      }
    }
  }
  __syncthreads();
}

template <typename T>
static __device__ __noinline__ void stage_rows_norm(const float* x, int B, int d, float* xs, T* xh, int mode, const float* w,
                                                    const float* bias, float eps, float* s_red, float* wb, int wb_ready, int rg = 0) {
  if (rg <= 0 || rg > B) rg = B;
  const uint32_t xs_s = smem_u32(xs);
  // rows in groups of rg (all of them at once unless the fp32 copy of B rows does not fit next to the 16-bit operand)
#pragma unroll 1
  for (int r0 = 0; r0 < B; r0 += rg) {
    const int rows = min(rg, B - r0), n = rows * d;
    const float* src = x + (long long)r0 * d;
#pragma unroll 4
    for (int i = threadIdx.x * 4; i < n; i += DEC_THREADS * 4) cp_async16(xs_s + (uint32_t)i * 4, src + i);
    if (r0 == 0 && !wb_ready) stage_norm_weights(w, mode == 1 ? bias : nullptr, d, wb);
    cp_async_wait_all();
    __syncthreads();
    norm_from_smem<T>(xs, rows, d, xh + (long long)r0 * (d + GV_XPAD), mode, eps, s_red, wb);   // ends with a __syncthreads()
  }
}

// Same, for a residual stream that is still in pieces: x_eff = x + add_bias + sum_p parts[p] (fixed order ->
// deterministic), with the n_parts partial out-projections of the previous phase (one per head) at stride
// part_stride.  All pieces land in `scratch` ((n_parts + 1) * B * d floats) through cp.async in one round trip;
// x_eff replaces piece 0, is normalised into xh and, when x_out != null (ONE designated CTA), written back as the new
// residual stream for the later phases.
template <typename T>
static __device__ __noinline__ void stage_rows_norm_sum(const float* x, const float* parts, int n_parts, long long part_stride,
                                                        const float* add_bias, float* x_out, int B, int d, float* scratch,
                                                        T* xh, int mode, const float* w, const float* bias, float eps,
                                                        float* s_red, float* wb, int wb_ready) {
  const int n = B * d;
  const uint32_t sc_s = smem_u32(scratch);
#pragma unroll 2
  for (int i = threadIdx.x * 4; i < n; i += DEC_THREADS * 4) {
    cp_async16(sc_s + (uint32_t)i * 4, x + i);
#pragma unroll 1
    for (int p = 0; p < n_parts; ++p) cp_async16(sc_s + (uint32_t)((p + 1) * n + i) * 4, parts + p * part_stride + i);
  }
  if (!wb_ready) stage_norm_weights(w, mode == 1 ? bias : nullptr, d, wb);
  cp_async_wait_all();
  // each thread sums the columns it copied itself: no barrier needed before the sum
#pragma unroll 1
  for (int i = threadIdx.x * 4; i < n; i += DEC_THREADS * 4) {
    float4 acc = *reinterpret_cast<const float4*>(scratch + i);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(add_bias + (i % d)));
    acc.x += bb.x; acc.y += bb.y; acc.z += bb.z; acc.w += bb.w;
#pragma unroll 4
    for (int p = 0; p < n_parts; ++p) {
      const float4 v = *reinterpret_cast<const float4*>(scratch + (p + 1) * n + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    *reinterpret_cast<float4*>(scratch + i) = acc;
    if (x_out) *reinterpret_cast<float4*>(x_out + i) = acc;
  }
  __syncthreads();
  norm_from_smem<T>(scratch, B, d, xh, mode, eps, s_red, wb);
}

// ---- stage B rows of a 16-bit activation (global [B, K], produced by other CTAs) into xh: cp.async 16-byte
// copies straight into the padded rows, all in flight together ----
template <typename T>
static __device__ __noinline__ void stage_rows_copy(const T* x, int B, int K, T* xh) {
  const int vpr = K >> 3;  // 16-byte vectors per row
  const int n = B * vpr;
  const uint32_t xh_s = smem_u32(xh);
  const uint32_t row_bytes = (uint32_t)(K + GV_XPAD) * 2;
  int row = threadIdx.x / vpr, col = threadIdx.x - row * vpr;  // (row, col) of vector index i
#pragma unroll 2
  for (int i = threadIdx.x; i < n; i += DEC_THREADS) {
    cp_async16(xh_s + row * row_bytes + (uint32_t)col * 16, reinterpret_cast<const uint4*>(x + (long long)row * K) + col);
    col += DEC_THREADS;
    while (col >= vpr) { col -= vpr; ++row; }
  }
  cp_async_wait_all();
  __syncthreads();
}

// ---- skinny GEMM: out[b][row] = sum_k W[row][k] * x[b][k], b < B <= 16 -----------------------------------
// ONE non-inlined routine serves every projection of every layer (runtime shapes and a runtime epilogue
// mode): the decode step executes each phase once per layer, so per-phase inlined copies (245 KB of SASS)
// turned the kernel into an instruction-cache streaming problem; sharing the routine keeps the hot loop resident.
//
// Tensor-core formulation (swap-AB): the batch is the m dimension of mma.sync.m16n8k16 (16 sessions, zero-padded),
// a tile of 8 weight rows is the n dimension, so the weight stream is the B operand and the accumulator fragment
// D[m = session][n = weight row] needs no cross-lane reduction; 1..16 sessions cost the same instruction stream.
// The k index inside an instruction may be permuted freely as long as A and B agree, so lane (g, t) feeds both
// from ONE 16-byte shared-memory load each: elements 8t..8t+7 of a 32-element k window serve two instructions.
//
// Work decomposition: tiles of 8 rows.  "Main rounds": while at least gridDim.x * 8 tiles remain, every warp of
// the grid owns one tile and its full K (no synchronisation at all).  "Tail": the remaining < gridDim.x * 8 tiles
// are split 2^ks_log ways along K so that all warps stream; the partial fragments of a tile meet in shared memory
// (one __syncthreads per tail round, fixed summation order -> deterministic).  The small projections of the
// Whisper decoder are all tail.
enum GemvEpi { EPI_STORE = 0, EPI_GELU = 1, EPI_RESID = 2, EPI_QKV = 3, EPI_LOGITS = 4,
               EPI_QKV_ROPE = 5 /* row pairs */, EPI_SWIGLU = 6 /* row pairs */ };
struct GemvArgs {
  const void* W; int N, K;     // W: TILED weights (see above), N rows (storage padded to a multiple of 8), K % 32 == 0
  const float* bias;           // [N] or null
  int mode;
  float* out; int ldo;         // STORE / RESID (in-place residual stream) / QKV (q rows): fp32
  void* out_h; int ldh;        // GELU / SWIGLU: 16-bit activation [B, ldh]
  // QKV: rows [d, 2d) -> k cache, [2d, 3d) -> v cache (16-bit), element (b, c) at kv0 + which*kv_which + b*kv_batch + c
  void* kv0; long long kv_which, kv_batch; int d;
  // LOGITS
  const unsigned char* suppress; int first_step; float* logits_out; long long logits_ld;  // logits_out + b*logits_ld + row
  // QKV_ROPE (Llama family): rows are stored so that rotate_half partners (j, j + hd/2) are adjacent (2j, 2j+1).
  // rows [0, q_rows) -> out (fp32 q, rotated); [q_rows, q_rows + k_rows) -> K cache (rotated); rest -> V cache.
  // cache element (b, c): kv0 + which*kv_which + slot[b]*kv_slot + pos[b]*kv_ld + c ; rope[pos][j] = (cos, sin)
  const int* pos; const int* slot; long long kv_slot; int kv_ld; const float2* rope; int hd, q_rows, k_rows;
  float q_scale;               // softmax scale folded into the stored q (head_dim^-0.5)
  float* kraw;                 // Qwen3 (qk_norm): non-null -> q and k are stored RAW (fp32: q -> out, k -> kraw[b][k_rows]); the
                               // per-head RMSNorm + RoPE + cache append run in the following phase (llama_decode.cu ld_qknorm)
  int plan_id;                 // index into GemvRing::plans_s (>= 0) or -1: plan on the fly
  // K-chunked operand (gemv_mma_chunked): kc > 0 -> the 16-bit activation [B, K] is NOT staged by the caller; it is staged
  // here kc columns at a time from xsrc (row stride xsrc_ld), so a K wider than shared memory allows serves large batches
  const void* xsrc; int xsrc_ld; int kc;
};

// epilogue of the row pair (row0, row0 + 1), row0 even, for session b.  v already carries the bias.
// LLAMA selects which modes exist in the instantiation (smaller code per model family).  Kept inline: with ~220 KB of
// the SM's 256 KB configured as shared memory the L1 data cache is tiny, so the stack traffic of a call (argument
// struct, saved registers) goes to L2 on every phase for a non-inlined epilogue / argument builder.
template <typename T, bool LLAMA>
__device__ __forceinline__ void gemv_pair_epilogue(const GemvArgs& a, int mode, int row0, int b, float v0, float v1,
                                                   float r0, float r1, int sup0, int sup1, float& best_v, int& best_i) {
  if (mode == EPI_STORE) {
    *reinterpret_cast<float2*>(a.out + (long long)b * a.ldo + row0) = make_float2(v0, v1);
  } else if (!LLAMA && mode == EPI_GELU) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(a.out_h) + (long long)b * a.ldh + row0) = DT<T>::pack2(gelu_erf(v0), gelu_erf(v1));
  } else if (mode == EPI_RESID) {
    *reinterpret_cast<float2*>(a.out + (long long)b * a.ldo + row0) = make_float2(r0 + v0, r1 + v1);
  } else if (!LLAMA && mode == EPI_QKV) {
    if (row0 < a.d) {
      *reinterpret_cast<float2*>(a.out + (long long)b * a.ldo + row0) = make_float2(v0, v1);
    } else {
      const int which = (row0 < 2 * a.d) ? 0 : 1;
      T* dst = reinterpret_cast<T*>(a.kv0) + which * a.kv_which + b * a.kv_batch + (row0 - (which + 1) * a.d);
      *reinterpret_cast<uint32_t*>(dst) = DT<T>::pack2(v0, v1);
    }
  } else if (mode == EPI_LOGITS) {
    if ((sup0 & 1) || (a.first_step && (sup0 & 2))) v0 = -INFINITY;
    if ((sup1 & 1) || (a.first_step && (sup1 & 2))) v1 = -INFINITY;
    const bool ok1 = row0 + 1 < a.N;
    if (a.logits_out) {
      a.logits_out[b * a.logits_ld + row0] = v0;
      if (ok1) a.logits_out[b * a.logits_ld + row0 + 1] = v1;
    }
    if (v0 > best_v || (v0 == best_v && row0 < best_i)) { best_v = v0; best_i = row0; }
    if (ok1 && (v1 > best_v || (v1 == best_v && row0 + 1 < best_i))) { best_v = v1; best_i = row0 + 1; }
  } else if (LLAMA && mode == EPI_SWIGLU) {
    reinterpret_cast<T*>(a.out_h)[(long long)b * a.ldh + (row0 >> 1)] = DT<T>::from_f((v0 / (1.0f + __expf(-v0))) * v1);
  } else if (LLAMA) {  // EPI_QKV_ROPE
    const int kv_end = a.q_rows + a.k_rows;
    const int p = __ldcg(a.pos + b);
    if (a.kraw && row0 < kv_end) {
      float* dst = row0 < a.q_rows ? a.out + (long long)b * a.ldo + row0 : a.kraw + (long long)b * a.k_rows + (row0 - a.q_rows);
      *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
      return;
    }
    if (row0 < kv_end) {
      const float2 cs = a.rope[(long long)p * (a.hd >> 1) + ((row0 % a.hd) >> 1)];
      const float t0 = v0 * cs.x - v1 * cs.y, t1 = v1 * cs.x + v0 * cs.y;
      v0 = t0; v1 = t1;
    }
    if (row0 < a.q_rows) {
      *reinterpret_cast<float2*>(a.out + (long long)b * a.ldo + row0) = make_float2(v0 * a.q_scale, v1 * a.q_scale);
    } else {
      const int which = (row0 < kv_end) ? 0 : 1;
      const int c = row0 - (which ? kv_end : a.q_rows);
      T* dst = reinterpret_cast<T*>(a.kv0) + which * a.kv_which + (long long)a.slot[b] * a.kv_slot + (long long)p * a.kv_ld + c;
      *reinterpret_cast<uint32_t*>(dst) = DT<T>::pack2(v0, v1);
    }
  }
}

// ---- weight streaming through a per-warp shared-memory ring filled by the bulk-copy engine ---------------
// Each warp owns `slots` slots of GV_ROWS x GV_UK 16-bit weights.  Lane 0 issues ONE cp.async.bulk per unit
// (global -> shared, completion on the slot's mbarrier; one request per 4 KB keeps the per-SM copy engine far from
// its request-rate limit, which 512-byte row copies approach); the warp then feeds the tensor core from
// shared memory.  Bytes in flight are bounded by shared memory (16 KB per warp), not by registers, and the copies
// are not droppable hints.  The warp is its own producer and consumer, so no cross-warp synchronisation is needed:
// slot reuse is ordered by program order + __syncwarp + fence.proxy.async.
struct GemvPlan {
  int n_tiles;       // ceil(N / 8)
  int main_rounds;   // rounds in which every warp of the grid owns one whole tile
  int tail_base;     // first tile of the tail
  int ks_log;        // tail: 2^ks_log warps share a tile, each streams K >> ks_log
  int slice;         // K >> ks_log
  int tail_rounds;   // tail rounds of this CTA (uniform over its warps)
  // The CTAs that share the projection and what they share.  Whole-grid projection: vgrid = gridDim.x, vbid =
  // blockIdx.x, identity tile map, whole rows.  Cluster-local projection (whisper_decode cluster kernel): the vgrid
  // CTAs of a cluster cut `n_tiles` LOCAL tiles; local tile lt is global tile map_base + (lt >> map_gshift) *
  // map_gstride + (lt & mask) (e.g. the q, k and v rows of one head), and only columns [k_off, k_off + K) of the
  // k_full-long weight rows are multiplied (e.g. one head's slice of an out-projection).
  int vgrid, vbid, map_base, map_gshift, map_gstride, k_off, k_full;
};
__host__ __device__ __forceinline__ int gemv_global_tile(const GemvPlan& pl, int lt) {
  return pl.map_base + (lt >> pl.map_gshift) * pl.map_gstride + (lt & ((1 << pl.map_gshift) - 1));
}

struct GemvRing {
  uint32_t base_s;       // this warp's ring: 32-bit shared-space address (16-byte aligned)
  uint32_t bars_s;       // this warp's mbarriers [slots], shared-space address
  int slots;
  unsigned int slot;     // next slot to consume and its phase parity; persist across phases (all lanes identical)
  unsigned int parity;
  // the NEXT gemv, prepared by gemv_prefetch(): its plan and the producer cursor after the units already issued
  int pre_valid, pre_pj, pre_pu, pre_nvalid;
  const void* pre_W;
  GemvPlan plan;
  const GemvPlan* plans_s;  // shared memory: plans of the kernel's projection shapes, computed once at kernel start
};

__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ uint4 lds16(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ void mbar_wait_s(uint32_t bar, uint32_t parity) {
  uint32_t ok, spins = 0;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (!ok && ++spins > (1u << 26)) __trap();
  } while (!ok);
}

// D[16x8] += A[16x16] * B[16x8], fp32 accumulate; a0/a2 = sessions 0-7 (k low / high half), a1/a3 = sessions 8-15
template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1);
template <>
__device__ __forceinline__ void mma16816<__half>(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                        uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// How n_tiles (local) tiles x K columns are cut into warp items on a (virtual) grid of vgrid CTAs.  K % 32 == 0.
__host__ __device__ __forceinline__ void gemv_make_plan_ex(int n_tiles, int K, int vgrid, int vbid, GemvPlan& pl) {
  const int grid = vgrid;
  const int slots = grid * DEC_WARPS;
  pl.n_tiles = n_tiles;
  pl.main_rounds = pl.n_tiles / slots;
  pl.tail_base = pl.main_rounds * slots;
  const int tail = pl.n_tiles - pl.tail_base;
  int best_log = 0, best_cost = 0x7fffffff;
#pragma unroll
  for (int lg = 0; lg <= 3; ++lg) {
    const int sl = K >> lg;
    if ((sl & 31) == 0 && sl >= 32) {
      const int per_round = grid * (DEC_WARPS >> lg);
      const int rounds = (tail + per_round - 1) / per_round;
      const int cost = rounds * (GV_LAT_ELEMS + sl);
      if (cost < best_cost) { best_cost = cost; best_log = lg; }
    }
  }
  pl.ks_log = best_log;
  pl.slice = K >> best_log;
  const int stride = grid * (DEC_WARPS >> best_log);
  pl.tail_rounds = (tail > vbid) ? (tail - vbid + stride - 1) / stride : 0;
  pl.vgrid = vgrid; pl.vbid = vbid; pl.map_base = 0; pl.map_gshift = 30; pl.map_gstride = 0; pl.k_off = 0; pl.k_full = K;
}
// whole-grid projection [N, K]
__device__ __forceinline__ void gemv_make_plan(int N, int K, GemvPlan& pl) {
  gemv_make_plan_ex((N + GV_ROWS - 1) >> 3, K, (int)gridDim.x, (int)blockIdx.x, pl);
}

// item j of warp `warp`: which (local) tile, which K range.  Tiles are interleaved across CTAs so that consecutive tiles
// stream on different SMs.  Returns false for an empty tail slot.
__host__ __device__ __forceinline__ bool gemv_item(const GemvPlan& pl, int K, int j, int warp, int& tile, int& k0, int& klen) {
  if (j < pl.main_rounds) {
    tile = (j * DEC_WARPS + warp) * pl.vgrid + pl.vbid; k0 = 0; klen = K;
    return true;
  }
  const int r = j - pl.main_rounds;
  const int sub = warp >> pl.ks_log, sl = warp & ((1 << pl.ks_log) - 1);
  tile = pl.tail_base + (r * (DEC_WARPS >> pl.ks_log) + sub) * pl.vgrid + pl.vbid;
  k0 = sl * pl.slice; klen = pl.slice;
  return tile < pl.n_tiles;
}

// producer side of unit u of item j (whole warp calls; lane 0 issues one contiguous bulk copy)
template <typename T>
__device__ __forceinline__ void gemv_issue_unit(const T* __restrict__ Wt, int K, const GemvPlan& pl, int j, int u,
                                                uint32_t dst, uint32_t bar) {
  int tile, k0, klen;
  gemv_item(pl, K, j, threadIdx.x >> 5, tile, k0, klen);
  const int kb = k0 + u * GV_UK;
  const int len = min(GV_UK, k0 + klen - kb);
  if ((threadIdx.x & 31) == 0) {
    const uint32_t bytes = (uint32_t)(GV_ROWS * len * 2);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic-proxy reads of the slot are done
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    bulk_g2s(dst, Wt + ((long long)gemv_global_tile(pl, tile) * pl.k_full + pl.k_off + kb) * GV_ROWS, bytes, bar);
  }
}

__host__ __device__ __forceinline__ int gemv_units_of(const GemvPlan& pl, int K, int j) {
  return ((j < pl.main_rounds ? K : pl.slice) + GV_UK - 1) >> 8;
}

// Plan the gemv and issue its first `slots` units into the (empty) ring.  Called between grid_arrive and
// grid_wait of the phase BEFORE the one that consumes them: the weight stream of the next projection is already
// landing in shared memory while the chip synchronises.
template <typename T>
__device__ __forceinline__ void gemv_prefetch(const GemvArgs& a, GemvRing& ring) {
  static_assert(GV_UK == 256, "gemv_units_of shifts by 8");
  // the ring state is ONE copy per warp in shared memory: lane 0 writes it, __syncwarp publishes it to the other lanes
  // (every lane writing the same values is the same hardware behaviour but a data race on paper -- racecheck flags it)
  const int lane0 = (threadIdx.x & 31) == 0;
  if (lane0) { if (a.plan_id >= 0) ring.plan = ring.plans_s[a.plan_id]; else gemv_make_plan(a.N, a.K, ring.plan); }
  __syncwarp();
  const GemvPlan& pl = ring.plan;
  const int warp = threadIdx.x >> 5;
  int nv = pl.main_rounds;
#pragma unroll 1
  for (int r = 0; r < pl.tail_rounds; ++r) {
    int tile, k0, klen;
    if (!gemv_item(pl, a.K, pl.main_rounds + r, warp, tile, k0, klen)) break;
    ++nv;
  }
  int pj = 0, pu = 0;
  unsigned int pslot = ring.slot;
#pragma unroll 1
  for (int n = 0; n < ring.slots && pj < nv; ++n) {
    gemv_issue_unit<T>(reinterpret_cast<const T*>(a.W), a.K, pl, pj, pu, ring.base_s + pslot * GV_SLOT_BYTES, ring.bars_s + pslot * 8);
    if (++pu == gemv_units_of(pl, a.K, pj)) { pu = 0; ++pj; }
    if (++pslot == (unsigned)ring.slots) pslot = 0;
  }
  __syncwarp();
  if (lane0) { ring.pre_nvalid = nv; ring.pre_valid = 1; ring.pre_W = a.W; ring.pre_pj = pj; ring.pre_pu = pu; }
  __syncwarp();
}

// Wait for prefetched units that will never be consumed (early exit) so no bulk copy is in flight at CTA exit.
__device__ __forceinline__ void gemv_drain(int K, GemvRing& ring) {
  if (!ring.pre_valid) return;
  const GemvPlan& pl = ring.plan;
  int total = 0;
  for (int j = 0; j < ring.pre_nvalid && total < ring.slots; ++j) total += gemv_units_of(pl, K, j);
  const int n_units = min(ring.slots, total);
  unsigned int cslot = ring.slot, cpar = ring.parity;
  for (int u = 0; u < n_units; ++u) {
    mbar_wait_s(ring.bars_s + cslot * 8, cpar);
    if (++cslot == (unsigned)ring.slots) { cslot = 0; cpar ^= 1u; }
  }
  __syncwarp();
  if ((threadIdx.x & 31) == 0) { ring.pre_valid = 0; ring.slot = cslot; ring.parity = cpar; }
  __syncwarp();
}

// best_v / best_i: running argmax of this lane for sessions g and g + 8 (EPI_LOGITS).
// red_s: 2 * DEC_THREADS float4 (tail-round partial fragments, double-buffered by round parity).
template <typename T, bool LLAMA>
__device__ __noinline__ void gemv_mma(const GemvArgs& a, uint32_t xh_s, int B, float (&best_v)[2], int (&best_i)[2],
                                      GemvRing& ring, float4* red_s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const T* __restrict__ W = reinterpret_cast<const T*>(a.W);
  const int N = a.N, K = a.K, mode = a.mode;
  if (ring.pre_valid && ring.pre_W != a.W) __trap();  // prefetch bookkeeping bug: the ring holds another matrix
  if (!ring.pre_valid) gemv_prefetch<T>(a, ring);
  const GemvPlan pl = ring.plan;
  int pj = ring.pre_pj, pu = ring.pre_pu;  // producer cursor (uniform over the warp)
  const int n_valid = ring.pre_nvalid;
  const unsigned int slot_in = ring.slot, parity_in = ring.parity;
  __syncwarp();                            // every lane has read the ring state before lane 0 updates it
  if (lane == 0) ring.pre_valid = 0;
  const int n_items = pl.main_rounds + pl.tail_rounds;
  const int ks = 1 << pl.ks_log;
  unsigned int cslot = slot_in, cpar = parity_in;
  const uint32_t xrow_lo = xh_s + (uint32_t)(g * (K + GV_XPAD) + t * 8) * 2;
  const uint32_t xrow_hi = xrow_lo + (uint32_t)(8 * (K + GV_XPAD)) * 2;
  const bool lo = g < B, hi = g + 8 < B;
  const uint32_t wlane = (uint32_t)lane * 16;
#pragma unroll 1
  for (int j = 0; j < n_items; ++j) {
    int tile, k0, klen;
    const bool valid = gemv_item(pl, K, j, warp, tile, k0, klen);
    const bool split = (j >= pl.main_rounds) && ks > 1;
    const bool owner = valid && (!split || (warp & (ks - 1)) == 0);  // this warp runs the tile's epilogue
    const int row0 = gemv_global_tile(pl, tile) * GV_ROWS + 2 * t;  // this lane's row pair
    const bool rows_ok = owner && row0 < N;
    // epilogue operands first: their round trip overlaps the weight stream
    float bias0 = 0.f, bias1 = 0.f, rl0 = 0.f, rl1 = 0.f, rh0 = 0.f, rh1 = 0.f;
    int sup0 = 0, sup1 = 0;
    if (rows_ok) {
      if (a.bias) { const float2 bb = __ldg(reinterpret_cast<const float2*>(a.bias + row0)); bias0 = bb.x; bias1 = bb.y; }
      if (mode == EPI_RESID) {
        if (lo) { const float2 r = __ldcg(reinterpret_cast<const float2*>(a.out + (long long)g * a.ldo + row0)); rl0 = r.x; rl1 = r.y; }
        if (hi) { const float2 r = __ldcg(reinterpret_cast<const float2*>(a.out + (long long)(g + 8) * a.ldo + row0)); rh0 = r.x; rh1 = r.y; }
      } else if (mode == EPI_LOGITS && a.suppress) {
        sup0 = __ldg(a.suppress + row0);
        sup1 = __ldg(a.suppress + min(row0 + 1, N - 1));
      }
    }
    float c[4] = {0.f, 0.f, 0.f, 0.f}, e[4] = {0.f, 0.f, 0.f, 0.f};  // two independent accumulator fragments
    if (valid) {
      const int upi = (klen + GV_UK - 1) >> 8;
#pragma unroll 1
      for (int u = 0; u < upi; ++u) {
        mbar_wait_s(ring.bars_s + cslot * 8, cpar);
        const uint32_t wsrc = ring.base_s + cslot * GV_SLOT_BYTES + wlane;
        const int len = min(GV_UK, klen - u * GV_UK);
        const uint32_t xk = (uint32_t)(k0 + u * GV_UK) * 2;
#pragma unroll 4
        for (int kk = 0; kk < len; kk += 32) {
          const uint4 w = lds16(wsrc + kk * (GV_WIN_BYTES / 32));
          uint4 xl = make_uint4(0u, 0u, 0u, 0u), xu = make_uint4(0u, 0u, 0u, 0u);
          if (lo) xl = lds16(xrow_lo + xk + kk * 2);
          if (hi) xu = lds16(xrow_hi + xk + kk * 2);
          mma16816<T>(c, xl.x, xu.x, xl.y, xu.y, w.x, w.y);
          mma16816<T>(e, xl.z, xu.z, xl.w, xu.w, w.z, w.w);
        }
        __syncwarp();
        if (pj < n_valid) {  // refill the slot just drained
          gemv_issue_unit<T>(W, K, pl, pj, pu, ring.base_s + cslot * GV_SLOT_BYTES, ring.bars_s + cslot * 8);
          if (++pu == gemv_units_of(pl, K, pj)) { pu = 0; ++pj; }
        }
        if (++cslot == (unsigned)ring.slots) { cslot = 0; cpar ^= 1u; }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) c[i] += e[i];
    if (split) {
      float4* buf = red_s + (j & 1) * DEC_THREADS;
      buf[threadIdx.x] = make_float4(c[0], c[1], c[2], c[3]);
      __syncthreads();
      if (owner) {
#pragma unroll 1
        for (int s = 1; s < ks; ++s) {
          const float4 o = buf[threadIdx.x + s * 32];
          c[0] += o.x; c[1] += o.y; c[2] += o.z; c[3] += o.w;
        }
      }
    }
    if (rows_ok) {
      if (lo) gemv_pair_epilogue<T, LLAMA>(a, mode, row0, g, c[0] + bias0, c[1] + bias1, rl0, rl1, sup0, sup1, best_v[0], best_i[0]);
      if (hi) gemv_pair_epilogue<T, LLAMA>(a, mode, row0, g + 8, c[2] + bias0, c[3] + bias1, rh0, rh1, sup0, sup1, best_v[1], best_i[1]);
    }
  }
  __syncwarp();
  if (lane == 0) { ring.slot = cslot; ring.parity = cpar; }
  __syncwarp();
}

// ---- the same projection with a K-chunked activation operand ----------------------------------------------------------
// For K wider than the shared-memory operand region (Llama-3-8B down-projection: K = 14336 at 8+ sessions) the activation
// [B, K] is staged kc columns at a time while the weights keep streaming through the ring.  The CTA -> tile assignment is
// fixed over the chunks (every warp owns ONE (tile, K-slice) item: the plan of a [N, kc] projection), the accumulator
// fragments live in registers across the chunks, and the K-split reduction + epilogue run once at the end -- so the result
// is the same sum in a different association from the unchunked routine, and deterministic.
// Host side: gemv_chunk_ok() says whether a shape satisfies the one-item-per-warp requirement.
__host__ __device__ inline bool gemv_chunk_ok(int N, int K, int kc, int grid) {
  if (kc <= 0 || (kc & 255) != 0 || K <= kc) return false;
  GemvPlan pl;
  gemv_make_plan_ex((N + GV_ROWS - 1) >> 3, kc, grid, 0, pl);
  if (pl.main_rounds != 0) return false;
  const int tail = pl.n_tiles, per_round = grid * (DEC_WARPS >> pl.ks_log);
  if (tail > per_round) return false;                       // more than one item per warp
  const int last = K % kc == 0 ? kc : K % kc;
  return (last % (32 << pl.ks_log)) == 0;                   // the short last chunk still splits into whole k-windows
}

template <typename T, bool LLAMA>
__device__ __noinline__ void gemv_mma_chunked(const GemvArgs& a, T* xh, int B, float (&best_v)[2], int (&best_i)[2], GemvRing& ring,
                                              float4* red_s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const T* __restrict__ W = reinterpret_cast<const T*>(a.W);
  const T* __restrict__ X = reinterpret_cast<const T*>(a.xsrc);
  const int N = a.N, K = a.K, KC = a.kc, mode = a.mode;
  const int n_chunks = (K + KC - 1) / KC;
  if (ring.pre_valid) __trap();                            // chunked projections are never prefetched across the barrier
  GemvPlan pl;
  gemv_make_plan(N, KC, pl);
  if (pl.main_rounds != 0 || pl.tail_rounds > 1) __trap();  // gemv_chunk_ok() was not honoured by the launcher
  const int ks = 1 << pl.ks_log, sl = warp & (ks - 1);
  int tile, k0_full, klen_full;
  const bool valid = pl.tail_rounds == 1 && gemv_item(pl, KC, 0, warp, tile, k0_full, klen_full);
  const bool owner = valid && sl == 0;
  const int row0 = tile * GV_ROWS + 2 * t;
  const bool rows_ok = owner && row0 < N;
  float bias0 = 0.f, bias1 = 0.f, rl0 = 0.f, rl1 = 0.f, rh0 = 0.f, rh1 = 0.f;
  const bool lo = g < B, hi = g + 8 < B;
  if (rows_ok) {
    if (a.bias) { const float2 bb = __ldg(reinterpret_cast<const float2*>(a.bias + row0)); bias0 = bb.x; bias1 = bb.y; }
    if (mode == EPI_RESID) {
      if (lo) { const float2 r = __ldcg(reinterpret_cast<const float2*>(a.out + (long long)g * a.ldo + row0)); rl0 = r.x; rl1 = r.y; }
      if (hi) { const float2 r = __ldcg(reinterpret_cast<const float2*>(a.out + (long long)(g + 8) * a.ldo + row0)); rh0 = r.x; rh1 = r.y; }
    }
  }
  // producer cursor over this warp's unit stream: chunk pc, unit pu inside the chunk's slice
  auto slice_of = [&](int c) { const int kcc = min(KC, K - c * KC); return kcc >> pl.ks_log; };
  int pc = 0, pu = 0;
  const unsigned int slot_in = ring.slot, parity_in = ring.parity;
  unsigned int pslot = slot_in;
  auto issue_next = [&](uint32_t dst, uint32_t bar) {
    const int slice = slice_of(pc);
    const int kb = pc * KC + sl * slice + pu * GV_UK;
    const int len = min(GV_UK, slice - pu * GV_UK);
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)(GV_ROWS * len * 2);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
      bulk_g2s(dst, W + ((long long)tile * K + kb) * GV_ROWS, bytes, bar);
    }
    if (++pu * GV_UK >= slice) { pu = 0; ++pc; }
  };
  if (valid)
    for (int n = 0; n < ring.slots && pc < n_chunks; ++n) {
      issue_next(ring.base_s + pslot * GV_SLOT_BYTES, ring.bars_s + pslot * 8);
      if (++pslot == (unsigned)ring.slots) pslot = 0;
    }
  unsigned int cslot = slot_in, cpar = parity_in;
  const uint32_t xh_s = smem_u32(xh);
  const uint32_t row_bytes = (uint32_t)(KC + GV_XPAD) * 2;
  const uint32_t xrow_lo = xh_s + (uint32_t)g * row_bytes + (uint32_t)t * 16;
  const uint32_t xrow_hi = xrow_lo + 8u * row_bytes;
  const uint32_t wlane = (uint32_t)lane * 16;
  float c[4] = {0.f, 0.f, 0.f, 0.f}, e[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
  for (int ch = 0; ch < n_chunks; ++ch) {
    const int kcc = min(KC, K - ch * KC);
    if (ch > 0) __syncthreads();                           // every warp is done with the previous chunk's operand
    {   // stage columns [ch * KC, ch * KC + kcc) of the B rows
      const int vpr = kcc >> 3, n = B * vpr;
      int row = threadIdx.x / vpr, col = threadIdx.x - row * vpr;
#pragma unroll 2
      for (int i = threadIdx.x; i < n; i += DEC_THREADS) {
        cp_async16(xh_s + row * row_bytes + (uint32_t)col * 16, reinterpret_cast<const uint4*>(X + (long long)row * a.xsrc_ld + ch * KC) + col);
        col += DEC_THREADS;
        while (col >= vpr) { col -= vpr; ++row; }
      }
      cp_async_wait_all();
      __syncthreads();
    }
    if (valid) {
      const int slice = kcc >> pl.ks_log, k0 = sl * slice, upi = (slice + GV_UK - 1) >> 8;
#pragma unroll 1
      for (int u = 0; u < upi; ++u) {
        mbar_wait_s(ring.bars_s + cslot * 8, cpar);
        const uint32_t wsrc = ring.base_s + cslot * GV_SLOT_BYTES + wlane;
        const int len = min(GV_UK, slice - u * GV_UK);
        const uint32_t xk = (uint32_t)(k0 + u * GV_UK) * 2;
#pragma unroll 4
        for (int kk = 0; kk < len; kk += 32) {
          const uint4 w = lds16(wsrc + kk * (GV_WIN_BYTES / 32));
          uint4 xl = make_uint4(0u, 0u, 0u, 0u), xu = make_uint4(0u, 0u, 0u, 0u);
          if (lo) xl = lds16(xrow_lo + xk + kk * 2);
          if (hi) xu = lds16(xrow_hi + xk + kk * 2);
          mma16816<T>(c, xl.x, xu.x, xl.y, xu.y, w.x, w.y);
          mma16816<T>(e, xl.z, xu.z, xl.w, xu.w, w.z, w.w);
        }
        __syncwarp();
        if (pc < n_chunks) issue_next(ring.base_s + cslot * GV_SLOT_BYTES, ring.bars_s + cslot * 8);   // refill the slot just drained
        if (++cslot == (unsigned)ring.slots) { cslot = 0; cpar ^= 1u; }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) c[i] += e[i];
  if (ks > 1) {
    red_s[threadIdx.x] = make_float4(c[0], c[1], c[2], c[3]);
    __syncthreads();
    if (owner)
#pragma unroll 1
      for (int s = 1; s < ks; ++s) {
        const float4 o = red_s[threadIdx.x + s * 32];
        c[0] += o.x; c[1] += o.y; c[2] += o.z; c[3] += o.w;
      }
  }
  if (rows_ok) {
    if (lo) gemv_pair_epilogue<T, LLAMA>(a, mode, row0, g, c[0] + bias0, c[1] + bias1, rl0, rl1, 0, 0, best_v[0], best_i[0]);
    if (hi) gemv_pair_epilogue<T, LLAMA>(a, mode, row0, g + 8, c[2] + bias0, c[3] + bias1, rh0, rh1, 0, 0, best_v[1], best_i[1]);
  }
  __syncwarp();
  if (lane == 0) { ring.slot = cslot; ring.parity = cpar; }
  __syncwarp();
}

// Per-CTA argmax candidates after an EPI_LOGITS gemv: merge the lanes of a session (t = 0..3), then the warps.
// sv / si: DEC_WARPS * DEC_MAX_B entries each.
__device__ __forceinline__ void gemv_argmax_candidates(float (&best_v)[2], int (&best_i)[2], int B, float* sv, int* si,
                                                       float* cand_val, int* cand_idx) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float bv = best_v[hh]; int bi = best_i[hh];
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (t == 0) { sv[warp * DEC_MAX_B + g + 8 * hh] = bv; si[warp * DEC_MAX_B + g + 8 * hh] = bi; }
  }
  __syncthreads();
  if (threadIdx.x < B) {
    const int b = threadIdx.x;
    float bv = -INFINITY; int bi = 0x7fffffff;
#pragma unroll 1
    for (int wv = 0; wv < DEC_WARPS; ++wv) {
      const float v = sv[wv * DEC_MAX_B + b]; const int i = si[wv * DEC_MAX_B + b];
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    cand_val[b * gridDim.x + blockIdx.x] = bv;
    cand_idx[b * gridDim.x + blockIdx.x] = bi;
  }
}

// ---- attention: CTA-level items ------------------------------------------------------------------------------
// One item = (session, head, key split).  The 8 warps of the CTA stride over the item's 32-key blocks; each warp keeps
// a running (m, l, o) over its blocks (one memory round trip per block: the 8 K and 8 V vectors of a block are
// loaded before any arithmetic; 8 lanes cover one key row), the warp records meet in shared memory and warp 0
// merges them into ONE global record [o[HD] unnormalised, m, l] per item.  The consumer phase (out-projection)
// therefore merges only `splits` records per (session, head) -- 1 when sessions x heads already cover the grid --
// instead of one record per 64 keys, which at 16 sessions made every CTA re-read 1.2 MB of records per layer.
constexpr int ATT_BLK = 32;

// How an attention phase is cut into items.  A warp walks its 32-key blocks serially (one memory round trip each).
//   CTA-level item  = (session, head, split): the 8 warps stride over the split's blocks, merge in shared memory;
//                     best when sessions x heads is small (few, short items; 1 block per warp at batch 1).
//   warp-level item = (session, head, split) owned by ONE warp, no CTA synchronisation at all; best when
//                     sessions x heads x splits can occupy every warp of the grid (large batches).
// Either way a split leaves one record and the last split to finish merges them (attn_finish_item).  The plan
// minimises  rounds x (serial blocks per item + ~2 block-times of finishing), CTA-level on ties.
// Returns splits | (warp_level << 7); splits <= 16 (CTA) / 32 (warp), bounded by the blocks and the record storage.
constexpr int ATTN_WARP_LEVEL = 0x80;
__host__ __device__ inline int attn_plan(int BH, int n_blocks, int s_max, int grid) {
  int best = 1, best_cost = 0x7fffffff;
  const int lim = n_blocks < s_max ? n_blocks : s_max;
  for (int S = 1; S <= (lim < 16 ? lim : 16); ++S) {
    const int bps = (n_blocks + S - 1) / S;
    const int cost = ((BH * S + grid - 1) / grid) * ((bps + DEC_WARPS - 1) / DEC_WARPS + 2);
    if (cost < best_cost) { best_cost = cost; best = S; }
  }
  for (int S = 1; S <= (lim < 32 ? lim : 32); ++S) {
    const int bpi = (n_blocks + S - 1) / S;
    const int cost = ((BH * S + grid * DEC_WARPS - 1) / (grid * DEC_WARPS)) * (bpi + 2);
    if (cost < best_cost) { best_cost = cost; best = S | ATTN_WARP_LEVEL; }
  }
  return best;
}

// q must already carry the softmax scale.  Blocks blk_first, blk_first + blk_stride, ... < blk_end (all start
// below n_keys).  Writes this warp's record (shared memory): m = -inf, l = 0, o = 0 if it had no block.
template <typename T, int HD>
__device__ __noinline__ void attend_blocks(const float* q /*global fp32 [HD]*/, const T* K, const T* V, long long ldk,
                                           long long ldv, int n_keys, int blk_first, int blk_end, int blk_stride, float* rec) {
  constexpr int PER = HD / 8;      // elements per lane
  constexpr int NV = PER / 8;      // 16-byte vectors per lane
  constexpr int KH = 8;            // keys per lane slot per block
  const int lane = threadIdx.x & 31;
  const int g = lane >> 3, j = lane & 7;
  float qr[PER];
#pragma unroll
  for (int i = 0; i < PER; i += 4) {
    const float4 t = __ldcg(reinterpret_cast<const float4*>(q + j * PER + i));
    qr[i] = t.x; qr[i + 1] = t.y; qr[i + 2] = t.z; qr[i + 3] = t.w;
  }
  float m = -INFINITY, l = 0.f;
  float o[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) o[i] = 0.f;

#pragma unroll 1
  for (int blk = blk_first; blk < blk_end; blk += blk_stride) {
    const int kbase = blk * ATT_BLK;
    if (blk + blk_stride < blk_end) {  // warm L2 with this warp's next block while the current one is in flight
      const int nk = kbase + blk_stride * ATT_BLK + lane;
      if (nk < n_keys) {
#pragma unroll
        for (int o128 = 0; o128 < HD * (int)sizeof(T); o128 += 128) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(K + (long long)nk * ldk) + o128));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(V + (long long)nk * ldv) + o128));
        }
      }
    }
    uint4 kr[KH][NV], vr[KH][NV];
#pragma unroll
    for (int i = 0; i < KH; ++i) {
      const int key = kbase + g + 4 * i;
      if (key < n_keys) {
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          kr[i][v] = __ldcg(reinterpret_cast<const uint4*>(K + (long long)key * ldk + j * PER + v * 8));
          vr[i][v] = __ldcg(reinterpret_cast<const uint4*>(V + (long long)key * ldv + j * PER + v * 8));
        }
      }
    }
    float s[KH];
    float mh = -INFINITY;
#pragma unroll
    for (int i = 0; i < KH; ++i) {
      const int key = kbase + g + 4 * i;
      float dot = 0.f;
      if (key < n_keys) {
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const float2 a = DT<T>::to_f2(kr[i][v].x), b = DT<T>::to_f2(kr[i][v].y);
          const float2 c = DT<T>::to_f2(kr[i][v].z), d = DT<T>::to_f2(kr[i][v].w);
          dot = fmaf(a.x, qr[v * 8 + 0], dot); dot = fmaf(a.y, qr[v * 8 + 1], dot);
          dot = fmaf(b.x, qr[v * 8 + 2], dot); dot = fmaf(b.y, qr[v * 8 + 3], dot);
          dot = fmaf(c.x, qr[v * 8 + 4], dot); dot = fmaf(c.y, qr[v * 8 + 5], dot);
          dot = fmaf(d.x, qr[v * 8 + 6], dot); dot = fmaf(d.y, qr[v * 8 + 7], dot);
        }
      }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      dot += __shfl_xor_sync(0xffffffffu, dot, 4);
      s[i] = (key < n_keys) ? dot : -INFINITY;
      mh = fmaxf(mh, s[i]);
    }
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, 8));
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, 16));
    const float m_new = fmaxf(m, mh);          // finite: the block holds at least one key
    const float corr = __expf(m - m_new);      // m = -inf on the first block -> 0
    l *= corr;
#pragma unroll
    for (int i = 0; i < PER; ++i) o[i] *= corr;
    m = m_new;
#pragma unroll
    for (int i = 0; i < KH; ++i) {
      const int key = kbase + g + 4 * i;
      if (key < n_keys) {
        const float p = __expf(s[i] - m);
        l += p;
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const float2 a = DT<T>::to_f2(vr[i][v].x), b = DT<T>::to_f2(vr[i][v].y);
          const float2 c = DT<T>::to_f2(vr[i][v].z), d = DT<T>::to_f2(vr[i][v].w);
          o[v * 8 + 0] = fmaf(p, a.x, o[v * 8 + 0]); o[v * 8 + 1] = fmaf(p, a.y, o[v * 8 + 1]);
          o[v * 8 + 2] = fmaf(p, b.x, o[v * 8 + 2]); o[v * 8 + 3] = fmaf(p, b.y, o[v * 8 + 3]);
          o[v * 8 + 4] = fmaf(p, c.x, o[v * 8 + 4]); o[v * 8 + 5] = fmaf(p, c.y, o[v * 8 + 5]);
          o[v * 8 + 6] = fmaf(p, d.x, o[v * 8 + 6]); o[v * 8 + 7] = fmaf(p, d.y, o[v * 8 + 7]);
        }
      }
    }
  }
  // merge the 4 key slots (lanes differing in bits 3,4): l and o are per-slot partial sums under the common m
  l += __shfl_xor_sync(0xffffffffu, l, 8);
  l += __shfl_xor_sync(0xffffffffu, l, 16);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 8);
    o[i] += __shfl_xor_sync(0xffffffffu, o[i], 16);
  }
  if (g == 0) {
#pragma unroll
    for (int i = 0; i < PER; i += 4)
      *reinterpret_cast<float4*>(rec + j * PER + i) = make_float4(o[i], o[i + 1], o[i + 2], o[i + 3]);
  }
  if (lane == 0) { rec[HD] = m; rec[HD + 1] = l; }
}

// one warp: merge n <= 32 global records [o[HD] unnormalised, m, l] of a (session, head) (one lane per record) and
// write the normalised head output as 16-bit into out16[HD] (global or shared)
template <typename T, int HD>
__device__ __forceinline__ void attn_merge_records(const float* part_bh, int n, T* out16) {
  constexpr int REC = HD + PART_PAD, DPL = HD / 32;
  const int lane = threadIdx.x & 31;
  float mc = -INFINITY, lc = 0.f;
  if (lane < n) {
    const float2 ml = __ldcg(reinterpret_cast<const float2*>(part_bh + (long long)lane * REC + HD));
    mc = ml.x; lc = ml.y;
  }
  float acc[DPL];
#pragma unroll
  for (int i = 0; i < DPL; ++i) acc[i] = 0.f;
  const float M2 = warp_max(mc);
  const float wc = (mc > -INFINITY) ? __expf(mc - M2) : 0.f;
  const float den2 = warp_sum(lc * wc);
#pragma unroll 4
  for (int u = 0; u < n; ++u) {
    const float wu = __shfl_sync(0xffffffffu, wc, u);
#pragma unroll
    for (int i = 0; i < DPL; ++i) acc[i] = fmaf(__ldcg(part_bh + (long long)u * REC + lane + 32 * i), wu, acc[i]);
  }
  const float inv = 1.f / den2;
#pragma unroll
  for (int i = 0; i < DPL; ++i) out16[lane + 32 * i] = DT<T>::from_f(acc[i] * inv);
}

// ---- finishing an attention item (warp 0 of the CTA) ---------------------------------------------------------
// Merge the n_rec warp records in shared memory (DEC_WARPS for a CTA-level item, 1 for a warp-level item).  splits == 1: the item is the whole (session, head): write the
// normalised head output as 16-bit into out16[HD].  Otherwise write the global record, then count the item in
// cnt (one counter per (session, head)); the CTA that completes the count merges the `splits` records and writes
// out16 -- so the consumer phase just copies B x d 16-bit values instead of every CTA re-merging every record.
// The grid barrier that ends the phase orders out16 before its readers; the counter is reset for the next use.
template <typename T, int HD>
__device__ __forceinline__ void attn_finish_item(const float* rec_s, int n_rec /*DEC_WARPS or 1*/, float* part_bh /*[s_max][REC]*/,
                                                 int s, int splits, unsigned int* cnt, T* out16) {
  constexpr int REC = HD + PART_PAD, DPL = HD / 32;
  const int lane = threadIdx.x & 31;
  __syncwarp();
  float mw = -INFINITY, lw = 0.f;
  if (lane < n_rec) { mw = rec_s[lane * REC + HD]; lw = rec_s[lane * REC + HD + 1]; }
  const float M = warp_max(mw);
  const float wt = (mw > -INFINITY) ? __expf(mw - M) : 0.f;  // empty warp records (and an all-empty item) weigh 0
  const float den = warp_sum(lw * wt);
  float o[DPL];
#pragma unroll
  for (int i = 0; i < DPL; ++i) o[i] = 0.f;
#pragma unroll
  for (int w = 0; w < DEC_WARPS; ++w) {
    if (w < n_rec) {
      const float ww = __shfl_sync(0xffffffffu, wt, w);
#pragma unroll
      for (int i = 0; i < DPL; ++i) o[i] = fmaf(rec_s[w * REC + lane + 32 * i], ww, o[i]);
    }
  }
  if (splits == 1) {
    const float inv = 1.f / den;
#pragma unroll
    for (int i = 0; i < DPL; ++i) out16[lane + 32 * i] = DT<T>::from_f(o[i] * inv);
    return;
  }
  float* out = part_bh + (long long)s * REC;
#pragma unroll
  for (int i = 0; i < DPL; ++i) out[lane + 32 * i] = o[i];
  if (lane == 0) { out[HD] = M; out[HD + 1] = den; }
  if (!cnt) return;  // the caller orders and merges the records itself (cluster kernel: barrier.cluster)
  __syncwarp();
  unsigned int prev = 0;
  if (lane == 0)  // release: the record (all lanes, ordered by the __syncwarp) happens-before the count; acquire: the
                  // other splits' records happen-before the merge below (read with ld.global.cg)
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(prev) : "l"(cnt) : "memory");
  prev = __shfl_sync(0xffffffffu, prev, 0);
  if (prev != (unsigned)splits - 1) return;
  // last split of this (session, head): merge the records
  attn_merge_records<T, HD>(part_bh, splits, out16);
  if (lane == 0) *cnt = 0u;
}
