// llama_decode_plan.cuh -- shared-memory plan of a persistent Llama-family decode launch (host side; the kernel derives the
// same layout from the plan's fields).  Kept in a header of its own so that tests/dev/decode_plan_check.cu can tabulate it
// without a GPU.
#pragma once
#include <algorithm>

#include "decode_common.cuh"

__host__ __device__ inline int ld_kmax(int d, int ffn, int qd) { return (d > ffn ? d : ffn) > qd ? (d > ffn ? d : ffn) : qd; }

// kmax = widest operand staged whole, rg = statistics rows per group (DEC_NORM_L2: no fp32 copy), kc = down-projection chunk
// (0 = unchunked), slots = weight-ring slots per warp.  assoc_b: the batch whose plan fixes the two reduction orders that
// depend on the batch rather than on the geometry -- the RMSNorm statistics (warps per row) and the attention split plan
// (attn_plan over assoc_b x heads items).  It is B in the first two tiers; in the third it is the batch of half a full
// launch, whose plan reduces the same way, so a session's arithmetic is that of the half launch it would otherwise be in.
struct LlamaDecPlan { int kmax, rg, kc, slots, assoc_b; };
constexpr int LD_ASSOC_B_L2 = DEC_MAX_B / 2;

// warps per row of norm_from_smem for a group of `rows` rows
inline int ld_norm_wpr(int rows) {
  int wpr = DEC_WARPS;
  while (wpr > 1 && wpr * rows > DEC_WARPS) wpr >>= 1;
  return wpr;
}

// Shared-memory plan of a batch on `grid` CTAs with `max_dyn` bytes of dynamic shared memory, in order of preference:
//   1. everything staged whole in one round trip (rg = B, kc = 0);
//   2. the ffn-wide down-projection operand in K-chunks of max(d, qd) columns and the fp32 statistics copy walked in row
//      groups (largest power of two that fits) -- Llama-3-8B: 4 sessions whole, up to 12 with chunks;
//   3. chunks as in 2 and no fp32 copy at all (rg = DEC_NORM_L2: stage_rows_norm_l2, 2 warps per row, the statistics order
//      of a 4-row group) -- Llama-3-8B: 13 to 16 sessions, with assoc_b = 8, whose plan is tier 2 with rg = 4.
// Each tier needs >= 2 weight-ring slots per warp; returns false when the batch does not fit.
inline bool llama_decode_plan(int B, int d, int ffn, int qd, int grid, long long max_dyn, LlamaDecPlan* pl) {
  {
    const int km = ld_kmax(d, ffn, qd);
    const int s = dec_ring_slots(dec_smem_layout(B, d, km, d, B), max_dyn);
    if (s >= 2) { *pl = LlamaDecPlan{km, B, 0, s, B}; return true; }
  }
  const int lim = ((std::max(d, qd) + 255) / 256) * 256;     // chunk = the widest operand that is staged whole anyway
  if (ffn <= lim || !gemv_chunk_ok(d, ffn, lim, grid)) return false;
  const int km = ld_kmax(d, lim, qd);
  for (int g = B; g >= 2; g >>= 1) {
    int gg = 1;
    while (gg * 2 <= g) gg *= 2;
    const int s = dec_ring_slots(dec_smem_layout(B, d, km, d, gg), max_dyn);
    if (s >= 2) { *pl = LlamaDecPlan{km, gg, lim, s, B}; return true; }
  }
  if (B <= LD_ASSOC_B_L2 || d > NORM_L2_MAX_D) return false;
  LlamaDecPlan half;   // the launch a session would otherwise be in must reduce exactly like stage_rows_norm_l2
  if (!llama_decode_plan(LD_ASSOC_B_L2, d, ffn, qd, grid, max_dyn, &half) || half.kc != lim || half.rg <= 0 ||
      LD_ASSOC_B_L2 % half.rg != 0 || ld_norm_wpr(half.rg) != NORM_L2_WPR)
    return false;
  const int s = dec_ring_slots(dec_smem_layout(B, d, km, d, DEC_NORM_L2), max_dyn);
  if (s >= 2) { *pl = LlamaDecPlan{km, DEC_NORM_L2, lim, s, LD_ASSOC_B_L2}; return true; }
  return false;
}

// largest batch per launch on `grid` CTAs that has a plan
inline int llama_decode_plan_max_batch(int d, int ffn, int qd, int grid, long long max_dyn) {
  LlamaDecPlan pl;
  for (int B = DEC_MAX_B; B >= 1; --B)
    if (llama_decode_plan(B, d, ffn, qd, grid, max_dyn, &pl)) return B;
  return 0;
}
