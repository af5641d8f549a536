// Host-side check of the Llama-family decode launch's shared-memory plan (llama_decode_plan.cuh), no GPU needed:
//  - Llama-3-8B plans 16 sessions per launch on a whole H100 (132 CTAs) and on one of two SM partitions (66 CTAs), with >= 2
//    weight-ring slots per warp, inside the sm_90 per-block opt-in limit next to the kernel's static shared memory, and with
//    the reduction orders (assoc_b) of the 8-session launch;
//  - every batch that had a plan under the previous planner (a fixed 220 KB budget, two tiers) keeps that plan (kmax, rg,
//    kc; at least as many ring slots) and assoc_b = B: Llama-3-8B up to 12 sessions, the Qwen3-TTS talker and code predictor and the
//    micro geometries up to 16.
// Built and run by tests/test_decode_smem_plan.py; prints the Llama-3-8B table.
#include <cstdio>
#include "../../speech_to_speech_b200/csrc/llama_decode_plan.cuh"

constexpr long long SM90_OPTIN = 232448;      // cudaDevAttrMaxSharedMemoryPerBlockOptin of sm_90
constexpr long long LD_STATIC_SMEM = 6144;    // llama_decode_kernel's static shared memory (nvcc -Xptxas -v)
constexpr long long MAX_DYN = SM90_OPTIN - LD_STATIC_SMEM;

// the previous planner, restated: ring slots against a fixed 220 KB budget, whole or K-chunked with fp32 row groups
static int old_slots(const DecSmem& L) {
  const long long avail = 220LL * 1024 - (long long)L.ring_off - 256;
  const long long s = avail / ((long long)DEC_WARPS * (GV_SLOT_BYTES + 8));
  return (int)(s > 4 ? 4 : s);
}
static bool old_plan(int B, int d, int ffn, int qd, int grid, LlamaDecPlan* pl) {
  {
    const int km = ld_kmax(d, ffn, qd);
    const int s = old_slots(dec_smem_layout(B, d, km, d, B));
    if (s >= 2) { *pl = LlamaDecPlan{km, B, 0, s, B}; return true; }
  }
  const int lim = ((std::max(d, qd) + 255) / 256) * 256;
  if (ffn <= lim || !gemv_chunk_ok(d, ffn, lim, grid)) return false;
  const int km = ld_kmax(d, lim, qd);
  for (int g = B; g >= 2; g >>= 1) {
    int gg = 1;
    while (gg * 2 <= g) gg *= 2;
    const int s = old_slots(dec_smem_layout(B, d, km, d, gg));
    if (s >= 2) { *pl = LlamaDecPlan{km, gg, lim, s, B}; return true; }
  }
  return false;
}

int main() {
  int bad = 0;
  struct Geo { const char* name; int d, ffn, qd; };
  const Geo geos[] = {{"llama-3-8b", 4096, 14336, 4096}, {"tts-12hz talker", 1024, 2048, 2048},
                      {"tts-12hz predictor", 1024, 3072, 2048}, {"mini", 1024, 3584, 1024}, {"micro", 256, 512, 256}};
  for (const Geo& g : geos)
    for (int grid : {132, 66})
      for (int B = 1; B <= DEC_MAX_B; ++B) {
        LlamaDecPlan o{}, n{};
        const bool had = old_plan(B, g.d, g.ffn, g.qd, grid, &o);
        const bool has = llama_decode_plan(B, g.d, g.ffn, g.qd, grid, MAX_DYN, &n);
        if (has) {
          const size_t dyn = dec_smem_bytes(dec_smem_layout(B, g.d, n.kmax, g.d, n.rg), n.slots);
          if (n.slots < 2 || (long long)dyn + LD_STATIC_SMEM > SM90_OPTIN) {
            printf("%s grid %d B %d: %d slots, %zu + %lld B of shared memory\n", g.name, grid, B, n.slots, dyn, LD_STATIC_SMEM); ++bad;
          }
          if (g.d == 4096) printf("%s grid %3d B %2d: kmax %5d rg %2d kc %4d slots %d assoc_b %2d dynamic %6zu B\n", g.name, grid, B,
                                  n.kmax, n.rg, n.kc, n.slots, n.assoc_b, dyn);
        }
        // the real limit is 1.2 KB above the old budget: a ring may get deeper (mini at 11 sessions: 3 -> 4 slots), never shallower
        if (had && has && n.slots != o.slots) printf("%s grid %d B %d: %d -> %d ring slots\n", g.name, grid, B, o.slots, n.slots);
        if (had && (!has || o.kmax != n.kmax || o.rg != n.rg || o.kc != n.kc || o.slots > n.slots || n.assoc_b != B)) {
          printf("%s grid %d B %d: plan changed (kmax %d rg %d kc %d slots %d -> %d %d %d %d, assoc_b %d)\n", g.name, grid, B, o.kmax,
                 o.rg, o.kc, o.slots, n.kmax, n.rg, n.kc, n.slots, n.assoc_b);
          ++bad;
        }
        if (!had && has && !(g.d == 4096 && B > 12)) { printf("%s grid %d B %d: unexpected new plan\n", g.name, grid, B); ++bad; }
        if (g.d == 4096 && B > 12) {
          LlamaDecPlan h{};
          if (!has || n.rg != DEC_NORM_L2 || n.assoc_b != 8 || !llama_decode_plan(8, g.d, g.ffn, g.qd, grid, MAX_DYN, &h) ||
              h.kc != n.kc || ld_norm_wpr(h.rg) != NORM_L2_WPR) {
            printf("%s grid %d B %d: no plan with the 8-session reduction orders\n", g.name, grid, B); ++bad;
          }
        }
      }
  for (int grid : {132, 66})
    if (llama_decode_plan_max_batch(4096, 14336, 4096, grid, MAX_DYN) != 16) { printf("llama-3-8b grid %d: max batch < 16\n", grid); ++bad; }
  printf(bad ? "FAILED %d\n" : "OK\n", bad);
  return bad ? 1 : 0;
}
