// Host-side check of the decode kernels' work decomposition (decode_common.cuh: gemv_make_plan_ex / gemv_item /
// gemv_global_tile / attn_plan): for every projection shape of the supported geometries, on the whole grid and on the
// cluster-local sub-plans, every (tile, k) is covered exactly once, slices are multiples of 32, and the ring-unit
// bookkeeping adds up.  Built and run by tests/test_gemv_plan.py (no GPU needed).
#include <cstdio>
#include <map>
#include <vector>
#include <algorithm>
#include "../../speech_to_speech_b200/csrc/decode_common.cuh"

static int check(int n_tiles, int K, int vgrid, int map_base, int gshift, int gstride, const char* what) {
  std::map<int, std::vector<std::pair<int, int>>> cover;
  for (int bid = 0; bid < vgrid; ++bid) {
    GemvPlan pl;
    gemv_make_plan_ex(n_tiles, K, vgrid, bid, pl);
    pl.map_base = map_base; pl.map_gshift = gshift; pl.map_gstride = gstride;
    if (pl.slice % 32 || pl.slice < 32) { printf("%s: bad slice %d\n", what, pl.slice); return 1; }
    for (int w = 0; w < DEC_WARPS; ++w) {
      bool seen_invalid = false;
      for (int j = 0; j < pl.main_rounds + pl.tail_rounds; ++j) {
        int tile, k0, klen;
        const bool ok = gemv_item(pl, K, j, w, tile, k0, klen);
        if (!ok) { seen_invalid = true; continue; }
        if (seen_invalid || tile >= pl.n_tiles) { printf("%s: item order / range\n", what); return 1; }
        if (gemv_units_of(pl, K, j) != (klen + GV_UK - 1) / GV_UK) { printf("%s: unit count\n", what); return 1; }
        cover[gemv_global_tile(pl, tile)].push_back({k0, klen});
      }
    }
  }
  if ((int)cover.size() != n_tiles) { printf("%s: %zu tiles covered, expected %d\n", what, cover.size(), n_tiles); return 1; }
  for (auto& kv : cover) {
    std::sort(kv.second.begin(), kv.second.end());
    int pos = 0;
    for (auto& seg : kv.second) { if (seg.first != pos) { printf("%s: tile %d gap at k=%d\n", what, kv.first, pos); return 1; } pos += seg.second; }
    if (pos != K) { printf("%s: tile %d covers %d of %d\n", what, kv.first, pos, K); return 1; }
  }
  return 0;
}

int main() {
  const int shapes[][2] = {{768, 768}, {2304, 768}, {3072, 768}, {768, 3072}, {51865, 768}, {128, 128}, {384, 128}, {512, 128}, {128, 512},
                           {4096, 128}, {384, 384}, {1152, 384}, {1536, 384}, {384, 1536}, {51865, 384}, {1280, 1280}, {3840, 1280},
                           {5120, 1280}, {1280, 5120}, {51866, 1280}, {6144, 4096}, {4096, 4096}, {28672, 4096}, {4096, 14336},
                           {128256, 4096}, {512, 256}, {256, 256}, {1024, 256}, {256, 512}, {2048, 256}, {1536, 1024}, {1024, 1024},
                           {7168, 1024}, {1024, 3584}, {32064, 1024}};
  int bad = 0;
  for (auto& s : shapes)
    for (int grid : {148, 144, 132, 120, 112, 66}) {
      char what[64]; snprintf(what, sizeof what, "[%d,%d] grid %d", s[0], s[1], grid);
      bad += check((s[0] + 7) / 8, s[1], grid, 0, 30, 0, what);
    }
  // cluster-local sub-plans of the Whisper cluster kernel: q/k/v rows of a head, cq rows of a head, out-projection slice
  for (int d : {128, 384, 768, 1280})
    for (int cs : {4, 8})
      for (int h = 0; h < d / 64; ++h) {
        char what[64];
        snprintf(what, sizeof what, "qkv head %d d %d cs %d", h, d, cs);
        {  // global tiles must be exactly the head's 8 q, 8 k and 8 v tiles
          std::vector<int> want;
          for (int g = 0; g < 3; ++g) for (int i = 0; i < 8; ++i) want.push_back(g * (d / 8) + 8 * h + i);
          GemvPlan pl; gemv_make_plan_ex(24, d, cs, 0, pl); pl.map_base = 8 * h; pl.map_gshift = 3; pl.map_gstride = d / 8;
          for (int lt = 0; lt < 24; ++lt) if (gemv_global_tile(pl, lt) != want[lt]) { printf("%s: tile map\n", what); ++bad; break; }
        }
        bad += check(24, d, cs, 8 * h, 3, d / 8, what) ? 1 : 0;  // note: check() counts distinct GLOBAL tiles
        snprintf(what, sizeof what, "cq head %d d %d cs %d", h, d, cs);
        bad += check(8, d, cs, 8 * h, 3, 0, what);
        snprintf(what, sizeof what, "out slice head %d d %d cs %d", h, d, cs);
        bad += check(d / 8, 64, cs, 0, 30, 0, what);
      }
  // attention plans: splits within bounds, items cover the grid sensibly
  for (int BH : {2, 6, 12, 20, 24, 32, 48, 96, 128, 192, 320, 512})
    for (int nb : {1, 2, 5, 14, 47, 64, 256})
      for (int smax : {4, 24, 128}) {
        const int p = attn_plan(BH, nb, smax, 132), S = p & 0x7f;
        if (S < 1 || S > nb || S > smax || S > ((p & ATTN_WARP_LEVEL) ? 32 : 16)) { printf("attn_plan(%d,%d,%d) = %d\n", BH, nb, smax, p); ++bad; }
      }
  // K-chunked projections (gemv_mma_chunked): for every accepted shape each (tile, k) of every chunk is covered exactly once by
  // the one-item-per-warp plan of a [N, kc] projection, including the short last chunk
  {
    const int cases[][3] = {{4096, 14336, 4096}, {2560, 9728, 4096}, {1024, 3584, 1024}, {4096, 14336, 2048}, {256, 1536, 256}};
    for (auto& cse : cases)
      for (int grid : {132, 66}) {
        const int N = cse[0], K = cse[1], kc = cse[2];
        if (!gemv_chunk_ok(N, K, kc, grid)) continue;
        const int n_tiles = (N + 7) / 8, n_chunks = (K + kc - 1) / kc;
        std::map<int, std::vector<std::pair<int, int>>> cover;
        for (int bid = 0; bid < grid; ++bid) {
          GemvPlan pl;
          gemv_make_plan_ex(n_tiles, kc, grid, bid, pl);
          if (pl.main_rounds != 0 || pl.tail_rounds > 1) { printf("chunk [%d,%d] kc %d: more than one item per warp\n", N, K, kc); ++bad; break; }
          for (int w = 0; w < DEC_WARPS && pl.tail_rounds == 1; ++w) {
            int tile, k0, klen;
            if (!gemv_item(pl, kc, 0, w, tile, k0, klen)) continue;
            const int sl = w & ((1 << pl.ks_log) - 1);
            for (int c = 0; c < n_chunks; ++c) {
              const int kcc = std::min(kc, K - c * kc), slice = kcc >> pl.ks_log;
              if (slice % 32) { printf("chunk [%d,%d] kc %d: slice %d\n", N, K, kc, slice); ++bad; }
              cover[tile].push_back({c * kc + sl * slice, slice});
            }
          }
        }
        if ((int)cover.size() != n_tiles) { printf("chunk [%d,%d] kc %d grid %d: %zu of %d tiles\n", N, K, kc, grid, cover.size(), n_tiles); ++bad; }
        for (auto& kv : cover) {
          std::sort(kv.second.begin(), kv.second.end());
          int pos = 0;
          for (auto& seg : kv.second) { if (seg.first != pos) { printf("chunk tile %d gap at %d\n", kv.first, pos); ++bad; break; } pos += seg.second; }
          if (pos != K) { printf("chunk tile %d covers %d of %d\n", kv.first, pos, K); ++bad; }
        }
      }
    for (int grid : {132, 66})  // a whole H100, and one of two SM partitions
      if (!gemv_chunk_ok(4096, 14336, 4096, grid)) { printf("Llama-3-8B down-projection must be chunkable on %d CTAs\n", grid); ++bad; }
  }
  printf(bad ? "FAILED %d\n" : "OK\n", bad);
  return bad ? 1 : 0;
}
