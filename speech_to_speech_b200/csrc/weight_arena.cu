// weight_arena.cu -- WeightArena's device-side steps: upload of a bound tensor, init_random, the finalize-time check.
#include <algorithm>

#include "kernels.cuh"
#include "weight_arena.cuh"

namespace {

int upload(const WeightSlot& s, const void* bytes) {
  const WeightUpload u = weight_upload(s);
  char* dst = reinterpret_cast<char*>(s.dst) + u.offset;
  if (u.height == 1) S2S_CHECK_CUDA(cudaMemcpy(dst, bytes, u.width, cudaMemcpyHostToDevice));
  else S2S_CHECK_CUDA(cudaMemcpy2D(dst, u.pitch, bytes, u.width, u.width, u.height, cudaMemcpyHostToDevice));
  return S2S_OK;
}

}  // namespace

int WeightArena::ensure_staging() {
  if (staging_) return S2S_OK;
  size_t most = 0;
  for (const auto& kv : slots) {
    const WeightSlot& t = kv.second;
    if (t.tN > 0) most = std::max(most, (size_t)t.n * (t.layout == W_INTERLEAVE ? 2 : 1) * 2);
  }
  S2S_CHECK_CUDA(cudaMalloc(&staging_, most ? most : 16));
  staging_bytes_ = most ? most : 16;
  s2s_count_device_bytes((long long)staging_bytes_);
  return S2S_OK;
}

// rows [0, rows) of the slot's tiled matrix source (`bytes`: host, or nullptr = already in the staging buffer) -> rows
// row0 + r * rstride of s.dst
int WeightArena::stage_tiled(const WeightSlot& s, const void* bytes, int64_t rows, int row0, int rstride) {
  S2S_CHECK(ensure_staging());
  if (bytes) S2S_CHECK_CUDA(cudaMemcpy(staging_, bytes, (size_t)rows * s.tK * 2, cudaMemcpyHostToDevice));
  return tile_rows_launch(staging_, (int)rows, s.tK, s.dst, s.tN, row0, rstride, tiled_format == S2S_FP8_E4M3, 0);
}

int WeightArena::bind(const char* who, const char* name, const void* data_h, const int64_t* shape, int ndim, int dtype,
                      int dtype16) {
  WeightSlot* s = find(name);
  if (!s) {
    s2s_set_error("%s bind_tensor: unknown tensor '%s'", who, name);
    return S2S_ERR_NOT_FOUND;
  }
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  S2S_REQUIRE(n == s->n, "%s bind_tensor: '%s' has %lld elements, expected %lld", who, name, (long long)n, (long long)s->n);
  std::vector<uint8_t> bytes;
  weight_layout(*s, data_h, dtype, dtype16, bytes);
  if (s->tN > 0) S2S_CHECK(stage_tiled(*s, bytes.data(), s->n / s->tK, s->row0, s->rstride));
  else S2S_CHECK(upload(*s, bytes.data()));
  s->bound = s->raw = true;
  return S2S_OK;
}

int WeightArena::init_random(uint64_t seed, int dtype16) {
  for (auto& kv : slots) {
    WeightSlot& s = kv.second;
    const uint64_t sd = s.seed ? seed ^ s.seed : weight_seed(seed, kv.first);
    const float rs = s.rnd_scale * s.scale;
    s.bound = s.raw = true;
    if (s.tN > 0) {
      // drawn row-major into the staging buffer, exactly as into a row-major matrix, then tiled
      if (s.layout == W_INTERLEAVE && s.p == 1) continue;   // the gate slot fills the whole interleaved [2 d0][d1] block
      const bool pair = s.layout == W_INTERLEAVE;
      S2S_CHECK(ensure_staging());
      S2S_CHECK(fill_random_launch(staging_, pair ? 2 * s.n : s.n, dtype16, rs, s.rnd_offset, sd, 0));
      S2S_CHECK(stage_tiled(s, nullptr, (pair ? 2 * s.n : s.n) / s.tK, pair ? 0 : s.row0, pair ? 1 : s.rstride));
    } else if (s.layout == W_INTERLEAVE) {
      if (s.p == 1) continue;   // the gate slot fills the whole interleaved [2 d0][d1] block
      S2S_CHECK(fill_random_launch(s.dst, 2 * s.n, dtype16, rs, s.rnd_offset, sd, 0));
    } else if (s.layout == W_LINEAR && s.ld > 0) {
      // column block of a shared fp32 matrix: drawn on the host (64-bit LCG), uploaded like a bound tensor
      std::vector<float> tmp((size_t)s.n);
      uint64_t st = sd;
      for (auto& v : tmp) { st = st * 6364136223846793005ull + 1442695040888963407ull; v = rs * (((st >> 40) & 0xffff) / 32768.0f - 1.0f); }
      S2S_CHECK(upload(s, tmp.data()));
    } else {
      S2S_CHECK(fill_random_launch(s.dst, s.n, s.half ? dtype16 : S2S_F32, rs, s.rnd_offset, sd, 0));
    }
  }
  S2S_CHECK_CUDA(cudaDeviceSynchronize());
  return S2S_OK;
}

int WeightArena::check_all_bound(const char* who) const {
  for (const auto& kv : slots)
    if (!kv.second.bound) {
      s2s_set_error("%s finalize: tensor '%s' was never bound", who, kv.first.c_str());
      return S2S_ERR_INVALID;
    }
  return S2S_OK;
}
