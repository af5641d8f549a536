// weight_arena.cuh -- the host-side weight machinery every model object owns (internal to libs2s_b200): tracked device
// allocations, the table of state-dict names -> kernel layouts, bind_tensor (convert, lay out, upload), init_random and the
// finalize-time "every tensor was bound" check.  A slot may live in a tiled matrix (weight_tiles.cu): its rows are laid out
// on the host as usual, staged on the device and tiled -- or quantised to FP8 -- straight into place, so no row-major copy
// of the matrix exists.  The layout step (weight_layout / weight_upload) is pure host code, so a
// CPU program can check it against a numpy statement of each layout (tests/test_weight_layouts.py).
//
// The weights live in a WeightStore of their own, held by std::shared_ptr: an object made by s2s_*_create_shared reads
// the store of its source instead of allocating one, and the store is freed with its last holder.  Everything else an
// object allocates (KV cache, workspaces, tables sized by its capacities, its device layer tables) is its own.
#pragma once
#include <string.h>

#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

// Source shapes are those of the transformers state dict; d0, d1, d2, p and ld are read as listed.
enum WeightLayout {
  W_PLAIN = 0,
  W_ROPE_PERM,    // [d0 rows][d1]: within each head of p rows, row j < p/2 -> 2j, row j >= p/2 -> 2(j - p/2) + 1
  W_INTERLEAVE,   // [d0 rows][d1] -> rows 2r + p of a [2 d0][d1] block (p = 0 gate, 1 up)
  W_LINEAR,       // [d0 = N][d1 = K] -> [K][N]; ld > 0: columns [p, p + N) of a shared [K][ld] matrix
  W_CONV,         // [d0 = O][d1 = C][d2 = k] -> [k][C][O]
  W_TCONV,        // [d0 = C][d1 = O][d2 = k], stride p, k = p or 2p -> k/p taps x [C][p*O]; tap 0 takes W[c][o][r + k - p]
  W_CONV_ROWS,    // [d0 = O][d1 = C][d2 = k] -> [O][k][C] (Whisper's conv as a windowed GEMM: K = k*C)
};

struct WeightSlot {
  void* dst = nullptr;
  bool half = false;          // stored in the model's 16-bit compute dtype, else fp32
  int layout = W_PLAIN;
  int64_t n = 0;              // elements of the source tensor
  int d0 = 0, d1 = 0, d2 = 0, p = 0, ld = 0;
  float scale = 1.f;          // folded into every stored value, bound or random
  float rnd_scale = 0.02f, rnd_offset = 0.f;
  uint64_t seed = 0;          // != 0: init_random draws from its seed ^ this instead of its seed ^ FNV-1a(name)
  bool bound = false;
  bool raw = false;           // written by bind / init_random since the last finalize (the model clears it)
  // tN > 0: dst is a tiled [tN, tK] 16-bit (or FP8, WeightArena::tiled_format) matrix and the slot's n / tK laid-out rows are
  // its rows row0 + r * rstride.  W_INTERLEAVE slots are tiled with row0 = p, rstride = 2.
  int tN = 0, tK = 0, row0 = 0, rstride = 1;
  WeightSlot& as(int l, int a0, int a1, int a2 = 0, int pp = 0, int ldd = 0) {
    layout = l; d0 = a0; d1 = a1; d2 = a2; p = pp; ld = ldd;
    return *this;
  }
  WeightSlot& tiled(int N, int K, int first_row = 0, int row_stride = 1) {
    tN = N; tK = K; row0 = first_row; rstride = row_stride;
    return *this;
  }
};

// ---- host conversion (the one copy the models share) ----
inline uint16_t f32_to_f16_bits(float f) { __half h = __float2half_rn(f); uint16_t u; memcpy(&u, &h, 2); return u; }
inline uint16_t f32_to_bf16_bits(float f) {   // round to nearest even; every NaN -> 0x7fc0
  uint32_t u; memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fc0;
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float src_to_f32(const void* data, int64_t i, int dtype) {
  if (dtype == S2S_F32) return reinterpret_cast<const float*>(data)[i];
  uint16_t u = reinterpret_cast<const uint16_t*>(data)[i];
  if (dtype == S2S_BF16) { uint32_t w = (uint32_t)u << 16; float f; memcpy(&f, &w, 4); return f; }
  __half h; memcpy(&h, &u, 2); return __half2float(h);
}

// init_random's seed for a tensor: seed ^ FNV-1a(name).  The offset basis is not FNV's published 0xcbf29ce484222325;
// changing it would change every init_random weight.
inline uint64_t weight_seed(uint64_t seed, const std::string& name) {
  uint64_t h = 1469598103934665603ull;
  for (char ch : name) h = (h ^ (uint64_t)(unsigned char)ch) * 1099511628211ull;
  return seed ^ h;
}

// The slot's source tensor (dtype) -> the bytes bind uploads: times s.scale, laid out, stored as fp32 or as dtype16 (s.half).
// INTERLEAVE and column-block LINEAR produce the slot's own rows; weight_upload places them.
inline void weight_layout(const WeightSlot& s, const void* src, int dtype, int dtype16, std::vector<uint8_t>& out) {
  out.resize((size_t)s.n * (s.half ? 2 : 4));
  float* f32 = reinterpret_cast<float*>(out.data());
  uint16_t* h16 = reinterpret_cast<uint16_t*>(out.data());
  const bool bf = dtype16 == S2S_BF16;
  auto put = [&](int64_t di, int64_t si) {
    const float v = src_to_f32(src, si, dtype) * s.scale;
    if (!s.half) f32[di] = v;
    else h16[di] = bf ? f32_to_bf16_bits(v) : f32_to_f16_bits(v);
  };
  const int64_t A = s.d0, B = s.d1, K = s.d2;
  switch (s.layout) {
    case W_ROPE_PERM: {
      const int64_t hd = s.p, half = hd / 2;
      for (int64_t r = 0; r < A; ++r) {
        const int64_t j = r % hd, dr = r - j + (j < half ? 2 * j : 2 * (j - half) + 1);
        for (int64_t c = 0; c < B; ++c) put(dr * B + c, r * B + c);
      }
      break;
    }
    case W_LINEAR:
      for (int64_t nn = 0; nn < A; ++nn)
        for (int64_t k = 0; k < B; ++k) put(k * A + nn, nn * B + k);
      break;
    case W_CONV:
      for (int64_t o = 0; o < A; ++o)
        for (int64_t c = 0; c < B; ++c)
          for (int64_t j = 0; j < K; ++j) put((j * B + c) * A + o, (o * B + c) * K + j);
      break;
    case W_TCONV: {
      // k = 2 s: tap 0 multiplies X[t0 - 1] -> W[c][o][r + s]; tap 1 multiplies X[t0] -> W[c][o][r].  k = s: one tap.
      const int64_t st = s.p, taps = K / st;
      for (int64_t c = 0; c < A; ++c)
        for (int64_t o = 0; o < B; ++o)
          for (int64_t t = 0; t < K; ++t) put(((taps - 1 - t / st) * A + c) * st * B + (t % st) * B + o, (c * B + o) * K + t);
      break;
    }
    case W_CONV_ROWS:
      for (int64_t o = 0; o < A; ++o)
        for (int64_t c = 0; c < B; ++c)
          for (int64_t t = 0; t < K; ++t) put((o * K + t) * B + c, (o * B + c) * K + t);
      break;
    default:   // W_PLAIN, W_INTERLEAVE
      for (int64_t i = 0; i < s.n; ++i) put(i, i);
  }
}

// Where weight_layout's bytes go in s.dst: `height` rows of `width` bytes, `pitch` bytes apart, from byte `offset`.
struct WeightUpload { size_t offset, pitch, width, height; };
inline WeightUpload weight_upload(const WeightSlot& s) {
  const size_t esz = s.half ? 2 : 4;
  if (s.layout == W_INTERLEAVE) return {(size_t)s.p * s.d1 * esz, 2 * (size_t)s.d1 * esz, (size_t)s.d1 * esz, (size_t)s.d0};
  if (s.layout == W_LINEAR && s.ld > 0) return {(size_t)s.p * esz, (size_t)s.ld * esz, (size_t)s.d0 * esz, (size_t)s.d1};
  return {0, (size_t)s.n * esz, (size_t)s.n * esz, 1};
}

// The weight allocations of one model object, in allocation order, shared by the objects that read them.
struct WeightStore {
  std::vector<std::pair<void*, size_t>> allocs;
  size_t bytes = 0;
  WeightStore() = default;
  WeightStore(const WeightStore&) = delete;
  WeightStore& operator=(const WeightStore&) = delete;
  ~WeightStore() {
    for (auto& a : allocs) cudaFree(a.first);
    s2s_count_device_bytes(-(long long)bytes);
  }
};

// s2s_*_create_shared: field f of the new object's configuration must equal the source's (only capacities may differ)
#define S2S_REQUIRE_SAME(cfg, src, f, who) \
  S2S_REQUIRE((cfg).f == (src).f, "%s: cfg." #f " differs from the source's (only capacities may differ)", who)

// One per model object.  Error messages start with `who`.
struct WeightArena {
  std::unordered_map<std::string, WeightSlot> slots;

  WeightArena() = default;
  WeightArena(const WeightArena&) = delete;
  WeightArena& operator=(const WeightArena&) = delete;
  ~WeightArena() {
    for (void* p : allocs_) cudaFree(p);
    s2s_count_device_bytes(-(long long)bytes_);
    release_staging();
  }

  // storage of the tiled slots: the 16-bit compute dtype (tiles) or S2S_FP8_E4M3 (codes + row scales, bf16 sources)
  int tiled_format = 0;

  // cudaMalloc (zeroed unless zero = false), freed with the arena: the object's own state
  template <typename P> int alloc(P** out, size_t bytes, bool zero = true) {
    void* p = nullptr;
    const size_t n = bytes ? bytes : 16;
    S2S_CHECK_CUDA(cudaMalloc(&p, n));
    allocs_.push_back(p);
    bytes_ += n;
    s2s_count_device_bytes((long long)n);
    if (zero) S2S_CHECK_CUDA(cudaMemset(p, 0, n));
    *out = reinterpret_cast<P*>(p);
    return S2S_OK;
  }
  // weight storage, zeroed, in the store.  An arena that borrows another object's store (borrow()) allocates nothing: the
  // k-th call returns the store's k-th allocation, which has the same size because the two objects' configurations differ
  // only in capacities, and the weights' sizes do not depend on those.
  template <typename P> int alloc_weights(P** out, size_t bytes) {
    const size_t n = bytes ? bytes : 16;
    if (borrowed_) {
      S2S_REQUIRE(next_ < store_->allocs.size() && store_->allocs[next_].second == n,
                  "shared weights: allocation %zu of %zu bytes does not match the source's store", next_, n);
      *out = reinterpret_cast<P*>(store_->allocs[next_++].first);
      return S2S_OK;
    }
    void* p = nullptr;
    S2S_CHECK_CUDA(cudaMalloc(&p, n));
    store_->allocs.push_back({p, n});
    store_->bytes += n;
    s2s_count_device_bytes((long long)n);
    S2S_CHECK_CUDA(cudaMemset(p, 0, n));
    *out = reinterpret_cast<P*>(p);
    return S2S_OK;
  }
  // read `src`'s weights from now on (before the first alloc_weights): the object shares its store and never writes it
  void borrow(const WeightArena& src) {
    store_ = src.store_;
    borrowed_ = true;
    next_ = 0;
    tiled_format = src.tiled_format;
  }
  bool borrowed() const { return borrowed_; }
  // bind_tensor / init_random / finalize (and anything else that writes weights) may run: the arena owns its store and no
  // other object reads it -- another lane may be mid-launch on shared bytes
  int check_writable(const char* who) const {
    S2S_REQUIRE(!borrowed_, "%s: the weights are shared from another object and are read-only", who);
    const long n = store_.use_count();
    S2S_REQUIRE(n == 1, "%s: %ld other objects read these weights (destroy them first)", who, n - 1);
    return S2S_OK;
  }
  size_t bytes() const { return bytes_ + store_->bytes; }   // device bytes the object reads (the staging buffer excluded)
  size_t weight_bytes() const { return store_->bytes; }     // ... of them in the (possibly shared) weight store
  // the device buffer bind / init_random stage a tiled slot's rows in (as large as the largest such slot); models free it
  // at finalize
  void release_staging() {
    if (staging_) {
      cudaFree(staging_);
      s2s_count_device_bytes(-(long long)staging_bytes_);
    }
    staging_ = nullptr;
    staging_bytes_ = 0;
  }
  WeightSlot& add(const std::string& name, void* dst, bool half, int64_t n, float rnd_scale = 0.02f, float rnd_offset = 0.f) {
    WeightSlot& s = slots[name];
    s = WeightSlot();
    s.dst = dst; s.half = half; s.n = n; s.rnd_scale = rnd_scale; s.rnd_offset = rnd_offset;
    return s;
  }
  WeightSlot* find(const std::string& name) {
    auto it = slots.find(name);
    return it == slots.end() ? nullptr : &it->second;
  }
  // lookup (S2S_ERR_NOT_FOUND), element count (S2S_ERR_INVALID), then weight_layout and one upload
  int bind(const char* who, const char* name, const void* data_h, const int64_t* shape, int ndim, int dtype, int dtype16);
  // every slot from fill_random_launch (seed ^ FNV-1a(name), or the slot's own seed), synchronised
  int init_random(uint64_t seed, int dtype16);
  int check_all_bound(const char* who) const;

 private:
  std::vector<void*> allocs_;
  size_t bytes_ = 0;
  std::shared_ptr<WeightStore> store_ = std::make_shared<WeightStore>();
  bool borrowed_ = false;
  size_t next_ = 0;
  void* staging_ = nullptr;
  size_t staging_bytes_ = 0;
  int ensure_staging();
  int stage_tiled(const WeightSlot& s, const void* bytes, int64_t rows, int row0, int rstride);
};
