// sampling.cuh -- token choice of one fp32 logits row by ONE CTA (any block size that is a multiple of 32, <= 1024).
// Semantics pinned to transformers' _get_logits_processor order (oracle/sampling_ref.py restates it in numpy):
//   1. repetition penalty over the slot's seen ids: z < 0 ? z * p : z / p          (RepetitionPenaltyLogitsProcessor)
//   2. the slot's EOS ids -> -inf until min_new tokens were produced              (MinNewTokensLengthLogitsProcessor)
//   greedy: argmax (ties -> lowest id).  do_sample:
//   3. z / temperature, top-k (ties with the k-th value kept; 0 or >= vocab = off), top-p (ascending sort, inclusive
//      cumulative softmax, remove cum <= 1 - top_p, keep >= 1)
//   4. Gumbel-max over the survivors: argmax_i(z_i - log(-log u_i)), ties -> lowest id, u_i from Philox4x64-10 keyed by the
//      slot's seed with counter (token id + 1, predicted position, stream, 0) -- the first block
//      numpy.random.Philox(key=seed, counter=[id, position, stream, 0]) produces -- so a token depends only on (seed,
//      position, stream, logits).  The LLM and the Qwen3-TTS talker draw from stream 0; the Qwen3-TTS code predictor,
//      whose positions repeat every frame, from stream 1 + the frame's index since the utterance's prefill.
// Top-k and top-p are exact radix selects over the order-preserving bits of the processed value (8 bits per level, 256-bin
// shared histograms; top-p's histogram sums probability mass in 2^-40 fixed point, so the sums are deterministic), so
// the vocabulary is never sorted.  Every pass recomputes the processed value from the row (L2-resident) instead of storing it.
#pragma once
#include <math.h>
#include <stdint.h>

struct SampSlot {               // per-session parameters of a launch (host-packed from the slot's table)
  int active;                   // 0: nothing below applies (the caller's plain argmax path)
  int do_sample, top_k, min_new, n_eos;
  int base;                     // position of the first token predicted after the slot's last prefill
  float temperature, top_p, penalty;
  int eos[8];
  unsigned long long seed;
  unsigned long long stream;    // Philox counter word 2
};
// the parameters of a greedy session
inline SampSlot samp_greedy() {
  SampSlot s{};
  s.temperature = 1.f; s.top_p = 1.f; s.penalty = 1.f;
  return s;
}

struct SampShared {             // shared scratch of sample_row
  unsigned long long hist[256];
  double rv[32];
  int ri[32];
  unsigned long long above, sum;
  unsigned int key;
  int tok;
};

__host__ __device__ __forceinline__ unsigned long long samp_philox(unsigned long long seed, unsigned long long c0,
                                                                   unsigned long long c1, unsigned long long c2) {
  unsigned long long x0 = c0, x1 = c1, x2 = c2, x3 = 0, k0 = seed, k1 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
    const unsigned long long m0 = 0xD2E7470EE14C6C93ull, m1 = 0xCA5A826395121157ull;
#ifdef __CUDA_ARCH__
    const unsigned long long hi0 = __umul64hi(m0, x0), hi1 = __umul64hi(m1, x2);
#else
    const unsigned long long hi0 = (unsigned long long)(((unsigned __int128)m0 * x0) >> 64),
                             hi1 = (unsigned long long)(((unsigned __int128)m1 * x2) >> 64);
#endif
    const unsigned long long lo0 = m0 * x0, lo1 = m1 * x2;
    x0 = hi1 ^ x1 ^ k0; x1 = lo1; x2 = hi0 ^ x3 ^ k1; x3 = lo0;
  }
  return x0;
}

// larger float -> larger key
__device__ __forceinline__ unsigned int samp_key(float z) {
  const unsigned int u = __float_as_uint(z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float samp_apply(float z, bool is_seen, const SampSlot& s, bool mask_eos, int i) {
  if (is_seen) z = z < 0.f ? z * s.penalty : z / s.penalty;
  if (mask_eos) {
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (e < s.n_eos && i == s.eos[e]) z = -INFINITY;
  }
  if (s.do_sample) z = z / s.temperature;
  return z;
}

// f(i, processed value) for every id of the row.  Each thread keeps SAMP_UNROLL 16-byte row loads in flight (a pass is
// bound by the L2 round trip, not by bandwidth); rows are 16-byte aligned with V % 4 == 0 (vocab % 64 == 0 at create),
// anything else takes the scalar loop.
constexpr int SAMP_UNROLL = 8;
template <typename F>
__device__ __forceinline__ void samp_for_each(const float* row, const unsigned int* seen, const SampSlot& s, bool mask_eos, int V,
                                              F&& f) {
  const int nt = blockDim.x;
  if ((V & 3) || (reinterpret_cast<uintptr_t>(row) & 15)) {
#pragma unroll 1
    for (int i = threadIdx.x; i < V; i += nt)
      f(i, samp_apply(__ldcg(row + i), seen && ((__ldcg(seen + (i >> 5)) >> (i & 31)) & 1u), s, mask_eos, i));
    return;
  }
  const int V4 = V >> 2;
  const float4* r4 = reinterpret_cast<const float4*>(row);
#pragma unroll 1
  for (int q0 = threadIdx.x; q0 < V4; q0 += SAMP_UNROLL * nt) {
    float4 z[SAMP_UNROLL];
    unsigned int w[SAMP_UNROLL];
#pragma unroll
    for (int u = 0; u < SAMP_UNROLL; ++u) {
      const int q = q0 + u * nt;
      z[u] = q < V4 ? __ldcg(r4 + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      w[u] = seen && q < V4 ? __ldcg(seen + (q >> 3)) : 0u;    // the 4 ids of a vector share one bitmap word
    }
#pragma unroll
    for (int u = 0; u < SAMP_UNROLL; ++u) {
      const int q = q0 + u * nt, i = 4 * q;
      if (q < V4) {
        const unsigned int b = w[u] >> (i & 31);
        f(i, samp_apply(z[u].x, b & 1u, s, mask_eos, i));
        f(i + 1, samp_apply(z[u].y, (b >> 1) & 1u, s, mask_eos, i + 1));
        f(i + 2, samp_apply(z[u].z, (b >> 2) & 1u, s, mask_eos, i + 2));
        f(i + 3, samp_apply(z[u].w, (b >> 3) & 1u, s, mask_eos, i + 3));
      }
    }
  }
}

// block argmax of (v, i), ties -> lowest i; the winner lands in sh.tok / sh.rv[0] (all threads return the id)
__device__ __forceinline__ int samp_block_argmax(double bv, int bi, SampShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { sh.rv[warp] = bv; sh.ri[warp] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (sh.rv[w] > bv || (sh.rv[w] == bv && sh.ri[w] < bi)) { bv = sh.rv[w]; bi = sh.ri[w]; }
    sh.rv[0] = bv; sh.tok = bi;
  }
  __syncthreads();
  return sh.tok;
}

// warp 0: walk sh.hist from bin 255 down, starting with sh.above, to the first bin where the running sum reaches `target`;
// append that bin to sh.key at `shift` and add the bins above it to sh.above
__device__ __forceinline__ void samp_pick_bin(SampShared& sh, double target, int shift) {
  const int lane = threadIdx.x & 31;
  unsigned long long c = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) c += sh.hist[255 - 8 * lane - j];
  unsigned long long inc = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  const unsigned int hit = __ballot_sync(0xffffffffu, (double)(sh.above + inc) >= target);
  const int first = hit ? __ffs(hit) - 1 : 31;
  if (lane == first) {
    unsigned long long run = sh.above + inc - c;
    int bin = 255 - 8 * lane - 7;
    for (int j = 0; j < 8; ++j) {
      const unsigned long long h = sh.hist[255 - 8 * lane - j];
      if ((double)(run + h) >= target) { bin = 255 - 8 * lane - j; break; }
      run += h;
    }
    sh.key |= (unsigned int)bin << shift;
    sh.above = run;
  }
}

// The token of one logits row (see the top of the file).  pred_pos: position of the predicted token; seen: the slot's
// bitmap (only read when penalty != 1).  Every thread of the block calls it and gets the id.
static __device__ __noinline__ int sample_row(const float* row, int V, const SampSlot s, const unsigned int* seen, int pred_pos,
                                       SampShared& sh) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const unsigned int* sn = s.penalty != 1.f ? seen : nullptr;
  const bool mask_eos = pred_pos - s.base < s.min_new;
  double bv = -INFINITY; int bi = 0x7fffffff;
  samp_for_each(row, sn, s, mask_eos, V, [&](int i, float zf) {
    const double z = zf;
    if (z > bv || (z == bv && i < bi)) { bv = z; bi = i; }
  });
  const int top = samp_block_argmax(bv, bi, sh);
  if (!s.do_sample) return top;
  const float zmax = (float)sh.rv[0];
  __syncthreads();

  // radix select of the threshold key: top-k on counts, then top-p on mass among the top-k survivors
  unsigned int thr = 0;
  const bool use_k = s.top_k > 0 && s.top_k < V, use_p = s.top_p < 1.f;
  for (int stage = 0; stage < 2; ++stage) {
    if (stage == 0 ? !use_k : !use_p) continue;
    double target;
    if (stage == 0) {
      target = (double)s.top_k;
    } else {
      unsigned long long part = 0;
      samp_for_each(row, sn, s, mask_eos, V, [&](int, float z) {
        if (samp_key(z) >= thr) part += __double2ull_rn((double)expf(z - zmax) * 1099511627776.0);
      });
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      if (tid == 0) sh.sum = 0;
      __syncthreads();
      if ((tid & 31) == 0) atomicAdd(&sh.sum, part);
      __syncthreads();
      target = (double)s.top_p * (double)sh.sum;
    }
    if (tid == 0) { sh.key = 0; sh.above = 0; }
    unsigned int prefix = 0, mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += nt) sh.hist[i] = 0;
      __syncthreads();
      samp_for_each(row, sn, s, mask_eos, V, [&](int, float z) {
        const unsigned int k = samp_key(z);
        if ((k & mask) == prefix && k >= thr)
          atomicAdd(&sh.hist[(k >> shift) & 255u], stage == 0 ? 1ull : __double2ull_rn((double)expf(z - zmax) * 1099511627776.0));
      });
      __syncthreads();
      if (tid < 32) samp_pick_bin(sh, target, shift);
      __syncthreads();
      prefix = sh.key;
      mask |= 255u << shift;
    }
    thr = prefix;
    __syncthreads();
  }

  // Gumbel-max draw over the survivors
  bv = -INFINITY; bi = 0x7fffffff;
  samp_for_each(row, sn, s, mask_eos, V, [&](int i, float z) {
    if (samp_key(z) < thr) return;
    const unsigned long long r = samp_philox(s.seed, (unsigned long long)i + 1ull, (unsigned long long)pred_pos, s.stream);
    const double u = (double)(r >> 11) * (1.0 / 9007199254740992.0);
    const double g = (double)z - log(-log(u));
    if (g > bv || (g == bv && i < bi)) { bv = g; bi = i; }
  });
  return samp_block_argmax(bv, bi, sh);
}
