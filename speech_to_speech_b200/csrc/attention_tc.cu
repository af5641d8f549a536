// attention_tc.cu -- fused softmax(Q K^T) V on Hopper tensor cores (wgmma + TMA).
//
// One CTA = 128 query rows of one head; two MMA warpgroups own 64 query rows each.  Per 64-key tile:
//   S = Q K^T        wgmma m64 n64 k16 x hd/16, Q and K tiles in shared memory (TMA, 128-byte swizzle), S in registers
//   softmax          in registers: a query row lives in one quad of lanes (online max/sum in fp32, exp2), the
//                    accumulators O are rescaled in place
//   O += P V         wgmma m64 n=hd k16 x 4 with P (16-bit) as the register A operand and the V^T tile
//                    [hd, 64 keys] in shared memory (TMA)
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = MMA + softmax + epilogue.
// K/V tiles are double buffered.  V is consumed as V^T (K-major B operand), produced once per call by a small
// transpose kernel into a caller-owned scratch [B, kv_heads, hd, Tpad].
// Reference ops: transformers modeling_whisper.py:215-239 (eager_attention_forward, encoder: non-causal 1500x1500),
// modeling_llama.py:187-222 (causal GQA, prefill).
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

namespace {

constexpr int QM = 128;  // queries per CTA
constexpr int KN = 64;   // keys per tile
constexpr int ATC_THREADS = 384;
constexpr int ATC_CONSUMERS = 256;

struct AtcParams {
  void* o;
  long long ldo;
  int B, Tq, Tk, heads, kv_heads;
  float scale_log2;
  int causal_off;  // query i sees keys <= i + causal_off
};

template <int HD> struct AtcSmem {
  static constexpr int Q_BYTES = QM * HD * 2;
  static constexpr int K_BYTES = KN * HD * 2;   // per stage
  static constexpr int V_BYTES = HD * KN * 2;   // per stage
  static constexpr int OFF_K = Q_BYTES;
  static constexpr int OFF_V = OFF_K + 2 * K_BYTES;
  static constexpr int OFF_BAR = OFF_V + 2 * V_BYTES;
  static constexpr int TOTAL = OFF_BAR + 256 + 1024;
};

template <typename T, int HD, bool CAUSAL>
__global__ void __launch_bounds__(ATC_THREADS, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
               const __grid_constant__ CUtensorMap map_vt, const AtcParams p) {
  using L = AtcSmem<HD>;
  constexpr int KK = HD / 64;  // 64-element (128-byte) swizzle atoms along the head dimension
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + L::OFF_K;
  uint8_t* sV = smem + L::OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2]

  const int wg = threadIdx.x >> 7;
  const int q0 = blockIdx.x * QM, h = blockIdx.y, b = blockIdx.z;
  const int kvh = h / (p.heads / p.kv_heads);

  int n_tiles = (p.Tk + KN - 1) / KN;
  if (CAUSAL) {
    const int last_key = min(p.Tk - 1, q0 + QM - 1 + p.causal_off);
    n_tiles = min(n_tiles, last_key / KN + 1);
    if (n_tiles < 1) n_tiles = 1;
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_vt);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1); mbar_init(&kv_full[1], 1);
    mbar_init(&kv_empty[0], ATC_CONSUMERS); mbar_init(&kv_empty[1], ATC_CONSUMERS);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ============================== TMA producer ==============================
    if (threadIdx.x == 0) {
      mbar_expect_tx(q_full, L::Q_BYTES);
#pragma unroll
      for (int kk = 0; kk < KK; ++kk) tma_load_2d(sQ + kk * (QM * 128), &map_q, q_full, h * HD + kk * 64, b * p.Tq + q0);
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t & 1;
        mbar_wait(&kv_empty[s], ((t >> 1) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], L::K_BYTES + L::V_BYTES);
#pragma unroll
        for (int kk = 0; kk < KK; ++kk)
          tma_load_2d(sK + s * L::K_BYTES + kk * (KN * 128), &map_k, &kv_full[s], kvh * HD + kk * 64, b * p.Tk + t * KN);
        tma_load_3d(sV + s * L::V_BYTES, &map_vt, &kv_full[s], t * KN, 0, b * p.kv_heads + kvh);
      }
    }
    return;
  }

  // ============================== MMA warpgroups: query rows [64 cw, 64 cw + 64) ==============================
  const int cw = wg - 1;
  const int tid = threadIdx.x & 127, w = tid >> 5, l = tid & 31;
  const int r0 = q0 + cw * 64 + w * 16 + (l >> 2);  // this thread's two query rows: r0 and r0 + 8
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};  // lsum: this thread's share of the row sum
  mbar_wait(q_full, 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int s = t & 1;
    mbar_wait(&kv_full[s], (t >> 1) & 1);
    // ---- S = Q K^T ----
    float sacc[KN / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KK; ++kk) {
      const uint64_t ad = wgmma_desc_sw128(smem_u32(sQ + kk * (QM * 128) + cw * (64 * 128)));
      const uint64_t bd = wgmma_desc_sw128(smem_u32(sK + s * L::K_BYTES + kk * (KN * 128)));
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<T, KN>(sacc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), (kk | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(sacc);
    // ---- online softmax ----
    const int kbase = t * KN + 2 * (l & 3);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < KN / 2; ++i) {
      const int key = kbase + (i >> 2) * 8 + (i & 1), hr = (i >> 1) & 1;
      bool ok = key < p.Tk;
      if (CAUSAL) ok = ok && (key <= r0 + hr * 8 + p.causal_off);
      sacc[i] = ok ? sacc[i] * p.scale_log2 : -INFINITY;
      mx[hr] = fmaxf(mx[hr], sacc[i]);
    }
    float corr[2], m_use[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
      const float m_new = fmaxf(m[hr], mx[hr]);
      m_use[hr] = (m_new == -INFINITY) ? 0.f : m_new;
      corr[hr] = exp2f(m[hr] - m_use[hr]);  // m = -inf -> 0
      m[hr] = m_new;
      lsum[hr] *= corr[hr];
    }
    uint32_t pk[KN / 4];  // P packed 2 x 16-bit, in the accumulator order = the A-operand order of the next product
#pragma unroll
    for (int i = 0; i < KN / 2; i += 2) {
      const int hr = (i >> 1) & 1;
      const float p0 = exp2f(sacc[i] - m_use[hr]), p1 = exp2f(sacc[i + 1] - m_use[hr]);
      lsum[hr] += p0 + p1;
      pk[i >> 1] = DT<T>::pack2(p0, p1);
    }
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] *= corr[(i >> 1) & 1];
    // ---- O += P V ----
    const uint64_t vd = wgmma_desc_sw128(smem_u32(sV + s * L::V_BYTES));
    wgmma_fence_operand(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KN / 16; ++k) {
      const uint32_t a[4] = {pk[4 * k], pk[4 * k + 1], pk[4 * k + 2], pk[4 * k + 3]};
      wgmma_rs<T, HD>(o, a, vd + (uint64_t)(k * 2), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(o);
    mbar_arrive(&kv_empty[s]);
  }
  // ---- epilogue: O / l -> 16-bit global ----
  float inv[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float lt = lsum[hr];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    inv[hr] = lt > 0.f ? 1.f / lt : 0.f;
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = r0 + hr * 8;
    if (q >= p.Tq) continue;
    T* orow = reinterpret_cast<T*>(p.o) + ((long long)b * p.Tq + q) * p.ldo + (long long)h * HD + 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + j * 8) = DT<T>::pack2(o[4 * j + 2 * hr] * inv[hr], o[4 * j + 2 * hr + 1] * inv[hr]);
  }
}

// v [B*Tk rows, ld] (offset to the V columns applied by the caller) -> vt [B, kv_heads, hd, Tpad]
template <typename T>
__global__ void __launch_bounds__(256) transpose_v_kernel(const T* __restrict__ v, long long ld, int Tk, int cols, int hd,
                                                          int Tpad, T* __restrict__ vt) {
  __shared__ T tile[64][66];
  const int t0 = blockIdx.x * 64, c0 = blockIdx.y * 64, b = blockIdx.z;
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    T val = DT<T>::from_f(0.f);
    if (t0 + r < Tk && c0 + c < cols) val = v[((long long)b * Tk + t0 + r) * ld + c0 + c];
    tile[r][c] = val;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int c = i >> 6, r = i & 63;  // r fastest: coalesced along keys
    const int col = c0 + c;
    if (col < cols && t0 + r < Tpad) {
      const int head = col / hd, dd = col % hd;
      vt[(((long long)b * (cols / hd) + head) * hd + dd) * Tpad + t0 + r] = tile[r][c];
    }
  }
}

template <typename T, int HD, bool CAUSAL>
int launch_atc(s2s_ctx* ctx, const void* q, const void* k, const void* v, void* o, int B, int Tq, int Tk, int heads,
               int kv_heads, long long ldq, long long ldk, long long ldv, long long ldo, float scale, void* vt, int Tpad,
               cudaStream_t stream) {
  using L = AtcSmem<HD>;
  {
    dim3 g((Tpad + 63) / 64, (kv_heads * HD + 63) / 64, B);
    transpose_v_kernel<T><<<g, 256, 0, stream>>>(reinterpret_cast<const T*>(v), ldv, Tk, kv_heads * HD, HD, Tpad,
                                                 reinterpret_cast<T*>(vt));
    S2S_LAUNCH_CHECK();
  }
  CUtensorMap mq, mk, mv;
  {
    cuuint64_t dims[2] = {(cuuint64_t)heads * HD, (cuuint64_t)B * Tq};
    cuuint64_t strides[1] = {(cuuint64_t)ldq * 2};
    cuuint32_t box[2] = {64, QM};
    S2S_CHECK(tma_encode_map(ctx, &mq, DT<T>::tma, 2, q, dims, strides, box));
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)kv_heads * HD, (cuuint64_t)B * Tk};
    cuuint64_t strides[1] = {(cuuint64_t)ldk * 2};
    cuuint32_t box[2] = {64, KN};
    S2S_CHECK(tma_encode_map(ctx, &mk, DT<T>::tma, 2, k, dims, strides, box));
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)Tpad, (cuuint64_t)HD, (cuuint64_t)B * kv_heads};
    cuuint64_t strides[2] = {(cuuint64_t)Tpad * 2, (cuuint64_t)HD * Tpad * 2};
    cuuint32_t box[3] = {64, HD, 1};
    S2S_CHECK(tma_encode_map(ctx, &mv, DT<T>::tma, 3, vt, dims, strides, box));
  }
  AtcParams p;
  p.o = o; p.ldo = ldo; p.B = B; p.Tq = Tq; p.Tk = Tk; p.heads = heads; p.kv_heads = kv_heads;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal_off = Tk - Tq;
  static bool attr_set = false;
  if (!attr_set) {
    S2S_CHECK_CUDA(cudaFuncSetAttribute(attn_tc_kernel<T, HD, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    attr_set = true;
  }
  dim3 grid((Tq + QM - 1) / QM, heads, B);
  attn_tc_kernel<T, HD, CAUSAL><<<grid, ATC_THREADS, L::TOTAL, stream>>>(mq, mk, mv, p);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

template <typename T>
int dispatch_atc(s2s_ctx* ctx, const void* q, const void* k, const void* v, void* o, int B, int Tq, int Tk, int heads,
                 int kv_heads, int hd, long long ldq, long long ldk, long long ldv, long long ldo, float scale, int causal,
                 void* vt, int Tpad, cudaStream_t st) {
#define ATC_GO(HD_, C_) return launch_atc<T, HD_, C_>(ctx, q, k, v, o, B, Tq, Tk, heads, kv_heads, ldq, ldk, ldv, ldo, scale, vt, Tpad, st)
  if (hd == 64) { if (causal) ATC_GO(64, true); else ATC_GO(64, false); }
  if (hd == 128) { if (causal) ATC_GO(128, true); else ATC_GO(128, false); }
#undef ATC_GO
  s2s_set_error("attention_tc: head_dim %d unsupported (64 or 128)", hd);
  return S2S_ERR_UNSUPPORTED;
}

}  // namespace

size_t attention_tc_scratch_elems(int B, int Tk, int kv_heads, int hd) {
  const int Tpad = (Tk + 63) / 64 * 64;
  return (size_t)B * kv_heads * hd * Tpad;
}

int attention_tc_launch(s2s_ctx* ctx, const void* q, const void* k, const void* v, void* o, int B, int Tq, int Tk,
                        int heads, int kv_heads, int hd, long long ldq, long long ldk, long long ldv, long long ldo,
                        float scale, int causal, int dtype, void* vt_scratch, size_t vt_elems, cudaStream_t stream) {
  S2S_REQUIRE(B > 0 && Tq > 0 && Tk > 0 && heads > 0 && kv_heads > 0 && heads % kv_heads == 0, "attention_tc: bad shape");
  S2S_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldo % 8 == 0, "attention_tc: row strides must be multiples of 8 elements");
  S2S_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(o) & 15) == 0, "attention_tc: q/k/o must be 16-byte aligned");
  const int Tpad = (Tk + 63) / 64 * 64;
  S2S_REQUIRE(vt_scratch && vt_elems >= attention_tc_scratch_elems(B, Tk, kv_heads, hd), "attention_tc: V^T scratch too small");
  if (dtype == S2S_F16)
    return dispatch_atc<__half>(ctx, q, k, v, o, B, Tq, Tk, heads, kv_heads, hd, ldq, ldk, ldv, ldo, scale, causal, vt_scratch, Tpad, stream);
  if (dtype == S2S_BF16)
    return dispatch_atc<__nv_bfloat16>(ctx, q, k, v, o, B, Tq, Tk, heads, kv_heads, hd, ldq, ldk, ldv, ldo, scale, causal, vt_scratch, Tpad, stream);
  s2s_set_error("attention_tc: unsupported dtype %d", dtype);
  return S2S_ERR_UNSUPPORTED;
}
