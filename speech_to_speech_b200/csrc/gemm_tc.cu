// gemm_tc.cu -- C = A * W^T on Hopper tensor cores (wgmma).
//
//   * operands: 16-bit (fp16 / bf16), K-major, staged global->shared by TMA (cp.async.bulk.tensor,
//     128-byte swizzle) through a STAGES-deep mbarrier ring;
//   * math: wgmma.mma_async m64 x N=BN x k16 from shared-memory descriptors, fp32 accumulators in registers;
//     each of the two consumer warpgroups owns 64 rows of the 128-row tile and keeps one k-block of MMAs in flight;
//   * epilogue: straight from the accumulator registers, fused bias, exact GELU, SwiGLU, fp32 residual add
//     (in-place residual stream or broadcast positional table) and the 16-bit / fp32 stores.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = MMA + epilogue.
//
// The weight operand W comes in one of three layouts (GemmProblem::w_layout, a template parameter of the kernel):
//   * row-major [N, ldw], 128-byte swizzle, as above (Whisper, the codec, s2s_gemm_ex);
//   * the fragment-major 16-bit tiles the decode kernels stream (weight_tiles.cu).  Each 32-k window of an 8-row tile is
//     a contiguous 8 x 64 B block, so a 4-D TMA map {32 k, 8 rows, windows, tiles} with the 64-byte swizzle lands the
//     k-block as [tile][window][8 rows][64 B] swizzle-64B atoms, which wgmma reads as a K-major operand (one 8-row group
//     = BK/32 atoms = 1024 B).  The wgmma sequence and its k order are those of the row-major path, so the result is
//     bit for bit the same;
//   * FP8 E4M3 codes in the same tiling + one power-of-two scale per row (bf16 only).  TMA loads the codes; warps 1-3 of
//     the producer warpgroup expand them times the row scale into the bf16 swizzle-64B buffer of the 16-bit tiled path
//     (exact: dq(Q) is a bf16 number) and then release the stage to the MMA warpgroups.  That warpgroup is otherwise
//     idle, so the MMA issue and the epilogue are those of the 16-bit paths.
// The Llama-family prefill reads its projections and lm_head in the tiled layouts, the one copy the decode kernel streams.
//
// Used for every GEMM-shaped op with M >= 64 on the hot path: Whisper conv1/conv2 (as strided-window
// GEMMs, no im2col), QKV / out-proj / fc1 / fc2 of the encoder, the cross-attention K/V projection and
// the LLM prefill projections.  (Reference ops: transformers modeling_whisper.py:284-357,380-414,619-625;
// modeling_llama.py:171-289.)
#include <cuda_fp8.h>

#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 16-bit = 128 B = one swizzle atom
constexpr int NTHREADS = 384;
constexpr int CONSUMERS = 256;  // threads of the two MMA warpgroups

constexpr int CONVERTERS = 96;  // FP8 weights: warps 1-3 of the producer warpgroup expand the codes

template <int BN, int WL> struct TileCfg {
  static constexpr bool F8 = WL == GEMM_W_TILED_FP8;
  static constexpr int STAGES = (BN == 64) ? 8 : (F8 ? 5 : 6);
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;     // the 16-bit weight tile wgmma reads
  static constexpr int Q_BYTES = F8 ? BN * BK : 0;  // FP8: the codes as loaded, expanded into the B buffer
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES + Q_BYTES;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + (F8 ? BN * 4 : 0) /*row scales*/;
};

struct EpiParams {
  const float* bias;
  int act;
  void* out_h;
  long long ldo_h;
  float* out_f;
  long long ldo_f;
  const float* resid;
  long long ld_resid;
  int resid_mode;
  long long out_batch_rows;
  long long out_row_offset;
  int head_major_rows;  // > 0: out_h is [row / hmr][N / 64][hmr][64] (64-column blocks contiguous per row range)
  int M, N, K;
};

// two adjacent output columns (n, n + 1) of row m
template <typename T>
__device__ __forceinline__ void epilogue_pair(const EpiParams& ep, int batch, int m, int n, float v0, float v1) {
  if (m >= ep.M) return;
  const long long orow = (long long)batch * ep.out_batch_rows + ep.out_row_offset + m;
  if (ep.bias) {
    const float2 b2 = *reinterpret_cast<const float2*>(ep.bias + n);
    v0 += b2.x; v1 += b2.y;
  }
  if (ep.act == 1) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
  if (ep.act == 2) {
    // SwiGLU over interleaved (gate, up) columns: out[n/2] = silu(v[n]) * v[n+1]; 16-bit output, ld = N/2
    reinterpret_cast<T*>(ep.out_h)[orow * ep.ldo_h + (n >> 1)] = DT<T>::from_f((v0 / (1.0f + __expf(-v0))) * v1);
    return;
  }
  if (ep.out_f) {
    if (ep.resid) {
      const long long rrow = (ep.resid_mode == 2) ? (long long)m : orow;
      const float2 q = *reinterpret_cast<const float2*>(ep.resid + rrow * ep.ld_resid + n);
      v0 += q.x; v1 += q.y;
    }
    *reinterpret_cast<float2*>(ep.out_f + orow * ep.ldo_f + n) = make_float2(v0, v1);
  }
  if (ep.out_h) {
    T* dst = reinterpret_cast<T*>(ep.out_h) + orow * ep.ldo_h + n;
    if (ep.head_major_rows > 0) {
      const long long ob = orow / ep.head_major_rows, ot = orow - ob * ep.head_major_rows;
      dst = reinterpret_cast<T*>(ep.out_h) + ((ob * (ep.N >> 6) + (n >> 6)) * ep.head_major_rows + ot) * 64 + (n & 63);
    }
    *reinterpret_cast<uint32_t*>(dst) = DT<T>::pack2(v0, v1);
  }
}

// FP8 weights: expand one stage's E4M3 codes (layout [tile][window][8 rows][32 B], as loaded) into the bf16 B buffer in
// the swizzle-64B layout TMA gives the 16-bit tiled operand, times the row scales: dq(Q) = Q * 2^e_n is a bf16 number,
// so the values wgmma multiplies by are exactly those of the 16-bit engine bound to dq(Q).
template <int BN>
__device__ __forceinline__ void expand_fp8_stage(const uint8_t* sq, uint8_t* sb, const float* s_scale, int ct) {
#pragma unroll 2
  for (int c = ct; c < BN * BK / 16; c += CONVERTERS) {  // 16 codes = half of one 32-k row of a window
    const uint4 q = *reinterpret_cast<const uint4*>(sq + c * 16);
    const int r = c >> 1, h = c & 1;                      // r = (tile * BK/32 + window) * 8 + row: one 64-B line of sb
    const float sc = s_scale[(r >> 4) * 8 + (r & 7)];
    const uint32_t qs[4] = {q.x, q.y, q.z, q.w};
    uint32_t o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(qs[i >> 1] >> (16 * (i & 1))), __NV_E4M3);
      o[i] = DT<__nv_bfloat16>::pack2(__half2float(__half(__half_raw{hr.x})) * sc, __half2float(__half(__half_raw{hr.y})) * sc);
    }
    const int sw = (r >> 1) & 3;                          // swizzle-64B: 16-B chunk ^= address bits [7, 9)
    *reinterpret_cast<uint4*>(sb + r * 64 + ((2 * h) ^ sw) * 16) = make_uint4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<uint4*>(sb + r * 64 + ((2 * h + 1) ^ sw) * 16) = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

template <typename T, int BN, int WL>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
               const float* __restrict__ w_scale, const EpiParams ep) {
  using Cfg = TileCfg<BN, WL>;
  constexpr bool F8 = Cfg::F8;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128-byte swizzle pattern (TMA and wgmma must agree)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  uint64_t* load_bar = empty_bar + Cfg::STAGES;   // FP8: the TMA loads of a stage; full_bar then means "codes expanded"
  float* s_scale = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + 256);

  const int wg = threadIdx.x >> 7;
  const int n_tile = blockIdx.x, m_tile = blockIdx.y, batch = blockIdx.z;
  const int num_kb = (ep.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_w);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], F8 ? CONVERTERS : 1);
      mbar_init(&empty_bar[s], CONSUMERS);
      if (F8) mbar_init(&load_bar[s], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % Cfg::STAGES;
        const uint32_t ph = (kb / Cfg::STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
        uint8_t* sb = sa + Cfg::A_BYTES;
        uint64_t* bar = F8 ? &load_bar[s] : &full_bar[s];
        mbar_expect_tx(bar, Cfg::A_BYTES + (F8 ? Cfg::Q_BYTES : Cfg::B_BYTES));
        tma_load_3d(sa, &map_a, bar, kb * BK, m_tile * BM, batch);
        if (WL == GEMM_W_ROW_MAJOR) tma_load_2d(sb, &map_w, bar, kb * BK, n_tile * BN);
        else tma_load_4d(F8 ? sb + Cfg::B_BYTES : sb, &map_w, bar, 0, 0, kb * (BK / 32), n_tile * (BN / 8));
      }
    } else if (F8 && threadIdx.x >= 32) {
      // The producer warpgroup is otherwise idle, so the expansion costs the MMA warpgroups nothing.
      const int ct = threadIdx.x - 32;
      for (int i = ct; i < BN; i += CONVERTERS) s_scale[i] = w_scale[n_tile * BN + i];
      asm volatile("bar.sync 1, %0;" ::"n"(CONVERTERS) : "memory");
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % Cfg::STAGES;
        mbar_wait(&load_bar[s], (kb / Cfg::STAGES) & 1);
        uint8_t* sb = smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES;
        expand_fp8_stage<BN>(sb + Cfg::B_BYTES, sb, s_scale, ct);
        fence_proxy_async();   // generic-proxy stores -> wgmma's async-proxy reads
        mbar_arrive(&full_bar[s]);
      }
    }
    return;
  }

  // ===================== MMA warpgroups: rows [64 cw, 64 cw + 64) of the tile =====================
  const int cw = wg - 1;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % Cfg::STAGES;
    if (F8) mbar_wait(&load_bar[s], (kb / Cfg::STAGES) & 1);   // the A tile
    mbar_wait(&full_bar[s], (kb / Cfg::STAGES) & 1);
    const uint32_t sa = smem_u32(smem + s * Cfg::STAGE_BYTES) + cw * (64 * 128);
    const uint32_t sb = smem_u32(smem + s * Cfg::STAGE_BYTES + Cfg::A_BYTES);
    const uint64_t adesc = wgmma_desc_sw128(sa);
    wgmma_fence_operand(acc);
    wgmma_fence();
    if (WL == GEMM_W_ROW_MAJOR) {
      const uint64_t bdesc = wgmma_desc_sw128(sb);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) wgmma_ss<T, BN>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
    } else {
      // tiled: [tile][window][8 rows][64 B] swizzle-64B atoms; one tile (8 rows) = BK/32 windows = 1024 B; k16 step k
      // reads window k/2 at byte (k%2) * 32
      const uint64_t bdesc = wgmma_desc_sw64(sb, (BK / 32) * 512);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        wgmma_ss<T, BN>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)((k >> 1) * 32 + (k & 1) * 2), 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage may be refilled
    wgmma_fence_operand(acc);
    if (kb > 0) mbar_arrive(&empty_bar[(kb - 1) % Cfg::STAGES]);
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);

  // ===================== epilogue: registers -> global =====================
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  const int m0 = m_tile * BM + cw * 64 + w * 16 + (l >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n_tile * BN + j * 8 + 2 * (l & 3);
    epilogue_pair<T>(ep, batch, m0, n, acc[4 * j], acc[4 * j + 1]);
    epilogue_pair<T>(ep, batch, m0 + 8, n, acc[4 * j + 2], acc[4 * j + 3]);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

int tma_encode_map(s2s_ctx* ctx, CUtensorMap* map, CUtensorMapDataType dt, int rank, const void* base,
                   const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  EncodeTiledFn fn = reinterpret_cast<EncodeTiledFn>(ctx->encode_tiled);
  if (!fn) {
    s2s_set_error("cuTensorMapEncodeTiled unavailable");
    return S2S_ERR_CUDA;
  }
  CUresult r = fn(map, dt, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    s2s_set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu] strides [%llu,%llu]", (int)r,
                  rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                  (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)strides_bytes[0],
                  (unsigned long long)(rank > 2 ? strides_bytes[1] : 0));
    return S2S_ERR_CUDA;
  }
  return S2S_OK;
}

namespace {

template <typename T, int BN, int WL>
int launch_impl(s2s_ctx* ctx, const GemmProblem& p, cudaStream_t stream) {
  using Cfg = TileCfg<BN, WL>;
  CUtensorMap map_a, map_w;
  {
    cuuint64_t dims[3] = {(cuuint64_t)p.K, (cuuint64_t)p.M, (cuuint64_t)p.batch};
    cuuint64_t strides[2] = {(cuuint64_t)p.a_row_stride * 2, (cuuint64_t)p.a_batch_stride * 2};
    if (p.batch == 1) strides[1] = (cuuint64_t)p.a_row_stride * 2 * (cuuint64_t)p.M;  // unused but must be valid
    cuuint32_t box[3] = {BK, BM, 1};
    S2S_CHECK(tma_encode_map(ctx, &map_a, DT<T>::tma, 3, p.a, dims, strides, box));
  }
  const float* w_scale = nullptr;
  if (WL == GEMM_W_ROW_MAJOR) {
    cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.N};
    cuuint64_t strides[1] = {(cuuint64_t)p.ldw * 2};
    cuuint32_t box[2] = {BK, BN};
    S2S_CHECK(tma_encode_map(ctx, &map_w, DT<T>::tma, 2, p.w, dims, strides, box));
  } else {
    // the tiled layout as (k in window, row in tile, window, tile): each 32-k window of an 8-row tile is an 8 x 32 block
    const cuuint64_t esz = Cfg::F8 ? 1 : 2;
    cuuint64_t dims[4] = {32, 8, (cuuint64_t)p.K / 32, (cuuint64_t)p.N / 8};
    cuuint64_t strides[3] = {32 * esz, 256 * esz, (cuuint64_t)p.K / 32 * 256 * esz};
    cuuint32_t box[4] = {32, 8, BK / 32, BN / 8};
    S2S_CHECK(tma_encode_map(ctx, &map_w, Cfg::F8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : DT<T>::tma, 4, p.w, dims, strides, box,
                             Cfg::F8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_64B));
    if (Cfg::F8) w_scale = reinterpret_cast<const float*>(reinterpret_cast<const char*>(p.w) + tiled_weight_elems(p.N, p.K));
  }
  EpiParams ep;
  ep.bias = p.bias; ep.act = p.act; ep.out_h = p.out_h; ep.ldo_h = p.ldo_h; ep.out_f = p.out_f; ep.ldo_f = p.ldo_f;
  ep.resid = p.resid; ep.ld_resid = p.ld_resid; ep.resid_mode = p.resid_mode;
  ep.out_batch_rows = p.out_batch_rows; ep.out_row_offset = p.out_row_offset; ep.head_major_rows = p.head_major_rows;
  ep.M = p.M; ep.N = p.N; ep.K = p.K;

  static bool attr_set = false;  // per (T,BN,WL) instantiation
  if (!attr_set) {
    S2S_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<T, BN, WL>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    attr_set = true;
  }
  dim3 grid(p.N / BN, (p.M + BM - 1) / BM, p.batch);
  gemm_tc_kernel<T, BN, WL><<<grid, NTHREADS, Cfg::SMEM, stream>>>(map_a, map_w, w_scale, ep);
  S2S_LAUNCH_CHECK();
  return S2S_OK;
}

template <typename T, int BN>
int launch_layout(s2s_ctx* ctx, const GemmProblem& p, cudaStream_t stream) {
  if (p.w_layout == GEMM_W_TILED16) return launch_impl<T, BN, GEMM_W_TILED16>(ctx, p, stream);
  return launch_impl<T, BN, GEMM_W_ROW_MAJOR>(ctx, p, stream);
}

}  // namespace

int gemm_tc_launch(s2s_ctx* ctx, const GemmProblem& p, int dtype, cudaStream_t stream) {
  S2S_REQUIRE(p.N % 64 == 0, "gemm: N=%d must be a multiple of 64", p.N);
  S2S_REQUIRE(p.K % 8 == 0 && p.K > 0, "gemm: K=%d must be a positive multiple of 8", p.K);
  S2S_REQUIRE(p.a_row_stride % 8 == 0, "gemm: row strides must be multiples of 8 elements");
  S2S_REQUIRE(p.w_layout >= GEMM_W_ROW_MAJOR && p.w_layout <= GEMM_W_TILED_FP8, "gemm: unknown weight layout %d", p.w_layout);
  if (p.w_layout == GEMM_W_ROW_MAJOR) S2S_REQUIRE(p.ldw % 8 == 0, "gemm: row strides must be multiples of 8 elements");
  else S2S_REQUIRE(p.K % 32 == 0, "gemm: K=%d must be a multiple of 32 with a tiled weight operand", p.K);
  S2S_REQUIRE(p.w_layout != GEMM_W_TILED_FP8 || dtype == S2S_BF16, "gemm: FP8 weights need bf16 activations");
  S2S_REQUIRE((reinterpret_cast<uintptr_t>(p.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.w) & 15) == 0,
              "gemm: operands must be 16-byte aligned");
  S2S_REQUIRE(p.M > 0 && p.batch > 0, "gemm: empty problem");
  // epilogue combinations epilogue_pair would silently ignore
  S2S_REQUIRE(p.out_h || p.out_f, "gemm: no output");
  S2S_REQUIRE(p.act >= 0 && p.act <= 2, "gemm: unknown act %d", p.act);
  S2S_REQUIRE(p.act != 2 || (p.out_h && !p.out_f && p.head_major_rows == 0),
              "gemm: SwiGLU (act 2) writes a plain 16-bit out_h only");
  S2S_REQUIRE(!p.resid || p.out_f, "gemm: a residual needs the fp32 output");
  S2S_REQUIRE(!p.resid || p.resid_mode == 1 || p.resid_mode == 2, "gemm: resid_mode %d (1 or 2 with a residual)", p.resid_mode);
  S2S_REQUIRE(p.head_major_rows >= 0 && (p.head_major_rows == 0 || p.out_h), "gemm: head_major_rows needs out_h");
  S2S_REQUIRE(p.bn == 0 || p.bn == 64 || (p.bn == 128 && p.N % 128 == 0), "gemm: bn=%d (0, 64, or 128 with N %% 128 == 0; N=%d)",
              p.bn, p.N);
  // Pick the N tile so the grid covers every SM when the problem allows it.
  const long long tiles128 = (long long)(p.N / 128) * ((p.M + BM - 1) / BM) * p.batch;
  const bool use128 = p.bn ? p.bn == 128 : (p.N % 128 == 0) && tiles128 >= ctx->num_sms;
  if (p.w_layout == GEMM_W_TILED_FP8) {
    return use128 ? launch_impl<__nv_bfloat16, 128, GEMM_W_TILED_FP8>(ctx, p, stream)
                  : launch_impl<__nv_bfloat16, 64, GEMM_W_TILED_FP8>(ctx, p, stream);
  }
  if (dtype == S2S_F16) {
    return use128 ? launch_layout<__half, 128>(ctx, p, stream) : launch_layout<__half, 64>(ctx, p, stream);
  } else if (dtype == S2S_BF16) {
    return use128 ? launch_layout<__nv_bfloat16, 128>(ctx, p, stream) : launch_layout<__nv_bfloat16, 64>(ctx, p, stream);
  }
  s2s_set_error("gemm: unsupported dtype %d", dtype);
  return S2S_ERR_UNSUPPORTED;
}
