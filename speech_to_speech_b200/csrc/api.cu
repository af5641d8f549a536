// api.cu -- context, error reporting and the thin C-ABI wrappers around the stand-alone kernels.
#include <stdarg.h>

#include <atomic>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};   // process-wide: lanes launch from several host threads
static std::atomic<long long> g_device_bytes{0};   // process-wide: lanes create and destroy objects from several host threads

void s2s_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void s2s_count_launch(int n) { g_launches += n; }
void s2s_count_device_bytes(long long delta) { g_device_bytes += delta; }

extern "C" {

const char* s2s_last_error(void) { return g_err; }

int64_t s2s_launch_count(s2s_ctx*, int reset) {
  return reset ? g_launches.exchange(0) : g_launches.load();
}

int s2s_allocated_bytes(int64_t* out) {
  S2S_REQUIRE(out, "s2s_allocated_bytes: null argument");
  *out = (int64_t)g_device_bytes.load();
  return S2S_OK;
}

int s2s_init(int device, s2s_ctx** out) {
  S2S_REQUIRE(out, "s2s_init: null out");
  int n = 0;
  S2S_CHECK_CUDA(cudaGetDeviceCount(&n));
  S2S_REQUIRE(device >= 0 && device < n, "s2s_init: device %d not in [0,%d)", device, n);
  S2S_CHECK_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  S2S_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    s2s_set_error("s2s_init: device %d is sm_%d%d; this library is built for sm_90a (Hopper, H100) only", device, prop.major,
                  prop.minor);
    return S2S_ERR_UNSUPPORTED;
  }
  s2s_ctx* c = new s2s_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  c->decode_ctas = 0;
  c->encode_tiled = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &c->encode_tiled, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !c->encode_tiled) {
    s2s_set_error("s2s_init: cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
    delete c;
    return S2S_ERR_CUDA;
  }
  *out = c;
  return S2S_OK;
}

int s2s_set_sm_partition(s2s_ctx* ctx, int32_t ctas) {
  S2S_REQUIRE(ctx, "s2s_set_sm_partition: null context");
  S2S_REQUIRE(ctas == 0 || (ctas >= 8 && ctas <= ctx->num_sms), "s2s_set_sm_partition: %d CTAs not in [8, %d] (0 = all SMs)", ctas,
              ctx->num_sms);
  ctx->decode_ctas = ctas;
  return S2S_OK;
}

int s2s_destroy(s2s_ctx* ctx) {
  delete ctx;
  return S2S_OK;
}

int s2s_gemm_ex(s2s_ctx* ctx, const s2s_gemm_args* g, void* stream) {
  S2S_REQUIRE(ctx && g && g->a && g->w, "s2s_gemm_ex: null argument");
  GemmProblem p{};
  p.a = g->a; p.a_row_stride = g->a_row_stride; p.a_batch_stride = g->a_batch_stride;
  p.w = g->w; p.ldw = g->ldw; p.w_layout = g->w_layout;
  p.M = g->M; p.N = g->N; p.K = g->K; p.batch = g->batch;
  p.bias = g->bias; p.act = g->act;
  p.out_h = g->out_h; p.ldo_h = g->ldo_h; p.out_f = g->out_f; p.ldo_f = g->ldo_f;
  p.resid = g->resid; p.ld_resid = g->ld_resid; p.resid_mode = g->resid_mode;
  p.out_batch_rows = g->out_batch_rows; p.out_row_offset = g->out_row_offset; p.head_major_rows = g->head_major_rows;
  p.bn = g->bn;
  return gemm_tc_launch(ctx, p, g->dtype, (cudaStream_t)stream);
}

int s2s_norm_rows(s2s_ctx* ctx, const float* x, const float* w, const float* bias, float eps, int64_t rows, int32_t d,
                  void* out_h, float* out_f, int32_t dtype, void* stream) {
  auto al = [](const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
  S2S_REQUIRE(ctx && x && w, "s2s_norm_rows: null argument");
  S2S_REQUIRE(out_h || out_f, "s2s_norm_rows: no output");
  S2S_REQUIRE(rows >= 1 && d >= 4 && d % 4 == 0, "s2s_norm_rows: rows %lld, d %d (a multiple of 4)", (long long)rows, d);
  S2S_REQUIRE(dtype == S2S_F16 || dtype == S2S_BF16, "s2s_norm_rows: dtype %d", dtype);
  S2S_REQUIRE(al(x, 16) && al(w, 16) && al(bias, 16) && al(out_f, 16) && al(out_h, 8),
              "s2s_norm_rows: x / w / bias / out_f must be 16-byte aligned, out_h 8-byte aligned");
  return norm_rows_launch(x, w, bias, eps, rows, d, out_h, out_f, dtype, (cudaStream_t)stream);
}

int64_t s2s_tiled_weight_bytes(int32_t N, int32_t K, int32_t format) {
  if (N < 1 || K < 32 || K % 32 != 0) return 0;
  if (format == S2S_FP8_E4M3) return (int64_t)tiled_fp8_weight_bytes(N, K);
  return (format == S2S_F16 || format == S2S_BF16) ? (int64_t)tiled_weight_elems(N, K) * 2 : 0;
}

int s2s_tile_weights(s2s_ctx* ctx, const void* w_d, int32_t N, int32_t K, int32_t format, void* out_d, void* stream) {
  S2S_REQUIRE(ctx && w_d && out_d, "s2s_tile_weights: null argument");
  S2S_REQUIRE(format == S2S_F16 || format == S2S_BF16 || format == S2S_FP8_E4M3, "s2s_tile_weights: unknown format %d", format);
  S2S_REQUIRE(N >= 8 && N % 8 == 0 && K >= 32 && K % 32 == 0, "s2s_tile_weights: N=%d must be a multiple of 8, K=%d of 32", N, K);
  S2S_REQUIRE((reinterpret_cast<uintptr_t>(w_d) & 15) == 0 && (reinterpret_cast<uintptr_t>(out_d) & 15) == 0,
              "s2s_tile_weights: buffers must be 16-byte aligned");
  return tile_rows_launch(w_d, N, K, out_d, N, 0, 1, format == S2S_FP8_E4M3, (cudaStream_t)stream);
}

int s2s_attention(s2s_ctx* ctx, const void* q_d, const void* k_d, const void* v_d, void* o_d, int32_t B, int32_t Tq,
                  int32_t Tk, int32_t heads, int32_t kv_heads, int32_t hd, int64_t ldq, int64_t ldk, int64_t ldv,
                  int64_t ldo, float scale, int32_t causal, int32_t dtype, void* stream) {
  S2S_REQUIRE(ctx && q_d && k_d && v_d && o_d, "s2s_attention: null argument");
  // test / bench entry point: the V^T scratch of the attention kernel is allocated per call here (the models own theirs)
  const size_t elems = attention_tc_scratch_elems(B, Tk, kv_heads, hd);
  void* vt = nullptr;
  S2S_CHECK_CUDA(cudaMalloc(&vt, elems * 2));
  const int rc = attention_tc_launch(ctx, q_d, k_d, v_d, o_d, B, Tq, Tk, heads, kv_heads, hd, ldq, ldk, ldv, ldo, scale, causal,
                                      dtype, vt, elems, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);
  cudaFree(vt);
  return rc;
}

}  // extern "C"
