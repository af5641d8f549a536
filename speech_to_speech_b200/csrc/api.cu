// api.cu -- context, error reporting and the thin C-ABI wrappers around the stand-alone kernels.
#include <stdarg.h>

#include <atomic>

#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};   // process-wide: lanes launch from several host threads

void s2s_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void s2s_count_launch(int n) { g_launches += n; }

extern "C" {

const char* s2s_last_error(void) { return g_err; }

int64_t s2s_launch_count(s2s_ctx*, int reset) {
  return reset ? g_launches.exchange(0) : g_launches.load();
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

int s2s_gemm(s2s_ctx* ctx, const void* a_d, const void* w_d, const float* bias_d, void* c_d, int32_t M, int32_t N,
             int32_t K, int32_t dtype, int32_t out_dtype, int32_t act, void* stream) {
  S2S_REQUIRE(ctx && a_d && w_d && c_d, "s2s_gemm: null argument");
  GemmProblem p{};
  p.a = a_d; p.a_row_stride = K; p.a_batch_stride = (int64_t)K * M; p.w = w_d; p.ldw = K;
  p.M = M; p.N = N; p.K = K; p.batch = 1; p.bias = bias_d; p.act = act;
  if (out_dtype == S2S_F32) { p.out_f = (float*)c_d; p.ldo_f = N; }
  else { S2S_REQUIRE(out_dtype == dtype, "s2s_gemm: out_dtype must be f32 or the operand dtype"); p.out_h = c_d; p.ldo_h = N; }
  return gemm_tc_launch(ctx, p, dtype, (cudaStream_t)stream);
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
