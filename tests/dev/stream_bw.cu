// Developer microbenchmark (not part of the library): HBM read bandwidth of GEMV-like access patterns on H100.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o stream_bw stream_bw.cu && ./stream_bw
#include <cstdio>
#include <cuda_runtime.h>
#include <cstdint>

__device__ __forceinline__ uint4 ld16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// mode 0: "row pairs": item i = 2 rows of K halfs (contiguous 4K bytes*?); warp reads item via k-chunks of 1024 elems x 2 rows
// mode 1: contiguous units of UNIT bytes, unit u -> global warp (u % W), 16B per lane, UNIT/512 loads in flight
template <int LOADS>
__global__ void k_rows(const char* base, long long n_rows, int K, unsigned* sink) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
  const long long gw = (long long)warp * gridDim.x + blockIdx.x, GW = (long long)gridDim.x * wpc;
  unsigned acc = 0;
  const long long row_bytes = (long long)K * 2;
  for (long long it = gw; it * 2 < n_rows; it += GW) {
    const char* r0 = base + it * 2 * row_bytes;
    for (int k0 = lane * 16; k0 < row_bytes; k0 += 512 * (LOADS / 2)) {
      uint4 v[LOADS];
#pragma unroll
      for (int u = 0; u < LOADS / 2; ++u) {
        const int k = k0 + u * 512;
        if (k < row_bytes) { v[2 * u] = ld16(r0 + k); v[2 * u + 1] = ld16(r0 + row_bytes + k); }
      }
#pragma unroll
      for (int u = 0; u < LOADS / 2; ++u) {
        const int k = k0 + u * 512;
        if (k < row_bytes) acc ^= v[2 * u].x ^ v[2 * u + 1].y;
      }
    }
  }
  if (acc == 0x12345678u) *sink = acc;
}

template <int LOADS>
__global__ void k_contig(const char* base, long long bytes, unsigned* sink) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
  const long long gw = (long long)warp * gridDim.x + blockIdx.x, GW = (long long)gridDim.x * wpc;
  const long long unit = 512LL * LOADS;
  unsigned acc = 0;
  for (long long u = gw; (u + 1) * unit <= bytes; u += GW) {
    const char* p = base + u * unit + lane * 16;
    uint4 v[LOADS];
#pragma unroll
    for (int i = 0; i < LOADS; ++i) v[i] = ld16(p + i * 512);
#pragma unroll
    for (int i = 0; i < LOADS; ++i) acc ^= v[i].x;
  }
  if (acc == 0x12345678u) *sink = acc;
}

template <typename F> float timeit(F f, int reps = 5) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  f(); cudaDeviceSynchronize();
  float best = 1e9;
  for (int i = 0; i < reps; ++i) { cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best; }
  return best;
}

int main() {
  const long long bytes = 2LL << 30;  // 2 GiB >> L2
  char* buf; cudaMalloc(&buf, bytes); cudaMemset(buf, 1, bytes);
  unsigned* sink; cudaMalloc(&sink, 4);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int K : {4096, 14336, 768}) {
    const long long n_rows = bytes / (K * 2);
    for (int threads : {256, 512}) for (int mult : {1, 2}) {
      float ms = timeit([&] { k_rows<8><<<sms * mult, threads>>>(buf, n_rows, K, sink); });
      printf("rows   K=%5d loads=8  grid=%dx%d: %.0f GB/s\n", K, sms * mult, threads, n_rows * K * 2 / 1e6 / ms);
      ms = timeit([&] { k_rows<16><<<sms * mult, threads>>>(buf, n_rows, K, sink); });
      printf("rows   K=%5d loads=16 grid=%dx%d: %.0f GB/s\n", K, sms * mult, threads, n_rows * K * 2 / 1e6 / ms);
    }
  }
  for (int threads : {256, 512, 1024}) for (int mult : {1, 2}) {
    float ms = timeit([&] { k_contig<8><<<sms * mult, threads>>>(buf, bytes, sink); });
    printf("contig unit=4KB  grid=%dx%d: %.0f GB/s\n", sms * mult, threads, bytes / 1e6 / ms);
    ms = timeit([&] { k_contig<16><<<sms * mult, threads>>>(buf, bytes, sink); });
    printf("contig unit=8KB  grid=%dx%d: %.0f GB/s\n", sms * mult, threads, bytes / 1e6 / ms);
    ms = timeit([&] { k_contig<32><<<sms * mult, threads>>>(buf, bytes, sink); });
    printf("contig unit=16KB grid=%dx%d: %.0f GB/s\n", sms * mult, threads, bytes / 1e6 / ms);
  }
  return 0;
}
