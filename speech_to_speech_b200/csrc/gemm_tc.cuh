// gemm_tc.cuh -- host interface of the wgmma + TMA GEMM (see gemm_tc.cu).
#pragma once
#include "common.cuh"

// C[b, m, n] = epilogue( sum_k A[b, m, k] * W[n, k] ), A and W K-major 16-bit, fp32 accumulate in registers.
// A is addressed through a 3-D TMA map (k, row, batch) so that convolution windows
// (overlapping rows: row stride < row length) need no im2col.
struct GemmProblem {
  const void* a;        // device, 16-bit
  int64_t a_row_stride; // elements between consecutive rows (>= K normally; < K for conv windows)
  int64_t a_batch_stride;
  const void* w;        // [N, ldw] device, 16-bit
  int64_t ldw;
  int32_t M;            // rows per batch
  int32_t N;            // multiple of 64
  int32_t K;            // any multiple of 8
  int32_t batch;
  // epilogue
  const float* bias;    // [N] or null
  int32_t act;          // 0 none, 1 exact GELU, 2 SwiGLU over interleaved (gate, up) columns -> out_h [.., N/2]
  void* out_h;          // 16-bit output or null
  int64_t ldo_h;
  float* out_f;         // fp32 output or null:  out_f = v (+ resid)
  int64_t ldo_f;
  const float* resid;   // fp32 residual or null
  int64_t ld_resid;
  int32_t resid_mode;   // 1: same row index as the output, 2: row index = m (broadcast over batch)
  int64_t out_batch_rows; // output row = b * out_batch_rows + out_row_offset + m
  int64_t out_row_offset;
  // > 0: out_h is written as [row / R][N / 64][R][64] (R = head_major_rows): every 64-column block (one attention head)
  // of a row range is contiguous -- the layout the decode kernels stream K/V in.  0: plain row-major with ldo_h.
  int32_t head_major_rows;
};

int gemm_tc_launch(s2s_ctx* ctx, const GemmProblem& p, int dtype, cudaStream_t stream);

// 128-byte-swizzled tiled TMA descriptor (cuTensorMapEncodeTiled through the runtime-resolved driver entry point)
int tma_encode_map(s2s_ctx* ctx, CUtensorMap* map, CUtensorMapDataType dt, int rank, const void* base,
                   const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box);
