"""float64 reference of the prefill / encoder GEMM (csrc/gemm_tc.cu, include/s2s_b200.h s2s_gemm_ex) and the layout helpers its
call sites imply.  Plain torch, so the same functions run on the CPU (tests/test_gemm_reference.py checks them against the
numpy oracle) and on the GPU (tests/test_gpu_gemm.py).

  * window_rows: A[b][m][k] = flat[b * batch_stride + m * row_stride + k] -- Whisper's convolutions read overlapping
    windows of the padded time-major activations (row stride C for conv1, 2 d for conv2, K = 3 C);
  * conv_rows: a [O][C][3] Conv1d weight in the W_CONV_ROWS order [O][3][C] (csrc/weight_arena.cuh) the GEMM multiplies;
  * untile: the tiled 16-bit / FP8 bytes of s2s_tile_weights -> the values the kernel multiplies (FP8: dq(Q) = Q * 2^e_n);
  * head_major_index: where the epilogue stores (row, column) of the cross-attention K/V projection, [b][layer][k|v][head][t][64];
  * swiglu / gelu: the epilogue's activations in float64 (SwiGLU over interleaved (gate, up) columns, W_INTERLEAVE)."""
import math

import torch


def window_rows(flat, row_stride, batch_stride, M, K, batch=1):
    """[batch, M, K] view of a flat tensor: element (b, m, k) at b * batch_stride + m * row_stride + k"""
    return torch.as_strided(flat, (batch, M, K), (batch_stride, row_stride, 1))


def conv_rows(w):
    """Conv1d weight [O][C][k] -> [O][k * C]: column t * C + c holds w[o][c][t] (W_CONV_ROWS)"""
    O, Cin, k = w.shape
    return w.permute(0, 2, 1).reshape(O, k * Cin)


def padded_time_major(x):
    """[C][T] -> [T + 2][C] with zero rows 0 and T + 1 (the padding of a k = 3, pad = 1 convolution)"""
    C, T = x.shape
    out = torch.zeros((T + 2, C), dtype=x.dtype, device=x.device)
    out[1:T + 1] = x.T
    return out


def untile(tiled, N, K, fmt):
    """tiled layout (include/s2s_b200.h s2s_tile_weights) -> [N, K] of the values the kernel multiplies: the 16-bit
    elements, or for fmt "fp8" dq(Q) = Q * 2^e_n in bfloat16 (exact: a 4-bit-significand code times a power of two)"""
    esz = 1 if fmt == "fp8" else 2
    dt = {"fp8": torch.float8_e4m3fn, "bf16": torch.bfloat16, "fp16": torch.float16}[fmt]
    rows = tiled[: N * K * esz].view(dt).view(N // 8, K // 32, 8, 4, 8).permute(0, 2, 1, 3, 4).reshape(N, K)
    if fmt != "fp8":
        return rows
    scale = tiled[N * K: N * K + 4 * N].view(torch.float32)
    return (rows.float() * scale[:, None]).to(torch.bfloat16)


def head_major_index(orow, n, N, R):
    """element offset of output (orow, n) with head_major_rows R: [orow / R][n / 64][orow % R][n % 64]"""
    ob, ot = orow // R, orow % R
    return ((ob * (N // 64) + n // 64) * R + ot) * 64 + n % 64


def gelu(v):
    return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))


def silu(g):
    return g / (1 + torch.exp(-g))


def swiglu(v):
    """columns 2j (gate) and 2j + 1 (up) -> silu(gate) * up in column j"""
    return silu(v[..., 0::2]) * v[..., 1::2]
