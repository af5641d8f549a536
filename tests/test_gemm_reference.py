"""CPU: the layout helpers of tests/gemm_ref.py, which tests/test_gpu_gemm.py builds its float64 reference from, against
the numpy oracle and the layouts the decoder and the weight arena state -- so the GPU file's reference is known to be right
before a GPU is involved."""
import numpy as np
import pytest
import torch

import gemm_ref as G
from oracle import llama_ref, whisper_ref


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("C,O,T", [(80, 64, 40), (128, 32, 24), (64, 48, 30)])
def test_conv_windows_equal_the_oracle_conv(stride, C, O, T):
    """conv1 (stride 1: windows of the padded mel, row stride C) and conv2 (stride 2: row stride 2 C) as the GEMM reads
    them, with the weight in the W_CONV_ROWS order, equal oracle/whisper_ref.conv1d_k3"""
    rng = np.random.default_rng(C + O + T + stride)
    x = rng.standard_normal((C, T))
    w = rng.standard_normal((O, C, 3))
    b = rng.standard_normal(O)
    want = whisper_ref.conv1d_k3(x, w, b, stride).T                          # [T_out, O]
    M = want.shape[0]
    xp = G.padded_time_major(torch.from_numpy(x))                              # [T + 2][C]
    flat = torch.cat([xp.reshape(-1), torch.full((8 * C,), float("nan"), dtype=torch.float64)])   # NaN past the last row
    A = G.window_rows(flat, stride * C, (T + 2) * C, M, 3 * C)[0]
    assert torch.isfinite(A).all()
    got = A @ G.conv_rows(torch.from_numpy(w)).T + torch.from_numpy(b)
    np.testing.assert_allclose(got.numpy(), want, rtol=1e-5, atol=1e-4)


def test_window_rows_batch_stride():
    """batch b reads its own padded sequence: rows b * (T + 2) + m ... of the flat buffer"""
    B, T, C = 3, 10, 8
    flat = torch.arange(B * (T + 2) * C, dtype=torch.float64)
    A = G.window_rows(flat, C, (T + 2) * C, T, 3 * C, B)
    for b in range(B):
        for m in (0, 4, T - 1):
            start = (b * (T + 2) + m) * C
            assert torch.equal(A[b, m], flat[start: start + 3 * C])


def test_conv_rows_matches_the_arena_order():
    """W_CONV_ROWS (csrc/weight_arena.cuh): element (o, c, t) of [O][C][k] goes to (o * k + t) * C + c"""
    O, C, k = 5, 7, 3
    w = torch.arange(O * C * k, dtype=torch.float64).view(O, C, k)
    flat = G.conv_rows(w).reshape(-1)
    for o in range(O):
        for c in range(C):
            for t in range(k):
                assert flat[(o * k + t) * C + c] == w[o, c, t]


@pytest.mark.parametrize("B,T,layers,heads", [(2, 1500, 2, 12), (3, 7, 4, 20)])
def test_head_major_index_is_the_decoder_layout(B, T, layers, heads):
    """the K/V projection's column n = ((layer * 2 + kv) * heads + head) * 64 + c of row b * T + t lands at
    [b][layer][k|v][head][t][c], the cross-attention layout the Whisper decoder reads (csrc/whisper_decode.cu: K of
    (b, layer, head) at ((b * layers + layer) * 2 * H + h) * T * 64, V H heads later)"""
    N = layers * 2 * heads * 64
    rows = torch.arange(B * T)[:, None]
    cols = torch.arange(N)[None]
    idx = G.head_major_index(rows, cols, N, T)
    b, t = rows // T, rows % T
    layer, kv, head, c = cols // (2 * heads * 64), cols // (heads * 64) % 2, cols // 64 % heads, cols % 64
    want = (((b * layers + layer) * 2 + kv) * heads + head) * T * 64 + t * 64 + c
    assert torch.equal(idx, want)
    assert torch.equal(idx.reshape(-1).sort().values, torch.arange(B * T * N))     # a permutation of the buffer


def test_swiglu_over_interleaved_rows_equals_the_oracle_mlp():
    """W_INTERLEAVE puts gate row r at 2 r and up row r at 2 r + 1; the epilogue's silu(v[2j]) * v[2j + 1] is then the
    oracle's silu(h gate^T) * (h up^T) (oracle/llama_ref.py)"""
    rng = np.random.default_rng(3)
    R, d, f = 9, 64, 48
    h = rng.standard_normal((R, d))
    gate, up = rng.standard_normal((f, d)) / 8, rng.standard_normal((f, d)) / 8
    w_gu = np.empty((2 * f, d))
    w_gu[0::2], w_gu[1::2] = gate, up
    got = G.swiglu(torch.from_numpy(h @ w_gu.T)).numpy()
    want = llama_ref.silu(h @ gate.T) * (h @ up.T)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)


def test_gelu_is_the_exact_erf_gelu():
    x = np.linspace(-6, 6, 1001)
    np.testing.assert_allclose(G.gelu(torch.from_numpy(x)).numpy(), whisper_ref.gelu(x), rtol=1e-6, atol=1e-7)


def test_untile_inverts_the_documented_layout():
    """element (row 8t+g, k 32w+8j+e) at ((t*K/32 + w)*32 + 4g + j)*8 + e (include/s2s_b200.h), 16-bit and FP8"""
    N, K = 24, 96
    w = torch.arange(N * K, dtype=torch.float32).view(N, K).to(torch.bfloat16)
    flat = torch.empty(N * K, dtype=torch.bfloat16)
    for r in range(N):
        t, g = divmod(r, 8)
        for k in range(K):
            wi, rem = divmod(k, 32)
            j, e = divmod(rem, 8)
            flat[((t * (K // 32) + wi) * 32 + 4 * g + j) * 8 + e] = w[r, k]
    assert torch.equal(G.untile(flat.view(torch.uint8), N, K, "bf16"), w)
    codes = torch.tensor([0x38, 0x40, 0xB8, 0x00], dtype=torch.uint8).repeat(N * K // 4)   # 1, 2, -1, 0
    scales = (2.0 ** torch.arange(-4, N - 4, dtype=torch.float32))
    q = torch.cat([codes, scales.view(torch.uint8)])
    dq = G.untile(q, N, K, "fp8").double()
    vals = torch.tensor([1.0, 2.0, -1.0, 0.0], dtype=torch.float64).repeat(N * K // 4)
    want = (vals.view(N // 8, K // 32, 8, 4, 8).permute(0, 2, 1, 3, 4).reshape(N, K)) * scales.double()[:, None]
    assert torch.equal(dq, want)
