"""CPU: the float64 reference of tests/rope_norm_ref.py, which tests/test_gpu_rope_norm.py holds the row norms, the prefill
RoPE / Qwen3 q/k norm and the decode own-key path to, against the numpy oracle (oracle/llama_ref.py) and torch's LayerNorm,
so the GPU file's reference is known to be right before a GPU is involved."""
import numpy as np
import pytest
import torch

import rope_norm_ref as R
from oracle import llama_ref
from oracle.weights import LlamaGeometry


def _geometry(hd, theta):
    return LlamaGeometry(d_model=4 * hd, layers=1, heads=4, kv_heads=2, head_dim=hd, ffn=128, vocab=64, rope_theta=theta)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
def test_rms_norm_equals_the_oracle(hd, eps):
    rng = np.random.default_rng(hd)
    x = rng.standard_normal((5, 3, hd)).astype(np.float32) * np.float32(1e-3)   # mean(x^2) near eps
    x[1] *= 1000
    w = (1 + 0.1 * rng.standard_normal(hd)).astype(np.float32)
    want = llama_ref.rms_norm(x, w, np.float32(eps))
    got = R.rms_norm(torch.from_numpy(x).double(), torch.from_numpy(w).double(), eps).numpy()
    np.testing.assert_allclose(got, want, rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("hd,theta", [(64, 1e6), (128, 5e5), (128, 1e6)])
def test_rope_equals_the_oracle_at_high_positions(hd, theta):
    """the table of build() and the transformers-form rotation agree with rope_cos_sin / apply_rope up to the last
    position of a 4096-position cache"""
    g = _geometry(hd, theta)
    pos = np.array([0, 1, 2, 511, 2047, 4094, 4095])
    cos, sin = llama_ref.rope_cos_sin(g, pos)
    tab = R.rope_table(4096, hd, theta)
    c, s = R.cos_sin(tab, torch.from_numpy(pos))
    np.testing.assert_allclose(c.numpy(), cos, rtol=0, atol=2e-7)
    np.testing.assert_allclose(s.numpy(), sin, rtol=0, atol=2e-7)
    rng = np.random.default_rng(hd)
    x = rng.standard_normal((len(pos), 3, hd)).astype(np.float32)
    want = llama_ref.apply_rope(x, cos, sin)
    got = R.rope(torch.from_numpy(x).double(), c, s).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("hd", [64, 128])
def test_pair_layout_round_trip_and_pairing(hd):
    """to_pairs puts the rotate_half partners (j, j + hd/2) of every head at (2j, 2j + 1) -- the W_ROPE_PERM rows -- and
    from_pairs undoes it; a rotation in the pair layout with table column j equals the natural-layout rope"""
    H = 3
    x = torch.arange(H * hd, dtype=torch.float64)[None]
    p = R.to_pairs(x, hd)
    for h in range(H):
        for j in range(hd // 2):
            assert p[0, h * hd + 2 * j] == h * hd + j and p[0, h * hd + 2 * j + 1] == h * hd + j + hd // 2
    assert torch.equal(R.from_pairs(p, hd), x)
    gen = torch.Generator().manual_seed(hd)
    v = torch.randn(2, H * hd, generator=gen, dtype=torch.float64)
    tab = R.rope_table(16, hd, 1e4)
    pos = torch.tensor([3, 15])
    c, s = R.cos_sin(tab, pos)
    want = R.to_pairs(R.rope(v.view(2, H, hd), c, s).reshape(2, -1), hd)
    vp = R.to_pairs(v, hd).view(2, H, hd // 2, 2)
    t = tab[pos].double()[:, None]                                   # [2, 1, hd / 2, 2]
    got = torch.stack([vp[..., 0] * t[..., 0] - vp[..., 1] * t[..., 1], vp[..., 1] * t[..., 0] + vp[..., 0] * t[..., 1]], -1)
    torch.testing.assert_close(got.reshape(2, -1), want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("d", [4, 36, 384, 1280])
def test_layer_norm_equals_torch(d):
    gen = torch.Generator().manual_seed(d)
    x = torch.randn(6, d, generator=gen, dtype=torch.float64) + 30
    x[2] = 1.5                                                       # constant row: variance 0, output = bias
    w = torch.randn(d, generator=gen, dtype=torch.float64)
    b = torch.randn(d, generator=gen, dtype=torch.float64)
    want = torch.nn.functional.layer_norm(x, (d,), w, b, 1e-5)
    torch.testing.assert_close(R.layer_norm(x, w, b, 1e-5), want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(R.layer_norm(x, w, b, 1e-5)[2], b, rtol=0, atol=0)
