"""float64 reference of the row norms (csrc/elementwise.cu norm_rows_kernel), the prefill RoPE / Qwen3 q/k norm + KV append
(csrc/llama.cu) and the Qwen3 decode q/k preparation (csrc/llama_decode.cu ld_qk_prepare), written in transformers' form.
Plain torch, so the same functions run on the CPU (tests/test_rope_norm_reference.py checks them against oracle/llama_ref.py)
and on the GPU (tests/test_gpu_rope_norm.py).

  * rope_table: the fp32 (cos, sin) table [max_pos][hd / 2][2] with the float32 arithmetic of llama.cu build();
  * to_pairs / from_pairs: the pair-adjacent head layout (W_ROPE_PERM, csrc/weight_arena.cuh) the kernels read -- element
    (j, j + hd / 2) of a head at (2j, 2j + 1) -- and back;
  * rotate_half / rope: LlamaRotaryEmbedding's apply_rotary_pos_emb on the unpermuted head, with cos / sin = cat(c, c);
  * rms_norm (LlamaRMSNorm / Qwen3RMSNorm) and layer_norm in float64."""
import numpy as np
import torch


def rope_table(max_pos, hd, theta):
    """float32 like build(): inv_j = 1 / theta^(2j / hd), angle = float32(p) * inv_j, (cos, sin) rounded to float32"""
    j = np.arange(hd // 2, dtype=np.float32)
    inv = (np.float32(1.0) / np.power(np.float32(theta), (np.float32(2.0) * j) / np.float32(hd))).astype(np.float32)
    ang = (np.arange(max_pos, dtype=np.float32)[:, None] * inv[None, :]).astype(np.float32)
    tab = np.stack([np.cos(ang.astype(np.float64)), np.sin(ang.astype(np.float64))], -1).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(tab))             # [max_pos][hd / 2][2]


def pair_perm(hd):
    """index p with paired[..., i] = natural[..., p[i]]: p[2j] = j, p[2j + 1] = j + hd / 2"""
    h = hd // 2
    return torch.stack([torch.arange(h), torch.arange(h) + h], -1).reshape(-1)


def to_pairs(x, hd):
    """natural head layout -> pair-adjacent, over the last dim of x [..., heads * hd] (or [..., hd])"""
    s = x.shape
    return x.reshape(*s[:-1], -1, hd)[..., pair_perm(hd).to(x.device)].reshape(s)


def from_pairs(x, hd):
    """pair-adjacent -> natural head layout (the inverse of to_pairs)"""
    s = x.shape
    inv = torch.argsort(pair_perm(hd)).to(x.device)
    return x.reshape(*s[:-1], -1, hd)[..., inv].reshape(s)


def cos_sin(tab, positions):
    """tab [max_pos][hd / 2][2], positions [T] -> cos, sin [T, hd] in float64 (transformers' cat(freqs, freqs))"""
    t = tab[positions].double()
    c, s = t[..., 0], t[..., 1]
    return torch.cat([c, c], -1), torch.cat([s, s], -1)


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat([-x[..., h:], x[..., :h]], -1)


def rope(x, cos, sin):
    """x [T, heads, hd] (natural layout), cos / sin [T, hd]"""
    return x * cos[:, None, :] + rotate_half(x) * sin[:, None, :]


def rope_abs(x, cos, sin):
    """|x0 c| + |x1 s| per rotated element: the magnitude the rotation's fp32 roundings are relative to"""
    return x.abs() * cos.abs()[:, None, :] + rotate_half(x).abs() * sin.abs()[:, None, :]


def rms_norm(x, w, eps):
    """Qwen3RMSNorm / LlamaRMSNorm: w * (x / sqrt(mean(x^2) + eps)) over the last dim"""
    return w * (x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps))


def layer_norm(x, w, b, eps):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * w + b
