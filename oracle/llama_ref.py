"""numpy restatement of the Llama-family arithmetic on the reference's LLM path (TEST INFRASTRUCTURE).

The reference (`speech_to_speech/LLM/language_model.py:800-892`) runs
`pipeline("text-generation")` over `AutoModelForCausalLM`; the math lives in transformers
(TF = site-packages/transformers/models/llama/modeling_llama.py):

  rms_norm          TF:53-71   (fp32 variance, weight * x_normed)
  rope_cos_sin      TF:73-137  (inv_freq = theta^(-2j/hd), float32)
  apply_rope        TF:140-168 (rotate_half convention: pairs (j, j + hd/2))
  attention         TF:187-289 (GQA repeat_kv, softmax in fp32, scaling hd^-0.5, causal)
  mlp               TF:171-184 (down(silu(gate(x)) * up(x)))
  forward / greedy  TF:355-500 + GenerationMixin greedy (argmax of the last position)
  qk_norm (Qwen3)   transformers models/qwen3/modeling_qwen3.py Qwen3Attention: RMSNorm(head_dim) on q and k before RoPE

Pinned against transformers by tests/golden/make_golden.py -> tests/golden/llama_*.npz.  float32 throughout.
"""
from __future__ import annotations

import numpy as np

from .weights import LlamaGeometry


def rms_norm(x, w, eps):
    var = (x.astype(np.float32) ** 2).mean(axis=-1, keepdims=True)
    return (w * (x * (1.0 / np.sqrt(var + eps)))).astype(np.float32)


def rope_cos_sin(g: LlamaGeometry, positions: np.ndarray):
    hd = g.head_dim
    inv_freq = (1.0 / (np.float32(g.rope_theta) ** (np.arange(0, hd, 2, dtype=np.float32) / np.float32(hd)))).astype(np.float32)
    freqs = positions.astype(np.float32)[:, None] * inv_freq[None, :]
    emb = np.concatenate([freqs, freqs], axis=-1)
    return np.cos(emb).astype(np.float32), np.sin(emb).astype(np.float32)  # [T, hd]


def rotate_half(x):
    h = x.shape[-1] // 2
    return np.concatenate([-x[..., h:], x[..., :h]], axis=-1)


def apply_rope(x, cos, sin):
    """x [T, heads, hd]; cos/sin [T, hd]."""
    return (x * cos[:, None, :] + rotate_half(x) * sin[:, None, :]).astype(np.float32)


def silu(x):
    return (x / (1.0 + np.exp(-x))).astype(np.float32)


def softmax(x):
    x = x - x.max(axis=-1, keepdims=True)
    e = np.exp(x)
    return e / e.sum(axis=-1, keepdims=True)


class KVCache:
    def __init__(self, g: LlamaGeometry):
        self.k = [np.zeros((0, g.kv_heads, g.head_dim), np.float32) for _ in range(g.layers)]
        self.v = [np.zeros((0, g.kv_heads, g.head_dim), np.float32) for _ in range(g.layers)]

    @property
    def length(self):
        return self.k[0].shape[0]


def forward(w, g: LlamaGeometry, ids: np.ndarray, cache: KVCache, return_hidden: bool = False, inputs_embeds=None):
    """ids [T] (or inputs_embeds [T, d], the `inputs_embeds=` path of the HF models) appended to the cache ->
    logits [T, vocab] (fp32)."""
    if inputs_embeds is not None:
        x = np.asarray(inputs_embeds, np.float32)
        T = x.shape[0]
    else:
        T = len(ids)
        x = w["model.embed_tokens.weight"][ids].astype(np.float32)
    past = cache.length
    cos, sin = rope_cos_sin(g, np.arange(past, past + T))
    hs = [x]
    grp = g.heads // g.kv_heads
    for i in range(g.layers):
        p = f"model.layers.{i}."
        h = rms_norm(x, w[p + "input_layernorm.weight"], g.rms_eps)
        q = (h @ w[p + "self_attn.q_proj.weight"].T).reshape(T, g.heads, g.head_dim)
        k = (h @ w[p + "self_attn.k_proj.weight"].T).reshape(T, g.kv_heads, g.head_dim)
        v = (h @ w[p + "self_attn.v_proj.weight"].T).reshape(T, g.kv_heads, g.head_dim)
        if getattr(g, "qk_norm", False):
            q = rms_norm(q, w[p + "self_attn.q_norm.weight"], g.rms_eps)
            k = rms_norm(k, w[p + "self_attn.k_norm.weight"], g.rms_eps)
        q, k = apply_rope(q, cos, sin), apply_rope(k, cos, sin)
        cache.k[i] = np.concatenate([cache.k[i], k], 0)
        cache.v[i] = np.concatenate([cache.v[i], v.astype(np.float32)], 0)
        kk = np.repeat(cache.k[i], grp, axis=1)  # [S, heads, hd]
        vv = np.repeat(cache.v[i], grp, axis=1)
        s = np.einsum("thd,shd->hts", q, kk) * np.float32(g.head_dim ** -0.5)
        S = past + T
        mask = np.triu(np.full((T, S), -np.inf, np.float32), k=past + 1)
        pr = softmax((s + mask[None]).astype(np.float32))
        a = np.einsum("hts,shd->thd", pr, vv).reshape(T, g.heads * g.head_dim).astype(np.float32)
        x = x + a @ w[p + "self_attn.o_proj.weight"].T
        h = rms_norm(x, w[p + "post_attention_layernorm.weight"], g.rms_eps)
        m = silu(h @ w[p + "mlp.gate_proj.weight"].T) * (h @ w[p + "mlp.up_proj.weight"].T)
        x = (x + m @ w[p + "mlp.down_proj.weight"].T).astype(np.float32)
        hs.append(x)
    xn = rms_norm(x, w["model.norm.weight"], g.rms_eps)
    logits = (xn @ w["lm_head.weight"].T).astype(np.float32)
    return (logits, hs, xn) if return_hidden else logits


def greedy_generate(w, g: LlamaGeometry, prompt: np.ndarray, max_new: int, eos_id: int = -1,
                    forced: np.ndarray | None = None, return_logits: bool = False):
    """Prefill + greedy decode.  ids[i] is always the argmax at step i; `forced` teacher-forces the feedback."""
    cache = KVCache(g)
    logits = forward(w, g, np.asarray(prompt), cache)[-1]
    ids, all_logits = [], []
    for step in range(max_new):
        nxt = int(np.argmax(logits))
        ids.append(nxt)
        if return_logits:
            all_logits.append(logits)
        if nxt == eos_id and forced is None:
            break
        feed = nxt if forced is None else int(forced[step])
        if step + 1 < max_new:
            logits = forward(w, g, np.asarray([feed]), cache)[-1]
    if return_logits:
        return ids, np.stack(all_logits)
    return ids
