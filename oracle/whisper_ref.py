"""numpy restatement of the Whisper arithmetic on the reference's STT path (TEST INFRASTRUCTURE).

The reference (`speech_to_speech/STT/whisper_stt_handler.py:83-87, 225-282`)
delegates to `transformers` (pinned >=4.57; 5.5.0 installed).  Each function cites the
transformers file it restates (TF = site-packages/transformers/models/whisper):

  log_mel_spectrogram  TF/feature_extraction_whisper.py:135-164 (+ pad/truncate :296-303)
  mel_filter_bank      transformers/audio_utils.py:453-545 (slaney scale + slaney norm)
  encoder_forward      TF/modeling_whisper.py:593-648, layer :380-414, attention :284-357
  cross_kv / decoder_step  TF/modeling_whisper.py:449-507, 691-797, proj_out :1081
  greedy_decode        TF/generation_whisper.py:383-968 short-form greedy with
                       SuppressTokens / SuppressTokensAtBegin (:1774-1813)
  detect_language      TF/generation_whisper.py:1610-1674

Pinned against transformers by tests/golden/make_golden.py -> tests/golden/whisper_*.npz.
All math is float32 (float64 only inside the FFT and the filter-bank construction).
"""
from __future__ import annotations

import math

import numpy as np

from .weights import WhisperGeometry

N_FFT = 400
HOP = 160
N_SAMPLES = 480000
N_FRAMES = 3000


# ----------------------------------------------------------------------------- features
def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    mels = 3.0 * f / 200.0
    logstep = 27.0 / np.log(6.4)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-30) / 1000.0) * logstep, mels)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    logstep = np.log(6.4) / 27.0
    return np.where(m >= 15.0, 1000.0 * np.exp(logstep * (m - 15.0)), 200.0 * m / 3.0)


def mel_filter_bank(n_mels: int, n_freq: int = 201, sr: int = 16000, fmax: float = 8000.0) -> np.ndarray:
    """[n_freq, n_mels] float64 triangular filters, slaney scale + slaney area norm."""
    mel_f = np.linspace(_hz_to_mel(0.0), _hz_to_mel(fmax), n_mels + 2)
    filt_hz = _mel_to_hz(mel_f)
    fft_hz = np.linspace(0, sr // 2, n_freq)
    diff = np.diff(filt_hz)
    slopes = filt_hz[None, :] - fft_hz[:, None]
    down = -slopes[:, :-2] / diff[:-1]
    up = slopes[:, 2:] / diff[1:]
    fb = np.maximum(0.0, np.minimum(down, up))
    fb *= (2.0 / (filt_hz[2 : n_mels + 2] - filt_hz[:n_mels]))[None, :]
    return fb


def hann_window(n: int = N_FFT) -> np.ndarray:
    """torch.hann_window(n) (periodic)."""
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)).astype(np.float32)


def log_mel_spectrogram(audio: np.ndarray, n_mels: int = 80) -> np.ndarray:
    """f32[N] -> f32[n_mels, 3000].  Pad/truncate to 30 s, centred reflect-padded STFT,
    drop last frame, |.|^2, mel, log10(clamp 1e-10), max(x, max-8), (x+4)/4."""
    x = np.zeros(N_SAMPLES, dtype=np.float32)
    n = min(len(audio), N_SAMPLES)
    x[:n] = audio[:n]
    xp = np.pad(x, (N_FFT // 2, N_FFT // 2), mode="reflect")
    idx = np.arange(N_FRAMES)[:, None] * HOP + np.arange(N_FFT)[None, :]
    frames = xp[idx] * hann_window()[None, :]  # [3000, 400] f32
    spec = np.fft.rfft(frames.astype(np.float64), axis=1)  # [3000, 201]
    power = (spec.real**2 + spec.imag**2).astype(np.float32)
    fb = mel_filter_bank(n_mels).astype(np.float32)  # [201, n_mels]
    mel = fb.T @ power.T  # [n_mels, 3000]
    log_spec = np.log10(np.maximum(mel, 1e-10))
    log_spec = np.maximum(log_spec, log_spec.max() - 8.0)
    return ((log_spec + 4.0) / 4.0).astype(np.float32)


# ----------------------------------------------------------------------------- primitives
def gelu(x: np.ndarray) -> np.ndarray:
    """Exact (erf) GELU, nn.functional.gelu default."""
    from scipy.special import erf

    return (0.5 * x * (1.0 + erf(x / np.float32(math.sqrt(2.0))))).astype(np.float32)


def layer_norm(x, w, b, eps=1e-5):
    mu = x.mean(axis=-1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=-1, keepdims=True)
    return ((x - mu) / np.sqrt(var + eps) * w + b).astype(np.float32)


def softmax(x):
    x = x - x.max(axis=-1, keepdims=True)
    e = np.exp(x)
    return e / e.sum(axis=-1, keepdims=True)


def linear(x, w, b=None):
    y = x @ w.T
    if b is not None:
        y = y + b
    return y.astype(np.float32)


def conv1d_k3(x, w, b, stride):
    """x [C_in, T], w [C_out, C_in, 3], padding 1 -> [C_out, T_out]."""
    xp = np.pad(x, ((0, 0), (1, 1)))
    t_out = (x.shape[1] + 2 - 3) // stride + 1
    out = np.zeros((w.shape[0], t_out), dtype=np.float32)
    for k in range(3):
        out += w[:, :, k] @ xp[:, k : k + stride * t_out : stride]
    return out + b[:, None]


def _split_heads(x, heads):
    t, d = x.shape
    return x.reshape(t, heads, d // heads).transpose(1, 0, 2)  # [H, T, hd]


def _merge_heads(x):
    h, t, hd = x.shape
    return x.transpose(1, 0, 2).reshape(t, h * hd)


def attention(w, prefix, x_q, kv_src, heads, mask=None, kv_cache=None):
    """WhisperAttention.forward: q is scaled BEFORE the matmul (modeling_whisper.py:305-310)."""
    hd = x_q.shape[-1] // heads
    q = linear(x_q, w[prefix + ".q_proj.weight"], w[prefix + ".q_proj.bias"]) * np.float32(hd**-0.5)
    if kv_cache is not None and "k" in kv_cache and kv_src is None:
        k, v = kv_cache["k"], kv_cache["v"]
    else:
        k = linear(kv_src, w[prefix + ".k_proj.weight"])
        v = linear(kv_src, w[prefix + ".v_proj.weight"], w[prefix + ".v_proj.bias"])
    qh, kh, vh = _split_heads(q, heads), _split_heads(k, heads), _split_heads(v, heads)
    s = qh @ kh.transpose(0, 2, 1)
    if mask is not None:
        s = s + mask
    p = softmax(s.astype(np.float32))
    o = _merge_heads((p @ vh).astype(np.float32))
    return linear(o, w[prefix + ".out_proj.weight"], w[prefix + ".out_proj.bias"]), k, v


# ----------------------------------------------------------------------------- encoder
def conv_frontend(w, g: WhisperGeometry, mel: np.ndarray) -> np.ndarray:
    """mel [n_mels, 3000] -> [1500, d]: conv1+GELU, conv2(stride 2)+GELU, + positions."""
    e = "model.encoder."
    h = gelu(conv1d_k3(mel, w[e + "conv1.weight"], w[e + "conv1.bias"], 1))
    h = gelu(conv1d_k3(h, w[e + "conv2.weight"], w[e + "conv2.bias"], 2))
    return (h.T + w[e + "embed_positions.weight"]).astype(np.float32)


def encoder_layer(w, g, i, x):
    p = f"model.encoder.layers.{i}."
    h = layer_norm(x, w[p + "self_attn_layer_norm.weight"], w[p + "self_attn_layer_norm.bias"])
    a, _, _ = attention(w, p + "self_attn", h, h, g.heads)
    x = x + a
    h = layer_norm(x, w[p + "final_layer_norm.weight"], w[p + "final_layer_norm.bias"])
    h = gelu(linear(h, w[p + "fc1.weight"], w[p + "fc1.bias"]))
    return (x + linear(h, w[p + "fc2.weight"], w[p + "fc2.bias"])).astype(np.float32)


def encoder_forward(w, g: WhisperGeometry, mel: np.ndarray, return_all: bool = False):
    x = conv_frontend(w, g, mel)
    hs = [x]
    for i in range(g.enc_layers):
        x = encoder_layer(w, g, i, x)
        hs.append(x)
    out = layer_norm(x, w["model.encoder.layer_norm.weight"], w["model.encoder.layer_norm.bias"])
    return (out, hs) if return_all else out


# ----------------------------------------------------------------------------- decoder
def cross_kv(w, g: WhisperGeometry, enc_out: np.ndarray):
    """Per decoder layer cross-attention K/V, computed once per utterance (modeling_whisper.py:325-336)."""
    out = []
    for i in range(g.dec_layers):
        p = f"model.decoder.layers.{i}.encoder_attn"
        k = linear(enc_out, w[p + ".k_proj.weight"])
        v = linear(enc_out, w[p + ".v_proj.weight"], w[p + ".v_proj.bias"])
        out.append((k, v))
    return out


class DecoderState:
    def __init__(self, g: WhisperGeometry, ckv):
        self.ckv = ckv
        self.self_k = [np.zeros((0, g.d_model), np.float32) for _ in range(g.dec_layers)]
        self.self_v = [np.zeros((0, g.d_model), np.float32) for _ in range(g.dec_layers)]
        self.pos = 0


def decoder_step(w, g: WhisperGeometry, st: DecoderState, token: int) -> np.ndarray:
    """One token through the decoder with KV cache -> f32 logits [vocab]."""
    d = "model.decoder."
    x = (w[d + "embed_tokens.weight"][token] + w[d + "embed_positions.weight"][st.pos])[None, :].astype(np.float32)
    for i in range(g.dec_layers):
        p = f"{d}layers.{i}."
        h = layer_norm(x, w[p + "self_attn_layer_norm.weight"], w[p + "self_attn_layer_norm.bias"])
        hd = g.d_model // g.heads
        q = linear(h, w[p + "self_attn.q_proj.weight"], w[p + "self_attn.q_proj.bias"]) * np.float32(hd**-0.5)
        k_new = linear(h, w[p + "self_attn.k_proj.weight"])
        v_new = linear(h, w[p + "self_attn.v_proj.weight"], w[p + "self_attn.v_proj.bias"])
        st.self_k[i] = np.concatenate([st.self_k[i], k_new], 0)
        st.self_v[i] = np.concatenate([st.self_v[i], v_new], 0)
        qh = _split_heads(q, g.heads)
        kh, vh = _split_heads(st.self_k[i], g.heads), _split_heads(st.self_v[i], g.heads)
        pr = softmax((qh @ kh.transpose(0, 2, 1)).astype(np.float32))
        a = _merge_heads((pr @ vh).astype(np.float32))
        x = x + linear(a, w[p + "self_attn.out_proj.weight"], w[p + "self_attn.out_proj.bias"])

        h = layer_norm(x, w[p + "encoder_attn_layer_norm.weight"], w[p + "encoder_attn_layer_norm.bias"])
        q = linear(h, w[p + "encoder_attn.q_proj.weight"], w[p + "encoder_attn.q_proj.bias"]) * np.float32(hd**-0.5)
        ck, cv = st.ckv[i]
        qh, kh, vh = _split_heads(q, g.heads), _split_heads(ck, g.heads), _split_heads(cv, g.heads)
        pr = softmax((qh @ kh.transpose(0, 2, 1)).astype(np.float32))
        a = _merge_heads((pr @ vh).astype(np.float32))
        x = x + linear(a, w[p + "encoder_attn.out_proj.weight"], w[p + "encoder_attn.out_proj.bias"])

        h = layer_norm(x, w[p + "final_layer_norm.weight"], w[p + "final_layer_norm.bias"])
        h = gelu(linear(h, w[p + "fc1.weight"], w[p + "fc1.bias"]))
        x = (x + linear(h, w[p + "fc2.weight"], w[p + "fc2.bias"])).astype(np.float32)
    x = layer_norm(x, w[d + "layer_norm.weight"], w[d + "layer_norm.bias"])
    st.pos += 1
    return (x @ w[d + "embed_tokens.weight"].T)[0].astype(np.float32)


def greedy_decode(
    w,
    g: WhisperGeometry,
    enc_out: np.ndarray,
    prefix: list[int],
    max_new_tokens: int,
    eos_id: int,
    suppress: list[int] | None = None,
    begin_suppress: list[int] | None = None,
    forced: list[int] | None = None,
    return_logits: bool = False,
):
    """Short-form greedy generate.  `forced` teacher-forces the fed-back token (margin-aware
    parity tests); returned ids are always the argmax at each step."""
    st = DecoderState(g, cross_kv(w, g, enc_out))
    logits = None
    for t in prefix:
        logits = decoder_step(w, g, st, int(t))
    ids, all_logits = [], []
    for step in range(max_new_tokens):
        lg = logits.copy()
        if suppress:
            lg[np.asarray(suppress)] = -np.inf
        if step == 0 and begin_suppress:
            lg[np.asarray(begin_suppress)] = -np.inf
        nxt = int(np.argmax(lg))
        ids.append(nxt)
        if return_logits:
            all_logits.append(lg)
        if nxt == eos_id and forced is None:
            break
        feed = nxt if forced is None else int(forced[step])
        if step + 1 < max_new_tokens:
            logits = decoder_step(w, g, st, feed)
    if return_logits:
        return ids, np.stack(all_logits)
    return ids


def detect_language(w, g: WhisperGeometry, enc_out: np.ndarray, sot_id: int, lang_ids: list[int]) -> int:
    """One decoder step from <|sot|>, non-language logits masked, argmax (generation_whisper.py:1610-1674)."""
    st = DecoderState(g, cross_kv(w, g, enc_out))
    logits = decoder_step(w, g, st, sot_id)
    mask = np.full_like(logits, -np.inf)
    mask[np.asarray(lang_ids)] = 0.0
    return int(np.argmax(logits + mask))


def transcribe_ids(w, g, audio, prefix, max_new_tokens, eos_id, suppress=None, begin_suppress=None):
    """audio f32[N] -> generated ids: the whole STT device path of WhisperSTTHandler.process."""
    mel = log_mel_spectrogram(audio, g.n_mels)
    enc = encoder_forward(w, g, mel)
    return greedy_decode(w, g, enc, prefix, max_new_tokens, eos_id, suppress, begin_suppress)
