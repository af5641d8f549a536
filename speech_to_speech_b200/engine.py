"""Thin Python objects over the C ABI.  torch supplies device tensors / streams only; every FLOP on the
hot path runs in libs2s_b200.so."""
from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass
from typing import Mapping, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import (S2S_BF16, S2S_F16, S2S_F32, DTYPE_CODES, CodecConfig, LlamaConfig, Qwen3TTSConfig, S2SError, WhisperConfig,
                   WhisperDecodeOpts, check)

_ctx_lock = threading.Lock()
_ctx_by_device: dict[tuple, C.c_void_p] = {}
_lane_streams: dict[tuple, "torch.cuda.Stream"] = {}


def get_context(device: int = 0, lane: int = 0, lanes: int = 1) -> C.c_void_p:
    """One library context per CUDA device and lane (created on first use).  lanes > 1 partitions the SMs: the persistent
    decode kernels of the engines built on lane i use num_sms // lanes CTAs (s2s_set_sm_partition), so the lanes' decode
    launches -- issued from different CUDA streams (lane_stream) -- run side by side on one GPU."""
    if not torch.cuda.is_available():
        raise S2SError("speech_to_speech_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    if not (lanes >= 1 and 0 <= lane < lanes):
        raise ValueError(f"lane {lane} not in [0, {lanes})")
    lib = _lib.load()
    key = (device, lane, lanes)
    with _ctx_lock:
        if key not in _ctx_by_device:
            h = C.c_void_p()
            check(lib.s2s_init(device, C.byref(h)), "s2s_init")
            if lanes > 1:
                sms = torch.cuda.get_device_properties(device).multi_processor_count
                check(lib.s2s_set_sm_partition(h, sms // lanes), "s2s_set_sm_partition")
            _ctx_by_device[key] = h
        return _ctx_by_device[key]


def lane_stream(device: int = 0, lane: int = 0, lanes: int = 1) -> "torch.cuda.Stream":
    """The CUDA stream all work of a lane is issued on (engines take the calling thread's current stream: wrap the calls in
    `with torch.cuda.stream(lane_stream(...))`).  One lane: the device's default stream, as before."""
    if lanes <= 1:
        return torch.cuda.default_stream(device)
    key = (device, lane, lanes)
    with _ctx_lock:
        if key not in _lane_streams:
            _lane_streams[key] = torch.cuda.Stream(device=device)
        return _lane_streams[key]


def lane_context(device: int = 0, lane: int = 0, lanes: int = 1):
    """Context manager that makes the lane's stream the calling thread's current stream (a no-op for one lane).  Every thread
    that touches a lane's engines -- handler threads, the session batchers' engine threads -- works inside it, so allocation
    and use of every tensor of a lane happen on one stream."""
    import contextlib
    return contextlib.nullcontext() if lanes <= 1 else torch.cuda.stream(lane_stream(device, lane, lanes))


def launch_count(device: int = 0, reset: bool = False) -> int:
    return int(_lib.load().s2s_launch_count(get_context(device), 1 if reset else 0))


def _stream_ptr(device: int) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _np_dtype_code(a: np.ndarray) -> int:
    if a.dtype == np.float32:
        return S2S_F32
    if a.dtype == np.float16:
        return S2S_F16
    raise TypeError(f"unsupported numpy dtype {a.dtype}")


@dataclass
class WhisperDecodeOptions:
    """What WhisperGenerationMixin.generate derives from generation_config + the handler's gen_kwargs."""

    prefix: Sequence[int]
    eos_id: int
    max_new_tokens: int = 128
    suppress: Sequence[int] = ()
    begin_suppress: Sequence[int] = ()
    prefix_rows: Optional[Sequence[Sequence[int]]] = None   # one prompt per utterance (same length as `prefix`)

    def to_c(self):
        pre, n_pre = _lib.i32_array(self.prefix)
        sup, n_sup = _lib.i32_array(self.suppress)
        beg, n_beg = _lib.i32_array(self.begin_suppress)
        rows = None
        if self.prefix_rows is not None:
            flat = [int(t) for r in self.prefix_rows for t in r]
            if any(len(r) != n_pre for r in self.prefix_rows):
                raise ValueError("every row of prefix_rows must have len(prefix) tokens")
            rows, _ = _lib.i32_array(flat)
        o = WhisperDecodeOpts(pre, n_pre, int(self.max_new_tokens), int(self.eos_id), sup, n_sup, beg, n_beg,
                              C.cast(rows, C.POINTER(C.c_int32)) if rows is not None else None)
        o._keep = (pre, sup, beg, rows)  # keep the arrays alive
        return o


class WhisperEngine:
    """Whisper STT on one H100: log-mel -> encoder -> greedy decoder, batched over utterances."""

    def __init__(self, geometry: Mapping[str, int], dtype: str = "float16", max_batch: int = 1, device: int = 0,
                 lane: int = 0, lanes: int = 1):
        self.lib = _lib.load()
        self.device = device
        self.ctx = get_context(device, lane, lanes)
        self.geometry = dict(geometry)
        self.dtype = dtype
        self.max_batch = max_batch
        g = self.geometry
        self.cfg = WhisperConfig(
            g["d_model"], g["heads"], g["enc_layers"], g["dec_layers"], g["ffn"], g["n_mels"], g["vocab"],
            g.get("max_source_positions", 1500), g.get("max_target_positions", 448), DTYPE_CODES[dtype], max_batch)
        self.handle = C.c_void_p()
        check(self.lib.s2s_whisper_create(self.ctx, C.byref(self.cfg), C.byref(self.handle)), "s2s_whisper_create")

    # -- weights -----------------------------------------------------------------------------
    def load_state_dict(self, weights: Mapping[str, "np.ndarray | torch.Tensor"]) -> None:
        for name, w in weights.items():
            if isinstance(w, torch.Tensor):
                w = w.detach().to("cpu", torch.float32).numpy()
            a = np.ascontiguousarray(w)
            if a.dtype not in (np.float32, np.float16):
                a = a.astype(np.float32)
            shape = (C.c_int64 * max(1, a.ndim))(*a.shape)
            check(self.lib.s2s_whisper_bind_tensor(self.handle, name.encode(), a.ctypes.data_as(C.c_void_p), shape,
                                                   a.ndim, _np_dtype_code(a)), f"bind_tensor({name})")
        check(self.lib.s2s_whisper_finalize(self.handle), "s2s_whisper_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_whisper_init_random(self.handle, seed), "s2s_whisper_init_random")
        check(self.lib.s2s_whisper_finalize(self.handle), "s2s_whisper_finalize")

    # -- device-resident API -------------------------------------------------------------------
    def logmel(self, pcm: torch.Tensor, n_samples: Sequence[int], return_mel: bool = False) -> Optional[torch.Tensor]:
        """pcm: cuda f32 [B, stride].  Leaves the features inside the engine for encode()."""
        assert pcm.is_cuda and pcm.dtype == torch.float32 and pcm.dim() == 2 and pcm.is_contiguous()
        B = pcm.shape[0]
        ns, _ = _lib.i32_array(n_samples)
        mel = torch.empty((B, self.geometry["n_mels"], 3000), dtype=torch.float32, device=pcm.device) if return_mel else None
        check(self.lib.s2s_whisper_logmel(self.handle, _ptr(pcm), pcm.shape[1], ns, B, _ptr(mel),
                                          _stream_ptr(self.device)), "s2s_whisper_logmel")
        return mel

    def encode(self, B: int, mel: Optional[torch.Tensor] = None, return_output: bool = False) -> Optional[torch.Tensor]:
        if mel is not None:
            assert mel.is_cuda and mel.dtype == torch.float32 and mel.is_contiguous()
        out = None
        if return_output:
            out = torch.empty((B, 1500, self.geometry["d_model"]), dtype=torch.float32, device=f"cuda:{self.device}")
        check(self.lib.s2s_whisper_encode(self.handle, _ptr(mel), B, _ptr(out), _stream_ptr(self.device)),
              "s2s_whisper_encode")
        return out

    def decode(self, B: int, opts: WhisperDecodeOptions, forced: Optional[torch.Tensor] = None,
               return_logits: bool = False):
        dev = f"cuda:{self.device}"
        ids = torch.empty((B, opts.max_new_tokens), dtype=torch.int32, device=dev)
        lens = torch.empty((B,), dtype=torch.int32, device=dev)
        logits = None
        if return_logits:
            logits = torch.empty((opts.max_new_tokens, B, self.geometry["vocab"]), dtype=torch.float32, device=dev)
        co = opts.to_c()
        check(self.lib.s2s_whisper_decode(self.handle, C.byref(co), B, _ptr(ids), _ptr(lens), _ptr(forced), _ptr(logits),
                                          _stream_ptr(self.device)), "s2s_whisper_decode")
        return (ids, lens, logits) if return_logits else (ids, lens)

    def set_trace(self, trace: Optional[torch.Tensor]) -> None:
        """trace: cuda int64 [2, capacity, 6] or None (profiling aid, see include/s2s_b200.h)."""
        cap = 0 if trace is None else trace.shape[1]
        check(self.lib.s2s_whisper_set_trace(self.handle, _ptr(trace), cap), "s2s_whisper_set_trace")

    def detect_language(self, B: int, sot_id: int, lang_ids: Sequence[int]) -> torch.Tensor:
        out = torch.empty((B,), dtype=torch.int32, device=f"cuda:{self.device}")
        la, n = _lib.i32_array(lang_ids)
        check(self.lib.s2s_whisper_detect_language(self.handle, int(sot_id), la, n, B, _ptr(out), _stream_ptr(self.device)),
              "s2s_whisper_detect_language")
        return out

    def detect_language_host(self, audio: np.ndarray, sot_id: int, lang_ids: Sequence[int]) -> int:
        """Host PCM in: H2D + log-mel + encoder + one masked decoder step -> language token id."""
        pcm = torch.from_numpy(audio)[None].to(f"cuda:{self.device}")
        self.logmel(pcm, [pcm.shape[1]])
        self.encode(1)
        return int(self.detect_language(1, sot_id, lang_ids)[0])

    # -- host-buffer API (what the handler calls) --------------------------------------------------
    def transcribe(self, audio: Sequence[np.ndarray], opts: WhisperDecodeOptions) -> list[list[int]]:
        """audio: list of f32 mono 16 kHz arrays (host).  H2D + log-mel + encode + greedy decode + D2H."""
        B = len(audio)
        n = [min(len(a), 480000) for a in audio]
        stride = max(max(n), 1)
        if B == 1 and audio[0].dtype == np.float32 and audio[0].flags.c_contiguous:
            pcm = audio[0]
        else:
            pcm = np.zeros((B, stride), dtype=np.float32)
            for i, a in enumerate(audio):
                pcm[i, : n[i]] = a[: n[i]]
        ns, _ = _lib.i32_array(n)
        ids = np.empty((B, opts.max_new_tokens), dtype=np.int32)
        lens = np.empty((B,), dtype=np.int32)
        co = opts.to_c()
        check(self.lib.s2s_whisper_transcribe(self.handle, C.byref(co), pcm.ctypes.data_as(C.c_void_p), stride, ns, B,
                                              ids.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p),
                                              _stream_ptr(self.device)), "s2s_whisper_transcribe")
        return [ids[b, : lens[b]].tolist() for b in range(B)]

    def transcribe_auto(self, audio: Sequence[np.ndarray], sot_id: int, lang_ids: Sequence[int], make_opts) -> tuple:
        """Language detection and transcription on ONE encoder pass, like the reference (`_detect_language` hands its
        `encoder_outputs` to `generate`, S/STT/whisper_stt_handler.py:166-197, 236-241): log-mel + encoder once, one masked
        decoder step -> language token per utterance, then greedy decode with a per-utterance prompt.
        make_opts(lang_tokens: list[int]) -> WhisperDecodeOptions with `prefix_rows` set.  -> (ids per utterance, language tokens)."""
        B = len(audio)
        n = [min(len(a), 480000) for a in audio]
        dev = f"cuda:{self.device}"
        pcm = torch.zeros((B, max(max(n), 1)), dtype=torch.float32, device=dev)
        for i, a in enumerate(audio):
            pcm[i, : n[i]] = torch.from_numpy(np.ascontiguousarray(a[: n[i]], dtype=np.float32)).to(dev, non_blocking=True)
        self.logmel(pcm, n)
        self.encode(B)
        langs = self.detect_language(B, sot_id, lang_ids).cpu().tolist()
        opts = make_opts(langs)
        ids, lens = self.decode(B, opts)
        ids, lens = ids.cpu().numpy(), lens.cpu().numpy()
        return [ids[b, : lens[b]].tolist() for b in range(B)], langs

    def close(self) -> None:
        if self.handle:
            self.lib.s2s_whisper_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: str = "none",
         out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """C = A @ W^T (+bias) through the wgmma kernel; a [M,K], w [N,K] fp16/bf16 cuda tensors."""
    assert a.is_cuda and w.is_cuda and a.dtype == w.dtype and a.is_contiguous() and w.is_contiguous()
    dev = a.device.index or 0
    M, K = a.shape
    N = w.shape[0]
    code = {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[a.dtype]
    out_dtype = out_dtype or a.dtype
    ocode = S2S_F32 if out_dtype == torch.float32 else code
    c = torch.empty((M, N), dtype=out_dtype, device=a.device)
    lib = _lib.load()
    check(lib.s2s_gemm(get_context(dev), _ptr(a), _ptr(w), _ptr(bias), _ptr(c), M, N, K, code, ocode,
                       1 if act == "gelu" else 0, _stream_ptr(dev)), "s2s_gemm")
    return c


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, kv_heads: int, scale: float,
              causal: bool = False) -> torch.Tensor:
    """q [B,Tq,heads*hd], k/v [B,Tk,kv_heads*hd] (last dim contiguous; row strides taken from the tensors)."""
    assert q.is_cuda and q.dtype in (torch.float16, torch.bfloat16)
    B, Tq, dq = q.shape
    Tk = k.shape[1]
    hd = dq // heads
    dev = q.device.index or 0
    o = torch.empty((B, Tq, dq), dtype=q.dtype, device=q.device)
    code = {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[q.dtype]
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    assert q.stride(0) == Tq * q.stride(1) and k.stride(0) == Tk * k.stride(1) and v.stride(0) == Tk * v.stride(1)
    lib = _lib.load()
    check(lib.s2s_attention(get_context(dev), _ptr(q), _ptr(k), _ptr(v), _ptr(o), B, Tq, Tk, heads, kv_heads, hd,
                            q.stride(1), k.stride(1), v.stride(1), o.stride(1), float(scale), 1 if causal else 0, code,
                            _stream_ptr(dev)), "s2s_attention")
    return o


class LlamaEngine:
    """Llama-family LLM on one H100: wgmma prefill + persistent greedy decode with a per-session KV cache."""

    def __init__(self, geometry: Mapping[str, float], dtype: str = "bfloat16", max_sessions: int = 1,
                 max_positions: int = 2048, max_prefill: int = 512, device: int = 0, lane: int = 0, lanes: int = 1):
        self.lib = _lib.load()
        self.device = device
        self.ctx = get_context(device, lane, lanes)
        self.geometry = dict(geometry)
        g = self.geometry
        self.cfg = LlamaConfig(
            int(g["d_model"]), int(g["layers"]), int(g["heads"]), int(g["kv_heads"]), int(g["head_dim"]), int(g["ffn"]),
            int(g["vocab"]), float(g.get("rope_theta", 500000.0)), float(g.get("rms_eps", 1e-5)), DTYPE_CODES[dtype],
            max_sessions, min(max_positions, int(g.get("max_positions", max_positions))), max_prefill,
            int(bool(g.get("qk_norm", False))),  # Qwen3-style per-head q/k RMSNorm before RoPE
            int(g.get("n_tables", 1)))
        self.max_positions = self.cfg.max_positions
        self.handle = C.c_void_p()
        check(self.lib.s2s_llama_create(self.ctx, C.byref(self.cfg), C.byref(self.handle)), "s2s_llama_create")

    def load_state_dict(self, weights: Mapping[str, "np.ndarray | torch.Tensor"]) -> None:
        for name, w in weights.items():
            if isinstance(w, torch.Tensor):
                w = w.detach().to("cpu", torch.float32).numpy()
            a = np.ascontiguousarray(w)
            if a.dtype not in (np.float32, np.float16):
                a = a.astype(np.float32)
            shape = (C.c_int64 * max(1, a.ndim))(*a.shape)
            check(self.lib.s2s_llama_bind_tensor(self.handle, name.encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim,
                                                 _np_dtype_code(a)), f"llama bind_tensor({name})")
        check(self.lib.s2s_llama_finalize(self.handle), "s2s_llama_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_llama_init_random(self.handle, seed), "s2s_llama_init_random")
        check(self.lib.s2s_llama_finalize(self.handle), "s2s_llama_finalize")

    def reset(self, slot: int = 0) -> None:
        check(self.lib.s2s_llama_session_reset(self.handle, slot), "s2s_llama_session_reset")

    def prefill(self, slot: int, ids: Sequence[int], return_logits: bool = False):
        """Append `ids` to the session.  Returns (next_id cuda int32[1], logits cuda f32[n, vocab] or None)."""
        arr, n = _lib.i32_array(ids)
        dev = f"cuda:{self.device}"
        nxt = torch.empty((1,), dtype=torch.int32, device=dev)
        logits = torch.empty((n, self.geometry["vocab"]), dtype=torch.float32, device=dev) if return_logits else None
        check(self.lib.s2s_llama_prefill(self.handle, slot, arr, n, _ptr(logits), _ptr(nxt), _stream_ptr(self.device)),
              "s2s_llama_prefill")
        return nxt, logits

    def prefill_batch(self, slots: Sequence[int], prompts: Sequence[Sequence[int]]) -> torch.Tensor:
        """Append prompts[i] to session slots[i], all sessions in ONE pass over the weights (total tokens <= max_prefill,
        at most 16 sessions).  -> next ids, cuda int32[B] (asynchronous)."""
        assert len(slots) == len(prompts) and len(slots) >= 1
        sl, B = _lib.i32_array(slots)
        flat, _ = _lib.i32_array([t for p in prompts for t in p])
        ns, _ = _lib.i32_array([len(p) for p in prompts])
        nxt = torch.empty((B,), dtype=torch.int32, device=f"cuda:{self.device}")
        check(self.lib.s2s_llama_prefill_batch(self.handle, sl, B, flat, ns, _ptr(nxt), _stream_ptr(self.device)), "s2s_llama_prefill_batch")
        return nxt

    def decode(self, slots: Sequence[int], first_ids: torch.Tensor, n_steps: int, eos_id: int = -1,
               forced: Optional[torch.Tensor] = None, return_logits: bool = False):
        B = len(slots)
        dev = f"cuda:{self.device}"
        sl, _ = _lib.i32_array(slots)
        ids = torch.empty((B, n_steps), dtype=torch.int32, device=dev)
        lens = torch.empty((B,), dtype=torch.int32, device=dev)
        logits = torch.empty((n_steps, B, self.geometry["vocab"]), dtype=torch.float32, device=dev) if return_logits else None
        check(self.lib.s2s_llama_decode(self.handle, sl, B, _ptr(first_ids), n_steps, eos_id, _ptr(ids), _ptr(lens),
                                        _ptr(forced), _ptr(logits), _stream_ptr(self.device)), "s2s_llama_decode")
        return (ids, lens, logits) if return_logits else (ids, lens)

    def max_decode_batch(self) -> int:
        """Sessions one decode launch can carry for this geometry (shared-memory budget of the kernel)."""
        return int(self.lib.s2s_llama_max_decode_batch(self.handle))

    def set_trace(self, trace: Optional[torch.Tensor]) -> None:
        cap = 0 if trace is None else trace.shape[0]
        check(self.lib.s2s_llama_set_trace(self.handle, _ptr(trace), cap), "s2s_llama_set_trace")

    def generate(self, prompt: Sequence[int], max_new_tokens: int, eos_id: int = -1, slot: int = 0) -> list[int]:
        """Host ids in, host ids out: (chunked) prefill + greedy decode.  generate() semantics of the reference."""
        arr, n = _lib.i32_array(prompt)
        out = np.empty((max_new_tokens,), dtype=np.int32)
        ln = np.zeros((1,), dtype=np.int32)
        check(self.lib.s2s_llama_generate(self.handle, slot, arr, n, max_new_tokens, eos_id, out.ctypes.data_as(C.c_void_p),
                                          ln.ctypes.data_as(C.c_void_p), _stream_ptr(self.device)), "s2s_llama_generate")
        return out[: int(ln[0])].tolist()

    def close(self) -> None:
        if self.handle:
            self.lib.s2s_llama_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _bind_all(lib_fn, handle, weights: Mapping[str, "np.ndarray | torch.Tensor"], what: str, prefix: str = "") -> None:
    for name, w in weights.items():
        if isinstance(w, torch.Tensor):
            w = w.detach().to("cpu", torch.float32).numpy()
        a = np.ascontiguousarray(w)
        if a.dtype not in (np.float32, np.float16):
            a = a.astype(np.float32)
        shape = (C.c_int64 * max(1, a.ndim))(*a.shape)
        check(lib_fn(handle, (prefix + name).encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim, _np_dtype_code(a)),
              f"{what} bind_tensor({prefix}{name})")


def codec_config(g: Mapping, max_frames: int = 40, precision: int = 1, max_batch: int = 1) -> CodecConfig:
    """CodecConfig from a geometry mapping (oracle.code2wav_ref.Code2WavGeometry.to_dict() field names)."""
    cfg = CodecConfig()
    cfg.codebook_size, cfg.hidden, cfg.heads, cfg.kv_heads = int(g["codebook_size"]), int(g["hidden"]), int(g["heads"]), int(g["kv_heads"])
    cfg.inter, cfg.layers, cfg.quantizers = int(g["inter"]), int(g["layers"]), int(g["quantizers"])
    rates, ratios = list(g["upsample_rates"]), list(g["upsampling_ratios"])
    cfg.n_upsample_rates, cfg.n_upsampling_ratios = len(rates), len(ratios)
    for i, r in enumerate(rates):
        cfg.upsample_rates[i] = int(r)
    for i, r in enumerate(ratios):
        cfg.upsampling_ratios[i] = int(r)
    cfg.decoder_dim, cfg.sliding_window = int(g["decoder_dim"]), int(g["sliding_window"])
    cfg.rope_theta, cfg.rms_eps = float(g.get("rope_theta", 10000.0)), float(g.get("rms_eps", 1e-5))
    cfg.max_frames = int(max_frames)
    cfg.max_batch = int(max_batch)
    cfg.precision = int(g.get("precision", precision))   # 0: fp32 parity mode, 1: fp16 tensor-core contractions
    return cfg


class CodecEngine:
    """Codebook ids -> 24 kHz waveform on one H100 (the codec-decoder half of the TTS slot; csrc/codec_decode.cu)."""

    def __init__(self, geometry: Mapping, max_frames: int = 40, device: int = 0, precision: int = 1, _handle=None, _owner=None):
        self.lib = _lib.load()
        self.device = device
        self.ctx = get_context(device)
        self.geometry = dict(geometry)
        self._owner = _owner            # a Qwen3TTSEngine that owns the handle
        if _handle is not None:
            self.handle = _handle
            return
        self.cfg = codec_config(self.geometry, max_frames, precision)
        self.handle = C.c_void_p()
        check(self.lib.s2s_codec_create(self.ctx, C.byref(self.cfg), C.byref(self.handle)), "s2s_codec_create")

    def load_state_dict(self, weights) -> None:
        _bind_all(self.lib.s2s_codec_bind_tensor, self.handle, weights, "codec")
        check(self.lib.s2s_codec_finalize(self.handle), "s2s_codec_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_codec_init_random(self.handle, seed), "s2s_codec_init_random")
        check(self.lib.s2s_codec_finalize(self.handle), "s2s_codec_finalize")

    def samples(self, T: int) -> int:
        return int(self.lib.s2s_codec_samples(self.handle, T))

    @property
    def total_upsample(self) -> int:
        return int(self.lib.s2s_codec_total_upsample(self.handle))

    def decode(self, codes: torch.Tensor, ctx_frames: int = 0, return_hidden: bool = False):
        """codes int32 cuda [T, quantizers] (frame-major) -> wav f32 cuda [samples of frames ctx_frames..T)."""
        T = int(codes.shape[0])
        dev = f"cuda:{self.device}"
        wav = torch.empty((self.samples(T),), dtype=torch.float32, device=dev)
        hid = torch.empty((T, self.geometry["hidden"]), dtype=torch.float32, device=dev) if return_hidden else None
        n = C.c_int32(0)
        check(self.lib.s2s_codec_decode(self.handle, _ptr(codes.contiguous()), T, ctx_frames, _ptr(wav), C.byref(n), _ptr(hid),
                                        _stream_ptr(self.device)), "s2s_codec_decode")
        return (wav[: n.value], hid) if return_hidden else wav[: n.value]

    def close(self) -> None:
        if self.handle and self._owner is None:
            self.lib.s2s_codec_destroy(self.handle)
        self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Qwen3TTSEngine:
    """Talker + code predictor + codec decoder of the TTS slot on one H100 (csrc/qwen3tts.cu).  Geometry mapping =
    oracle.qwen3tts_ref.TTSGeometry.to_dict(); codec geometry = oracle.code2wav_ref.Code2WavGeometry.to_dict()."""

    def __init__(self, geometry: Mapping, codec_geometry: Mapping, dtype: str = "bfloat16", max_sessions: int = 4,
                 max_positions: int = 1024, max_text: int = 256, codec_max_frames: int = 40, device: int = 0, codec_precision: int = 1,
                 lane: int = 0, lanes: int = 1):
        self.lib = _lib.load()
        self.device = device
        self.ctx = get_context(device, lane, lanes)
        self.geometry = dict(geometry)
        g, t, p = self.geometry, dict(geometry["talker"]), dict(geometry["predictor"])
        cfg = Qwen3TTSConfig()
        cfg.d_model, cfg.layers, cfg.heads, cfg.kv_heads = int(t["d_model"]), int(t["layers"]), int(t["heads"]), int(t["kv_heads"])
        cfg.head_dim, cfg.ffn, cfg.vocab = int(t["head_dim"]), int(t["ffn"]), int(t["vocab"])
        assert int(p["d_model"]) == cfg.d_model, "talker and code predictor share the hidden width"
        cfg.cp_layers, cfg.cp_heads, cfg.cp_kv_heads = int(p["layers"]), int(p["heads"]), int(p["kv_heads"])
        cfg.cp_head_dim, cfg.cp_ffn, cfg.cp_vocab = int(p["head_dim"]), int(p["ffn"]), int(p["vocab"])
        cfg.n_groups, cfg.text_vocab, cfg.text_hidden = int(g["n_groups"]), int(g["text_vocab"]), int(g["text_hidden"])
        cfg.rope_theta, cfg.rms_eps = float(t["rope_theta"]), float(t["rms_eps"])
        cfg.compute_dtype = DTYPE_CODES[dtype]
        cfg.max_sessions, cfg.max_positions, cfg.max_text = max_sessions, max_positions, max_text
        for k in ("codec_eos", "codec_nothink", "codec_think_bos", "codec_think_eos", "codec_pad", "codec_bos",
                  "tts_bos", "tts_eos", "tts_pad", "im_start", "assistant", "newline"):
            setattr(cfg, k, int(g[k]))
        cfg.codec = codec_config(codec_geometry, codec_max_frames, codec_precision, max_batch=min(16, max_sessions))
        self.cfg = cfg
        self.n_groups = cfg.n_groups
        self.codec_eos = cfg.codec_eos
        self.handle = C.c_void_p()
        check(self.lib.s2s_qwen3tts_create(self.ctx, C.byref(cfg), C.byref(self.handle)), "s2s_qwen3tts_create")
        self.codec = CodecEngine(codec_geometry, device=device, _handle=C.c_void_p(self.lib.s2s_qwen3tts_codec(self.handle)), _owner=self)

    def load_state_dict(self, weights, codec_weights) -> None:
        _bind_all(self.lib.s2s_qwen3tts_bind_tensor, self.handle, weights, "qwen3tts")
        _bind_all(self.lib.s2s_qwen3tts_bind_tensor, self.handle, codec_weights, "qwen3tts", prefix="code2wav.")
        check(self.lib.s2s_qwen3tts_finalize(self.handle), "s2s_qwen3tts_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_qwen3tts_init_random(self.handle, seed), "s2s_qwen3tts_init_random")
        check(self.lib.s2s_qwen3tts_finalize(self.handle), "s2s_qwen3tts_finalize")

    def max_batch(self) -> int:
        return int(self.lib.s2s_qwen3tts_max_batch(self.handle))

    def prefill(self, slot: int, text_ids: Sequence[int], speaker_id: int) -> None:
        arr, n = _lib.i32_array(text_ids)
        check(self.lib.s2s_qwen3tts_prefill(self.handle, slot, arr, n, int(speaker_id), _stream_ptr(self.device)), "s2s_qwen3tts_prefill")

    def decode_frames(self, slots: Sequence[int], n_frames: int, forced: Optional[torch.Tensor] = None) -> torch.Tensor:
        """-> codes int32 cuda [B, n_frames, n_groups] (asynchronous).  forced (int32 cuda, same shape): teacher-forced
        feedback for parity tests; the returned codes are still the models' own decisions."""
        sl, B = _lib.i32_array(slots)
        codes = torch.empty((B, n_frames, self.n_groups), dtype=torch.int32, device=f"cuda:{self.device}")
        if forced is not None:
            forced = forced.to(torch.int32).contiguous()
            assert tuple(forced.shape) == (B, n_frames, self.n_groups)
        check(self.lib.s2s_qwen3tts_decode_frames(self.handle, sl, B, n_frames, _ptr(codes), _ptr(forced), _stream_ptr(self.device)),
              "s2s_qwen3tts_decode_frames")
        return codes

    def frames(self, slot: int) -> int:
        return int(self.lib.s2s_qwen3tts_frames(self.handle, slot))

    def set_frames(self, slot: int, n: int) -> None:
        check(self.lib.s2s_qwen3tts_set_frames(self.handle, slot, n), "s2s_qwen3tts_set_frames")

    def decode_audio(self, slot: int, n_new: int, left_context: int = 25) -> torch.Tensor:
        """Waveform (f32 cuda, 24 kHz) of the newest n_new frames of the slot."""
        cap = self.codec.samples(min(n_new + left_context, self.cfg.codec.max_frames))
        wav = torch.empty((cap,), dtype=torch.float32, device=f"cuda:{self.device}")
        n = C.c_int32(0)
        check(self.lib.s2s_qwen3tts_decode_audio(self.handle, slot, n_new, left_context, _ptr(wav), C.byref(n), _stream_ptr(self.device)),
              "s2s_qwen3tts_decode_audio")
        return wav[: n.value]

    def decode_audio_batch(self, slots: Sequence[int], n_new: int, left_context: int = 25) -> list:
        """Waveforms of the newest n_new frames of several sessions whose chunks have the same shape, in ONE launch sequence.
        -> list of f32 cuda tensors (views of one buffer)."""
        sl, B = _lib.i32_array(slots)
        cap = self.codec.samples(min(n_new + left_context, self.cfg.codec.max_frames))
        wav = torch.empty((B, cap), dtype=torch.float32, device=f"cuda:{self.device}")
        n = C.c_int32(0)
        check(self.lib.s2s_qwen3tts_decode_audio_batch(self.handle, sl, B, n_new, left_context, _ptr(wav), cap, C.byref(n),
                                                       _stream_ptr(self.device)), "s2s_qwen3tts_decode_audio_batch")
        return [wav[b, : n.value] for b in range(B)]

    def history_context(self, slot: int, n_new: int, left_context: int = 25) -> int:
        """Frames of history the next decode_audio(slot, n_new) will decode behind (chunked_decode's rule)."""
        start = self.frames(slot) - n_new
        return left_context if start - left_context > 0 else start

    def close(self) -> None:
        if self.handle:
            self.lib.s2s_qwen3tts_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
