"""Thin Python objects over the C ABI.  torch supplies device tensors / streams only; every FLOP on the
hot path runs in libs2s_b200.so."""
from __future__ import annotations

import ctypes as C
import threading
from dataclasses import dataclass
from typing import Any, Mapping, Optional, Sequence

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


def allocated_bytes(device: int = 0) -> int:
    """Device bytes the library's model objects hold right now, counted at every allocation and free (include/s2s_b200.h
    s2s_allocated_bytes).  The count is process-wide, over all devices and lanes; other processes on the GPU do not move it."""
    get_context(device)
    n = C.c_int64(0)
    check(_lib.load().s2s_allocated_bytes(C.byref(n)), "s2s_allocated_bytes")
    return int(n.value)


def _device_bytes(fn, handle, what: str) -> tuple[int, int]:
    w, t = C.c_int64(0), C.c_int64(0)
    check(fn(handle, C.byref(w), C.byref(t)), what)
    return int(w.value), int(t.value)


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
        _bind_all(self.lib.s2s_whisper_bind_tensor, self.handle, weights, "whisper")
        check(self.lib.s2s_whisper_finalize(self.handle), "s2s_whisper_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_whisper_init_random(self.handle, seed), "s2s_whisper_init_random")
        check(self.lib.s2s_whisper_finalize(self.handle), "s2s_whisper_finalize")

    def share(self, lane: int, lanes: int, max_batch: Optional[int] = None) -> "WhisperEngine":
        """A new engine on lane `lane` of `lanes` that reads this engine's weights (one copy per GPU): its own workspaces and
        caches, sized by max_batch (default: this engine's).  This engine must be loaded; neither can be reloaded while both
        live.  Bit for bit what an engine loaded with the same weights computes (include/s2s_b200.h shared weights)."""
        eng = object.__new__(WhisperEngine)
        eng.lib, eng.device, eng.geometry, eng.dtype = self.lib, self.device, dict(self.geometry), self.dtype
        eng.ctx = get_context(self.device, lane, lanes)
        eng.cfg = WhisperConfig.from_buffer_copy(self.cfg)
        if max_batch is not None:
            eng.cfg.max_batch = max_batch
        eng.max_batch = eng.cfg.max_batch
        eng.handle = C.c_void_p()
        check(self.lib.s2s_whisper_create_shared(eng.ctx, self.handle, C.byref(eng.cfg), C.byref(eng.handle)),
              "s2s_whisper_create_shared")
        return eng

    def device_bytes(self) -> tuple[int, int]:
        """(weights, total): device bytes of the weights the engine reads (its own, or those it shares) and that plus
        what the engine allocated itself (log-mel tables, workspaces, KV caches)."""
        return _device_bytes(self.lib.s2s_whisper_device_bytes, self.handle, "s2s_whisper_device_bytes")

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
GEMM_W_LAYOUTS = {"row_major": 0, "tiled": 1, "float8_e4m3": 2}
GEMM_ACTS = {"none": 0, "gelu": 1, "swiglu": 2}


def gemm_ex(a: torch.Tensor, w: torch.Tensor, M: int, N: int, K: int, *, dtype: Optional[torch.dtype] = None,
            **fields: Any) -> None:
    """One call of the prefill / encoder GEMM in any form the engines use (include/s2s_b200.h s2s_gemm_ex), written into
    the caller's tensors.  `fields` maps the other s2s_gemm_args field names to values: cuda tensors are passed as their
    device pointers (a view's pointer is its first element), `w_layout` and `act` may be names (GEMM_W_LAYOUTS,
    GEMM_ACTS).  Defaults: a_row_stride = ldw = K, a_batch_stride = M * a_row_stride, batch 1, dtype = a's 16-bit type
    (a uint8 view of the operand needs dtype).  Asynchronous on the current stream."""
    assert a.is_cuda and w.is_cuda
    g = _lib.GemmArgs()
    g.a, g.w, g.M, g.N, g.K = a.data_ptr(), w.data_ptr(), M, N, K
    g.a_row_stride, g.ldw, g.batch = K, K, 1
    for k, v in fields.items():
        if isinstance(v, torch.Tensor):
            assert v.is_cuda, k
            v = v.data_ptr()
        elif k == "w_layout" and isinstance(v, str):
            v = GEMM_W_LAYOUTS[v]
        elif k == "act" and isinstance(v, str):
            v = GEMM_ACTS[v]
        elif v is None:
            v = 0
        setattr(g, k, v)
    if "a_batch_stride" not in fields:
        g.a_batch_stride = M * g.a_row_stride
    g.dtype = {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[dtype or a.dtype]
    dev = a.device.index or 0
    check(_lib.load().s2s_gemm_ex(get_context(dev), C.byref(g), _stream_ptr(dev)), "s2s_gemm_ex")


def _gemm_out(M: int, N: int, a: torch.Tensor, out_dtype: Optional[torch.dtype]) -> tuple[torch.Tensor, dict]:
    out_dtype = out_dtype or a.dtype
    assert out_dtype in (torch.float32, a.dtype), "out_dtype must be float32 or the operand dtype"
    c = torch.empty((M, N), dtype=out_dtype, device=a.device)
    return c, (dict(out_f=c, ldo_f=N) if out_dtype == torch.float32 else dict(out_h=c, ldo_h=N))


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: str = "none",
         out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """C = A @ W^T (+bias) through the wgmma kernel; a [M,K], w [N,K] fp16/bf16 cuda tensors."""
    assert a.is_cuda and w.is_cuda and a.dtype == w.dtype and a.is_contiguous() and w.is_contiguous()
    M, K = a.shape
    N = w.shape[0]
    c, out = _gemm_out(M, N, a, out_dtype)
    gemm_ex(a, w, M, N, K, bias=bias, act=act, **out)
    return c


def tile_weights(w: torch.Tensor, weight_dtype: Optional[str] = None) -> torch.Tensor:
    """w [N, K] fp16/bf16 cuda (N a multiple of 8, K of 32) -> the tiled layout the Llama-family engines store their
    projections in (include/s2s_b200.h s2s_tile_weights), as a flat uint8 cuda tensor: 16-bit tiles, or with
    weight_dtype="float8_e4m3" (bf16 w) E4M3 codes followed by the fp32 row scales."""
    assert w.is_cuda and w.dim() == 2 and w.is_contiguous() and w.dtype in (torch.float16, torch.bfloat16)
    N, K = w.shape
    fmt = _lib.WEIGHT_FORMAT_CODES[weight_dtype] if weight_dtype else {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[w.dtype]
    lib = _lib.load()
    nbytes = int(lib.s2s_tiled_weight_bytes(N, K, fmt))
    if nbytes <= 0:
        raise ValueError(f"no tiled layout for a [{N}, {K}] matrix")
    out = torch.empty((nbytes,), dtype=torch.uint8, device=w.device)
    dev = w.device.index or 0
    check(lib.s2s_tile_weights(get_context(dev), _ptr(w), N, K, fmt, _ptr(out), _stream_ptr(dev)), "s2s_tile_weights")
    return out


def gemm_tiled(a: torch.Tensor, wt: torch.Tensor, N: int, weight_dtype: Optional[str] = None, bias: Optional[torch.Tensor] = None,
               act: str = "none", out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """gemm() with the weight operand in the tiled layout of tile_weights(): a [M, K] fp16/bf16 cuda, wt from
    tile_weights(w [N, K], weight_dtype).  FP8 computes exactly gemm(a, dq(q(w)))."""
    assert a.is_cuda and wt.is_cuda and a.is_contiguous() and wt.is_contiguous()
    M, K = a.shape
    fmt = _lib.WEIGHT_FORMAT_CODES[weight_dtype] if weight_dtype else {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[a.dtype]
    assert wt.numel() * wt.element_size() >= int(_lib.load().s2s_tiled_weight_bytes(N, K, fmt)), "wt is smaller than the tiled [N, K] matrix"
    c, out = _gemm_out(M, N, a, out_dtype)
    gemm_ex(a, wt, M, N, K, w_layout=weight_dtype or "tiled", bias=bias, act=act, **out)
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


def decode_attention(q: torch.Tensor, kv: torch.Tensor, slots: Sequence[int], lens: Sequence[int], heads: int, kv_heads: int,
                     *, grid: int = 0, assoc_b: int = 0, kraw: Optional[torch.Tensor] = None, q_norm: Optional[torch.Tensor] = None,
                     k_norm: Optional[torch.Tensor] = None, rope: Optional[torch.Tensor] = None, eps: float = 1e-6,
                     qn_out: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, int]:
    """One attention phase of the Llama-family decode by itself (include/s2s_b200.h s2s_decode_attention).  q: cuda f32
    [B, heads, hd], softmax scale applied; kv: 16-bit [slots, 2, max_pos, kv_heads * hd] (K rows, then V rows, per slot);
    session b attends the first lens[b] keys of slot slots[b].  -> (out [B, heads, hd] in kv's dtype, the split plan:
    splits | 0x80 for warp-level items).  Synchronous.
    Qwen3 mode (kraw given): q is the raw q, kraw f32 [B, kv_heads, hd] the step's raw keys, q_norm / k_norm f32 [hd]
    (pair-adjacent), rope f32 [max_pos, hd / 2, 2] (cos, sin); the kernel normalises, rotates and scales q (into qn_out
    [B, heads, hd] when given) and writes key lens[b] - 1 of every session into kv before it attends."""
    assert q.is_cuda and q.dtype == torch.float32 and q.dim() == 3 and q.is_contiguous()
    assert kv.is_cuda and kv.dtype in (torch.float16, torch.bfloat16) and kv.dim() == 4 and kv.shape[1] == 2 and kv.is_contiguous()
    B, H, hd = q.shape
    assert H == heads and kv.shape[3] == kv_heads * hd and len(slots) == B and len(lens) == B
    out = torch.empty((B, heads, hd), dtype=kv.dtype, device=q.device)
    sl, _ = _lib.i32_array(slots)
    ln, _ = _lib.i32_array(lens)
    a = _lib.DecAttnArgs(q=q.data_ptr(), kv=kv.data_ptr(), max_pos=kv.shape[2], slots_h=sl, lens_h=ln, B=B, heads=heads,
                         kv_heads=kv_heads, hd=hd, dtype={torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[kv.dtype],
                         grid=grid, assoc_b=assoc_b, out=out.data_ptr())
    if kraw is not None:
        for t in (kraw, q_norm, k_norm, rope, qn_out):
            assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
        a.qk_norm, a.kraw, a.q_norm, a.k_norm, a.rope = 1, kraw.data_ptr(), _ptr(q_norm), _ptr(k_norm), _ptr(rope)
        a.eps, a.qn_out = float(eps), _ptr(qn_out)
    plan = C.c_int32(0)
    dev = q.device.index or 0
    check(_lib.load().s2s_decode_attention(get_context(dev), C.byref(a), C.byref(plan), _stream_ptr(dev)),
          "s2s_decode_attention")
    return out, int(plan.value)


_CODE16 = {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}


def norm_rows(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, eps: float = 1e-5, *,
              out_h: Optional[torch.Tensor] = None, out_f: Optional[torch.Tensor] = None, dtype: Optional[torch.dtype] = None) -> None:
    """The prefill / encoder row norm (include/s2s_b200.h s2s_norm_rows) over x f32 [rows, d]: LayerNorm with `bias`, RMSNorm
    without, written into out_h (16-bit) and / or out_f (f32), [rows, d] each.  dtype: the 16-bit type (default out_h's,
    else bfloat16).  Asynchronous on the current stream."""
    for t in (x, w, bias, out_h, out_f):
        assert t is None or (t.is_cuda and t.is_contiguous())
    rows, d = x.shape
    code = _CODE16[dtype or (out_h.dtype if out_h is not None else torch.bfloat16)]
    dev = x.device.index or 0
    check(_lib.load().s2s_norm_rows(get_context(dev), _ptr(x), _ptr(w), _ptr(bias), float(eps), rows, d, _ptr(out_h), _ptr(out_f),
                                    code, _stream_ptr(dev)), "s2s_norm_rows")


def prefill_rope(qkv: torch.Tensor, heads: int, kv_heads: int, past: int, rope: torch.Tensor, kcache: torch.Tensor,
                 vcache: torch.Tensor, *, q_norm: Optional[torch.Tensor] = None, k_norm: Optional[torch.Tensor] = None,
                 eps: float = 1e-6) -> None:
    """The RoPE / KV-append step of a Llama-family prefill (include/s2s_b200.h s2s_prefill_rope): qkv 16-bit [n, (heads +
    2 kv_heads) hd] (pair-adjacent q / k), rope f32 [max_pos, hd / 2, 2], caches 16-bit [max_pos, kv_heads * hd]; q_norm /
    k_norm f32 [hd] select the Qwen3 q/k norm.  q is rewritten in place, rows [past, past + n) of the caches are written.
    Asynchronous on the current stream."""
    for t in (qkv, rope, kcache, vcache, q_norm, k_norm):
        assert t is None or (t.is_cuda and t.is_contiguous())
    n = qkv.shape[0]
    hd = qkv.shape[1] // (heads + 2 * kv_heads)
    dev = qkv.device.index or 0
    check(_lib.load().s2s_prefill_rope(get_context(dev), _ptr(qkv), n, heads, kv_heads, hd, past, _ptr(rope), kcache.shape[0],
                                       _ptr(q_norm), _ptr(k_norm), float(eps), _ptr(kcache), _ptr(vcache), _CODE16[qkv.dtype],
                                       _stream_ptr(dev)), "s2s_prefill_rope")


def argmax_row(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The greedy token choice after a prefill (include/s2s_b200.h s2s_argmax_row) over logits f32 [n] -> int32 [1]
    (into `out` when given).  Asynchronous on the current stream."""
    assert logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous()
    out = torch.empty((1,), dtype=torch.int32, device=logits.device) if out is None else out
    dev = logits.device.index or 0
    check(_lib.load().s2s_argmax_row(get_context(dev), _ptr(logits), logits.numel(), _ptr(out), _stream_ptr(dev)), "s2s_argmax_row")
    return out


GEMV_MODES = {"store": 0, "gelu": 1, "resid": 2, "qkv": 3, "logits": 4, "qkv_rope": 5, "swiglu": 6}
GEMV_INPUTS = {"copy": 0, "norm": 1, "norm_sum": 2, "chunked": 3}


def decode_gemv(projs: Sequence[Mapping[str, Any]], B: int, dtype: torch.dtype, *, weight_dtype: Optional[str] = None,
                llama: bool = True, grid: int = 0, slots: int = 0, prefetch: bool = False, use_plans: bool = False,
                drain: bool = False, cluster: int = 0, heads: int = 0) -> list[tuple[int, ...]]:
    """1..3 projections of the decode kernels' skinny GEMM in one launch (include/s2s_b200.h s2s_decode_gemv).  Each entry of
    `projs` maps s2s_dec_gemv_proj field names to values: contiguous cuda tensors are passed as their device pointers,
    `mode` and `input` may be names (GEMV_MODES, GEMV_INPUTS); w comes from tile_weights().  The epilogues write into the
    caller's tensors.  -> per projection (n_tiles, main_rounds, ks_log, slice, tail_rounds) of CTA 0.  Synchronous."""
    a = _lib.DecGemvArgs()
    for i, pr in enumerate(projs):
        dst = a.proj[i]
        for k, v in pr.items():
            if isinstance(v, torch.Tensor):
                assert v.is_cuda and v.is_contiguous(), k
                v = v.data_ptr()
            elif k == "mode" and isinstance(v, str):
                v = GEMV_MODES[v]
            elif k == "input" and isinstance(v, str):
                v = GEMV_INPUTS[v]
            setattr(dst, k, v)
    code = {torch.float16: S2S_F16, torch.bfloat16: S2S_BF16}[dtype]
    a.n_proj, a.B, a.dtype, a.llama = len(projs), B, code, int(llama)
    a.weight_format = _lib.WEIGHT_FORMAT_CODES[weight_dtype] if weight_dtype else code
    a.grid, a.slots, a.prefetch, a.use_plans, a.drain = grid, slots, int(prefetch), int(use_plans), int(drain)
    a.cluster, a.heads = cluster, heads
    plans = (C.c_int32 * (5 * 3))()
    dev = torch.cuda.current_device()
    check(_lib.load().s2s_decode_gemv(get_context(dev), C.byref(a), plans, _stream_ptr(dev)), "s2s_decode_gemv")
    return [tuple(plans[5 * i: 5 * i + 5]) for i in range(len(projs))]


def codec_contract(x: Optional[torch.Tensor], w: torch.Tensor, y: torch.Tensor, *, path: int = 0,
                   x16: Optional[torch.Tensor] = None, T_in: Optional[int] = None, T_out: Optional[int] = None, x_row0: int = 0,
                   dil: int = 1, bias: Optional[torch.Tensor] = None, bias_mod: Optional[int] = None, act: int = 0,
                   scale: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None, t0: int = 0) -> None:
    """One codec-decoder contraction written into `y` on kernel `path` (0 fp32, 1 tensor cores converting, 2 tensor cores
    reading `x16`; include/s2s_b200.h s2s_codec_contract).  Contiguous cuda tensors: x f32 / x16 f16 [B, rows, ldx] (or
    [rows, ldx]), w f32 [k, C_in, N], y and resid f32 [B, rows, ld]; resid may be y.  Row and sequence strides come from the
    shapes; T_in / T_out default to the row counts of x and y.  Synchronous."""
    xs = x if x is not None else x16
    for t in (xs, w, y, x16, bias, scale, resid):
        assert t is None or (t.is_cuda and t.is_contiguous())
    assert w.dtype == torch.float32 and w.dim() == 3 and xs.dim() == y.dim() and xs.dim() in (2, 3)
    k, C_in, N = w.shape
    batch = xs.shape[0] if xs.dim() == 3 else 1
    if x16 is not None:
        assert x16.dtype == torch.float16 and (x is None or x16.shape == x.shape)
    if resid is not None:
        assert resid.dim() == y.dim() and (resid.dim() == 2 or resid.shape[0] == batch)
    seq = lambda t: t.shape[-2] * t.shape[-1] if t is not None and t.dim() == 3 else 0
    a = _lib.ConvArgs(
        x=_ptr(x).value, ldx=xs.shape[-1], T_in=xs.shape[-2] if T_in is None else T_in, x_row0=x_row0, x16=_ptr(x16).value,
        w=w.data_ptr(), k=k, dil=dil, C_in=C_in, N=N, bias=_ptr(bias).value, bias_mod=N if bias_mod is None else bias_mod,
        act=act, scale=_ptr(scale).value, resid=_ptr(resid).value, ldr=0 if resid is None else resid.shape[-1],
        y=y.data_ptr(), ldy=y.shape[-1], T_out=y.shape[-2] if T_out is None else T_out, t0=t0,
        batch=batch, x_bs=seq(xs), y_bs=seq(y), r_bs=seq(resid))
    dev = y.device.index or 0
    check(_lib.load().s2s_codec_contract(get_context(dev), C.byref(a), path, _stream_ptr(dev)), "s2s_codec_contract")


class LlamaEngine:
    """Llama-family LLM on one H100: wgmma prefill + persistent decode (greedy, or sampled per slot) with a per-session KV cache."""

    def __init__(self, geometry: Mapping[str, float], dtype: str = "bfloat16", max_sessions: int = 1,
                 max_positions: int = 2048, max_prefill: int = 512, device: int = 0, lane: int = 0, lanes: int = 1,
                 weight_dtype: Optional[str] = None):
        """weight_dtype: None = the projections are stored as `dtype`; "float8_e4m3" = weight-only FP8 with a power-of-two
        scale per row (bfloat16 compute only), quantised from the 16-bit weights when they are loaded.  Halves the bytes a
        decode step streams; the engine then computes, bit for bit, what a 16-bit engine bound to the dequantised weights does."""
        if weight_dtype is not None and weight_dtype not in _lib.WEIGHT_FORMAT_CODES:
            raise ValueError(f"weight_dtype {weight_dtype!r}: supported values are None and {sorted(_lib.WEIGHT_FORMAT_CODES)}")
        self.lib = _lib.load()
        self.device = device
        self.ctx = get_context(device, lane, lanes)
        self.geometry = dict(geometry)
        self.weight_dtype = weight_dtype
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
        if weight_dtype is not None:
            check(self.lib.s2s_llama_set_weight_format(self.handle, _lib.WEIGHT_FORMAT_CODES[weight_dtype]),
                  "s2s_llama_set_weight_format")

    def load_state_dict(self, weights: Mapping[str, "np.ndarray | torch.Tensor"]) -> None:
        _bind_all(self.lib.s2s_llama_bind_tensor, self.handle, weights, "llama")
        check(self.lib.s2s_llama_finalize(self.handle), "s2s_llama_finalize")

    def init_random(self, seed: int = 0) -> None:
        check(self.lib.s2s_llama_init_random(self.handle, seed), "s2s_llama_init_random")
        check(self.lib.s2s_llama_finalize(self.handle), "s2s_llama_finalize")

    def share(self, lane: int, lanes: int, max_sessions: Optional[int] = None, max_positions: Optional[int] = None,
              max_prefill: Optional[int] = None) -> "LlamaEngine":
        """A new engine on lane `lane` of `lanes` that reads this engine's weights (one copy per GPU) in their format: its
        own KV cache, workspaces and sampling state, sized by the given capacities (default: this engine's).  This engine
        must be loaded; neither can be reloaded while both live, and they may be closed in any order.  Bit for bit what an
        engine loaded with the same weights computes (include/s2s_b200.h shared weights)."""
        eng = object.__new__(LlamaEngine)
        eng.lib, eng.device, eng.geometry, eng.weight_dtype = self.lib, self.device, dict(self.geometry), self.weight_dtype
        eng.ctx = get_context(self.device, lane, lanes)
        cfg = LlamaConfig.from_buffer_copy(self.cfg)
        if max_sessions is not None:
            cfg.max_sessions = max_sessions
        if max_positions is not None:
            cfg.max_positions = min(max_positions, int(self.geometry.get("max_positions", max_positions)))
        if max_prefill is not None:
            cfg.max_prefill = max_prefill
        eng.cfg, eng.max_positions = cfg, cfg.max_positions
        eng.handle = C.c_void_p()
        check(self.lib.s2s_llama_create_shared(eng.ctx, self.handle, C.byref(cfg), C.byref(eng.handle)), "s2s_llama_create_shared")
        return eng

    def reset(self, slot: int = 0) -> None:
        check(self.lib.s2s_llama_session_reset(self.handle, slot), "s2s_llama_session_reset")

    def set_sampling(self, slot: int, *, do_sample: bool = False, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                     repetition_penalty: float = 1.0, min_new_tokens: int = 0, eos_ids: Sequence[int] = (), seed: int = 0) -> None:
        """Token choice of `slot` for the following prefill and decode calls (include/s2s_b200.h s2s_llama_set_sampling):
        repetition penalty and min_new_tokens apply to greedy slots too; temperature / top_k / top_p only with do_sample.
        The defaults are greedy argmax.  Set it before the response's prefill."""
        eos = [int(e) for e in eos_ids]
        if len(eos) > 8:
            raise ValueError(f"at most 8 EOS ids, got {len(eos)}")
        s = _lib.Sampling(int(bool(do_sample)), float(temperature), int(top_k), float(top_p), float(repetition_penalty),
                          int(min_new_tokens), len(eos), (C.c_int32 * 8)(*eos), int(seed) & 0xFFFFFFFFFFFFFFFF)
        check(self.lib.s2s_llama_set_sampling(self.handle, slot, C.byref(s)), "s2s_llama_set_sampling")

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

    def weight_format(self) -> int:
        """The S2S_* code of the streamed projections' storage (S2S_FP8_E4M3, or the compute dtype's code)."""
        return int(self.lib.s2s_llama_weight_format(self.handle))

    def max_decode_batch(self) -> int:
        """Sessions one decode launch can carry for this geometry (shared-memory budget of the kernel)."""
        return int(self.lib.s2s_llama_max_decode_batch(self.handle))

    def device_bytes(self) -> tuple[int, int]:
        """(weights, total): device bytes the engine holds for its weights (embedding, norms, the one tiled copy of the
        projections and lm_head) and in all (KV cache and workspaces included).  An engine made by share() reports the
        weights it reads, so total - weights is what it allocated itself."""
        return _device_bytes(self.lib.s2s_llama_device_bytes, self.handle, "s2s_llama_device_bytes")

    def set_trace(self, trace: Optional[torch.Tensor]) -> None:
        """trace: cuda int64 [2, capacity, 6] or None (profiling aid, see include/s2s_b200.h)."""
        cap = 0 if trace is None else trace.shape[1]
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
        self._create(cfg, dict(codec_geometry), None)

    def _create(self, cfg: Qwen3TTSConfig, codec_geometry: dict, source: Optional["Qwen3TTSEngine"]) -> None:
        self.cfg = cfg
        self.n_groups = cfg.n_groups
        self.codec_eos = cfg.codec_eos
        self.handle = C.c_void_p()
        if source is None:
            check(self.lib.s2s_qwen3tts_create(self.ctx, C.byref(cfg), C.byref(self.handle)), "s2s_qwen3tts_create")
        else:
            check(self.lib.s2s_qwen3tts_create_shared(self.ctx, source.handle, C.byref(cfg), C.byref(self.handle)),
                  "s2s_qwen3tts_create_shared")
        self.codec = CodecEngine(codec_geometry, device=self.device, _handle=C.c_void_p(self.lib.s2s_qwen3tts_codec(self.handle)),
                                 _owner=self)

    def share(self, lane: int, lanes: int, max_sessions: Optional[int] = None, max_positions: Optional[int] = None,
              max_text: Optional[int] = None, codec_max_frames: Optional[int] = None) -> "Qwen3TTSEngine":
        """A new engine on lane `lane` of `lanes` that reads this engine's weights -- talker, code predictor, codec and text
        side, one copy per GPU -- with its own sessions, history and workspaces, sized by the given capacities (default:
        this engine's; the codec batches min(16, max_sessions) sequences).  This engine must be loaded; neither can be
        reloaded while both live.  Bit for bit what an engine loaded with the same weights computes."""
        eng = object.__new__(Qwen3TTSEngine)
        eng.lib, eng.device, eng.geometry = self.lib, self.device, dict(self.geometry)
        eng.ctx = get_context(self.device, lane, lanes)
        cfg = Qwen3TTSConfig.from_buffer_copy(self.cfg)
        if max_sessions is not None:
            cfg.max_sessions = max_sessions
            cfg.codec.max_batch = min(16, max_sessions)
        if max_positions is not None:
            cfg.max_positions = max_positions
        if max_text is not None:
            cfg.max_text = max_text
        if codec_max_frames is not None:
            cfg.codec.max_frames = codec_max_frames
        eng._create(cfg, dict(self.codec.geometry), self)
        return eng

    def device_bytes(self) -> tuple[int, int]:
        """(weights, total) of talker, code predictor, codec and text side together, as LlamaEngine.device_bytes."""
        return _device_bytes(self.lib.s2s_qwen3tts_device_bytes, self.handle, "s2s_qwen3tts_device_bytes")

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

    def set_sampling(self, slot: int, *, talker: Optional[Mapping[str, Any]] = None, predictor: Optional[Mapping[str, Any]] = None,
                     seed: int = 0) -> None:
        """Token choice of the utterance just prefilled in `slot` (prefill resets it to greedy): `talker` / `predictor` take
        the keywords of LlamaEngine.set_sampling (do_sample, temperature, top_k, top_p, repetition_penalty), None = greedy.
        One seed serves both models (include/s2s_b200.h s2s_qwen3tts_set_sampling)."""
        def conv(d):
            if d is None:
                return None
            d = dict(d)
            unknown = set(d) - {"do_sample", "temperature", "top_k", "top_p", "repetition_penalty", "min_new_tokens"}
            if unknown:
                raise ValueError(f"unknown sampling options {sorted(unknown)}")
            return C.byref(_lib.Sampling(int(bool(d.get("do_sample", False))), float(d.get("temperature", 1.0)), int(d.get("top_k", 0)),
                                         float(d.get("top_p", 1.0)), float(d.get("repetition_penalty", 1.0)),
                                         int(d.get("min_new_tokens", 0)), 0, (C.c_int32 * 8)(), int(seed) & 0xFFFFFFFFFFFFFFFF))
        check(self.lib.s2s_qwen3tts_set_sampling(self.handle, slot, conv(talker), conv(predictor)), "s2s_qwen3tts_set_sampling")

    def decode_frames(self, slots: Sequence[int], n_frames: int, forced: Optional[torch.Tensor] = None, return_logits: bool = False):
        """-> codes int32 cuda [B, n_frames, n_groups] (asynchronous).  forced (int32 cuda, same shape): teacher-forced
        feedback for parity tests; the returned codes are still the models' own decisions.  return_logits: also the rows
        the codes were chosen from, (codes, talker f32 [n_frames, B, vocab], predictor f32 [n_frames, n_groups, B, cp_vocab]
        whose step 0 is unused)."""
        sl, B = _lib.i32_array(slots)
        dev = f"cuda:{self.device}"
        codes = torch.empty((B, n_frames, self.n_groups), dtype=torch.int32, device=dev)
        if forced is not None:
            forced = forced.to(torch.int32).contiguous()
            assert tuple(forced.shape) == (B, n_frames, self.n_groups)
        if not return_logits:
            check(self.lib.s2s_qwen3tts_decode_frames(self.handle, sl, B, n_frames, _ptr(codes), _ptr(forced), _stream_ptr(self.device)),
                  "s2s_qwen3tts_decode_frames")
            return codes
        tl = torch.empty((n_frames, B, self.cfg.vocab), dtype=torch.float32, device=dev)
        pl = torch.full((n_frames, self.n_groups, B, self.cfg.cp_vocab), float("nan"), dtype=torch.float32, device=dev)
        check(self.lib.s2s_qwen3tts_decode_frames_logits(self.handle, sl, B, n_frames, _ptr(codes), _ptr(forced), _ptr(tl), _ptr(pl),
                                                         _stream_ptr(self.device)), "s2s_qwen3tts_decode_frames_logits")
        return codes, tl, pl

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
