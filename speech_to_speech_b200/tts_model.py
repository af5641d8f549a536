"""B200Qwen3TTS -- the object the TTS handler slot holds in `self.model`, on libs2s_b200.so.

It stands where the reference puts `FasterQwen3TTS.from_pretrained(model_name, device=, dtype=, attn_implementation=,
backend=, ...)` (speech_to_speech/TTS/qwen3_tts_handler.py:213-249) and offers the calls the handler
makes on it: `warmup(prefill_len=100)` (:555-572), `generate_custom_voice_streaming(text, speaker, language, instruct,
chunk_size, max_new_tokens, non_streaming_mode)` (:946-978) yielding `(audio_f32, 24000, timing)` per chunk -- the tuple
contract the reference's tests pin with fakes (T/test_qwen3_tts_handler_backend.py:756-762) -- `get_supported_speakers()`
(:579-593) and `model.model.tts_model_type` (:574-580).

The arithmetic (talker, code predictor, codec decoder: csrc/qwen3tts.cu, csrc/codec_decode.cu) follows the published
cousin of Qwen3-TTS in transformers (Qwen3-Omni talker + Code2Wav) and is UNPINNED against faster-qwen3-tts, which is
absent everywhere (DESIGN.md).  Deliberate differences, all stated there: code selection is greedy unless asked otherwise
(upstream samples by default; `sampling=COUSIN_SAMPLING` or the per-call qwen-tts keywords `do_sample, temperature, top_k,
top_p, repetition_penalty, subtalker_dosample, subtalker_temperature, subtalker_top_k, subtalker_top_p` switch the
device sampler on), `language` / `instruct` are accepted and ignored (the cousin's prompt has no slot for them), voice
cloning and voice design need the upstream speaker encoder and raise.  No CPU fallback.

Concurrent sessions: one engine per (checkpoint, dtype, device) is shared by all handler instances of the process
(`max_sessions` slots); the chunk requests of concurrently speaking sessions are merged by the SessionBatcher into ONE
`s2s_qwen3tts_decode_frames` call -- 3 persistent launches per frame for up to 16 sessions."""
from __future__ import annotations

import contextlib
import json
import logging
import os
import random
import threading
import types
from time import perf_counter
from typing import Any, Callable, Iterator, Mapping, Optional, Sequence

import numpy as np

from .batcher import SessionBatcher

logger = logging.getLogger(__name__)

SAMPLE_RATE = 24000
LEFT_CONTEXT_FRAMES = 25     # Qwen3OmniMoeForConditionalGeneration.generate: chunked_decode(..., left_context_size=25)

# Published cousin geometry (Qwen3OmniMoeTalker{Text,CodePredictor}Config / Code2WavConfig defaults, dense talker MLP).
TTS_GEOMETRIES: dict[str, dict] = {
    "qwen3-tts-12hz": dict(
        talker=dict(d_model=1024, layers=20, heads=16, kv_heads=2, head_dim=128, ffn=2048, vocab=3072, rope_theta=1000000.0, rms_eps=1e-6),
        predictor=dict(d_model=1024, layers=5, heads=16, kv_heads=8, head_dim=128, ffn=3072, vocab=2048, rope_theta=1000000.0, rms_eps=1e-6),
        text_vocab=151936, text_hidden=2048, n_groups=16,
        codec_eos=2150, codec_nothink=2155, codec_think_bos=2156, codec_think_eos=2157, codec_pad=2148, codec_bos=2149,
        tts_bos=151672, tts_eos=151673, tts_pad=151671, im_start=151644, assistant=77091, newline=198),
    "micro": dict(
        talker=dict(d_model=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=3072, rope_theta=1000000.0, rms_eps=1e-6),
        predictor=dict(d_model=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=2048, rope_theta=1000000.0, rms_eps=1e-6),
        text_vocab=512, text_hidden=192, n_groups=16,
        codec_eos=2150, codec_nothink=2155, codec_think_bos=2156, codec_think_eos=2157, codec_pad=2148, codec_bos=2149,
        tts_bos=500, tts_eos=501, tts_pad=502, im_start=503, assistant=504, newline=505),
}
CODEC_GEOMETRIES: dict[str, dict] = {
    "qwen3-tts-12hz": dict(codebook_size=2048, hidden=1024, heads=16, kv_heads=16, inter=3072, layers=8, quantizers=16,
                           upsample_rates=(8, 5, 4, 3), upsampling_ratios=(2, 2), decoder_dim=1536, sliding_window=72,
                           rope_theta=10000.0, rms_eps=1e-5),
    "micro": dict(codebook_size=2048, hidden=64, heads=4, kv_heads=4, inter=96, layers=2, quantizers=16,
                  upsample_rates=(4, 3), upsampling_ratios=(2,), decoder_dim=48, sliding_window=6, rope_theta=10000.0, rms_eps=1e-5),
}
DEFAULT_SPEAKERS = {"aiden": 2301, "ethan": 2302, "chelsie": 2303}   # codec-vocabulary ids of the preset voices (random-init models)

# The sampling of the published cousin (transformers Qwen3-Omni): talker.generate(do_sample=True, top_k=50, top_p=1.0,
# temperature=0.9, repetition_penalty=1.05) and, for every frame, code_predictor.generate(do_sample=True, top_k=50,
# top_p=0.8) at the predictor's default temperature 1.0 (modeling_qwen3_omni_moe.py:3905-3909, 3251-3259).
COUSIN_SAMPLING = {
    "talker": dict(do_sample=True, temperature=0.9, top_k=50, top_p=1.0, repetition_penalty=1.05),
    "predictor": dict(do_sample=True, temperature=1.0, top_k=50, top_p=0.8),
}
# qwen-tts / faster-qwen3-tts generation keywords -> (model, Qwen3TTSEngine.set_sampling keyword)
SAMPLING_KEYWORDS = {
    "do_sample": ("talker", "do_sample"), "temperature": ("talker", "temperature"), "top_k": ("talker", "top_k"),
    "top_p": ("talker", "top_p"), "repetition_penalty": ("talker", "repetition_penalty"),
    "subtalker_dosample": ("predictor", "do_sample"), "subtalker_temperature": ("predictor", "temperature"),
    "subtalker_top_k": ("predictor", "top_k"), "subtalker_top_p": ("predictor", "top_p"),
}
# generation options the device sampler does not implement, with the value at which they do nothing
_UNSUPPORTED_SAMPLING = {"min_p": 0.0, "typical_p": 1.0, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0, "num_beams": 1,
                         "no_repeat_ngram_size": 0, "min_new_tokens": 0, "subtalker_min_p": 0.0, "subtalker_typical_p": 1.0,
                         "subtalker_repetition_penalty": 1.0}
_NEUTRAL = dict(do_sample=False, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0)


def resolve_sampling(base: Optional[Mapping] = None, **options: Any) -> dict:
    """The token choice of an utterance: `base` ({"talker": dict | None, "predictor": dict | None}, None = greedy) overlaid
    by the qwen-tts keywords in `options` (SAMPLING_KEYWORDS; None values are ignored).  A model's unset values come from
    its base dict, else from the neutral ones (T 1, top_k 0 = off, top_p 1, penalty 1).  -> {"talker": ..., "predictor":
    ...}, each the keywords of Qwen3TTSEngine.set_sampling or None when that model decodes greedily.  Raises ValueError for
    keywords the device sampler does not implement and for out-of-range values."""
    base = dict(base or {})
    unknown = set(base) - {"talker", "predictor"}
    if unknown:
        raise ValueError(f"sampling presets have 'talker' and 'predictor' entries only, got {sorted(unknown)}")
    over: dict = {"talker": {}, "predictor": {}}
    for k, v in options.items():
        if v is None:
            continue
        if k in _UNSUPPORTED_SAMPLING:
            off = _UNSUPPORTED_SAMPLING[k]
            if v != off and not (k == "num_beams" and int(v) <= 1):
                raise ValueError(f"`{k}` (={v}) is not supported by the Qwen3-TTS device sampler: it implements do_sample, temperature, "
                                 f"top_k, top_p, repetition_penalty (talker) and their subtalker_* counterparts (code predictor)")
            continue
        if k not in SAMPLING_KEYWORDS:
            raise ValueError(f"unknown Qwen3-TTS generation option `{k}`")
        model, key = SAMPLING_KEYWORDS[k]
        over[model][key] = v
    out: dict = {}
    for model in ("talker", "predictor"):
        b = base.get(model)
        if b is not None and set(b) - set(_NEUTRAL):
            raise ValueError(f"unknown {model} sampling options {sorted(set(b) - set(_NEUTRAL))}")
        if b is None and not over[model]:
            out[model] = None
            continue
        c = {**_NEUTRAL, **(b or {}), **over[model]}
        c = dict(do_sample=bool(c["do_sample"]), temperature=float(c["temperature"]), top_k=int(c["top_k"]), top_p=float(c["top_p"]),
                 repetition_penalty=float(c["repetition_penalty"]))
        if c["do_sample"] and not c["temperature"] > 0.0:
            raise ValueError(f"{model} `temperature` (={c['temperature']}) has to be a strictly positive float when sampling")
        if c["do_sample"] and not 0.0 < c["top_p"] <= 1.0:
            raise ValueError(f"{model} `top_p` has to be a float in (0, 1], but is {c['top_p']}")
        if c["top_k"] < 0:
            raise ValueError(f"{model} `top_k` has to be >= 0, but is {c['top_k']}")
        if not c["repetition_penalty"] > 0.0:
            raise ValueError(f"{model} `repetition_penalty` has to be a strictly positive float, but is {c['repetition_penalty']}")
        if model == "predictor" and c["repetition_penalty"] != 1.0:
            raise ValueError("the code predictor has no repetition penalty")
        if not c["do_sample"]:
            c.update(temperature=1.0, top_k=0, top_p=1.0)
        out[model] = c if (c["do_sample"] or c["repetition_penalty"] != 1.0) else None
    return out


def is_greedy(sampling: Mapping) -> bool:
    return sampling.get("talker") is None and sampling.get("predictor") is None


class DeviceAudio:
    """A chunk of 24 kHz fp32 audio that is still on the GPU.  `np.asarray(chunk)` copies it to the host, so a consumer
    that only knows the `(np.float32[n], sr, timing)` contract (the reference's `_prepare_audio_chunk`, :682-693) works
    unchanged; the GPU handler keeps it on the device and runs resample + int16 there."""

    __slots__ = ("tensor",)

    def __init__(self, tensor: Any):
        self.tensor = tensor

    @property
    def size(self) -> int:
        return int(self.tensor.numel())

    def __len__(self) -> int:
        return self.size

    def __array__(self, dtype=None, copy=None):
        a = self.tensor.detach().cpu().numpy()
        return a.astype(dtype) if dtype is not None and a.dtype != dtype else a


def byte_tokenizer(text_vocab: int, reserved: int = 16) -> Callable[[str], list]:
    """Stand-in tokenizer for random-init models (no tokenizer files exist offline, SURVEY.md 0.7): UTF-8 bytes folded into
    the text vocabulary below the special ids.  Real checkpoints bring their own tokenizer (from_pretrained)."""
    lim = max(1, int(text_vocab) - reserved)

    def tok(text: str) -> list:
        b = text.encode("utf-8") or b" "
        return [int(x) % lim for x in b]
    return tok


class B200Qwen3TTS:
    def __init__(self, engine: Any, tokenize: Callable[[str], Sequence[int]], speakers: Mapping[str, int], max_sessions: int = 1,
                 batch_wait_s: float = 0.012, tts_model_type: str = "custom_voice", lane: int = 0, lanes: int = 1,
                 batch_gap_s: Optional[float] = 0.003, sampling: Optional[Mapping] = None, sampling_seed: Optional[int] = None):
        # batch_gap_s: a session needs a few ms of host work between two chunk requests (resample + int16 + D2H of the chunk it
        # just received); the gap must cover it, or the sessions of the launch that just ended miss the next one and two groups
        # alternate in half-full launches (measured: mean batch 7.8 of 16 with a 0.6 ms gap)
        self.engine = engine
        self.lane, self.lanes = int(lane), int(lanes)
        self.max_sessions = int(max_sessions)
        self._options = dict(batch_wait_s=batch_wait_s, tts_model_type=tts_model_type, batch_gap_s=batch_gap_s,
                             sampling=sampling, sampling_seed=sampling_seed)
        self.tokenize = tokenize
        # default token choice of generate_custom_voice_streaming (None = greedy; COUSIN_SAMPLING = the cousin's) and one
        # 64-bit Philox seed per sampled utterance, drawn from a generator seeded by sampling_seed (OS entropy when None)
        self.sampling = resolve_sampling(sampling)
        self._seed_rng = random.Random(int(sampling_seed) if sampling_seed is not None else int.from_bytes(os.urandom(8), "little"))
        self.speakers = {str(k).lower(): int(v) for k, v in speakers.items()}
        self.sample_rate = SAMPLE_RATE
        self._lock = threading.Lock()           # one thread at a time talks to the engine handle
        self._free = list(range(max_sessions))
        self._slot_cv = threading.Condition()
        mb = max(1, min(int(engine.max_batch()), max_sessions))
        self.batcher = SessionBatcher(self._run_frames, mb, batch_wait_s, "s2s-tts-batcher",
                                      thread_context=self.lane_context, idle_gap_s=batch_gap_s) if max_sessions > 1 else None
        # what the reference handler inspects: model.model.tts_model_type, get_supported_speakers (qwen3_tts_handler.py:574-593)
        inner = types.SimpleNamespace(tts_model_type=tts_model_type, get_supported_speakers=self.get_supported_speakers)
        self.model = types.SimpleNamespace(model=inner, get_supported_speakers=self.get_supported_speakers)

    def lane_context(self):
        """The lane's CUDA stream as the calling thread's current stream (no-op for one lane): engine.lane_context."""
        if self.lanes <= 1:
            return contextlib.nullcontext()
        from . import engine as E
        return E.lane_context(self.engine.device, self.lane, self.lanes)

    # ---- construction -------------------------------------------------------------------------------------------------
    @classmethod
    def from_random(cls, geometry: "str | Mapping" = "qwen3-tts-12hz", codec_geometry: "str | Mapping | None" = None, seed: int = 0,
                    dtype: str = "bfloat16", device: int = 0, max_sessions: int = 1, max_positions: int = 2048, max_text: int = 512,
                    tokenize: Optional[Callable] = None, speakers: Optional[Mapping[str, int]] = None, codec_precision: int = 1,
                    lane: int = 0, lanes: int = 1, **kw: Any) -> "B200Qwen3TTS":
        from . import engine as E
        g = TTS_GEOMETRIES[geometry] if isinstance(geometry, str) else dict(geometry)
        cg = codec_geometry if codec_geometry is not None else (geometry if isinstance(geometry, str) else "qwen3-tts-12hz")
        cg = CODEC_GEOMETRIES[cg] if isinstance(cg, str) else dict(cg)
        eng = E.Qwen3TTSEngine(g, cg, dtype=dtype, max_sessions=max_sessions, max_positions=max_positions, max_text=max_text,
                               codec_max_frames=LEFT_CONTEXT_FRAMES + 16, device=device, codec_precision=codec_precision,
                               lane=lane, lanes=lanes)
        eng.init_random(seed)
        return cls(eng, tokenize or byte_tokenizer(g["text_vocab"]), speakers or DEFAULT_SPEAKERS, max_sessions=max_sessions,
                   lane=lane, lanes=lanes, **kw)

    @classmethod
    def from_pretrained(cls, model_name: str, device: Any = "cuda", dtype: Any = None, attn_implementation: str = "eager",
                        backend: str = "torch", max_sessions: int = 1, codec_precision: int = 1, lane: int = 0, lanes: int = 1,
                        sampling: Optional[Mapping] = None, sampling_seed: Optional[int] = None, **_ignored: Any) -> "B200Qwen3TTS":
        """Load a checkpoint DIRECTORY in the cousin's layout: `config.json` with {"talker": ..., "code2wav": ..., "speaker_id":
        ...}, `model.safetensors` with the talker state dict (+ "text_embedding.weight", "code2wav.*") and tokenizer files.
        Hub ids cannot be resolved offline, and the real Qwen3-TTS checkpoint layout is unverified (upstream absent): both
        raise an actionable error instead of guessing."""
        if str(device).startswith("cpu"):
            raise ValueError("speech_to_speech_b200 has no CPU path: qwen3_tts_device must be a CUDA device")
        if not os.path.isdir(model_name) or not os.path.exists(os.path.join(model_name, "config.json")):
            raise OSError(
                f"B200Qwen3TTS.from_pretrained: '{model_name}' is not a local checkpoint directory (config.json + model.safetensors "
                "in the Qwen3-Omni talker / code2wav tensor layout).  Use model_name='random:qwen3-tts-12hz' for a seeded "
                "random-init model of the published geometry.")
        import torch
        from safetensors.torch import load_file
        from transformers import AutoTokenizer
        from . import engine as E
        with open(os.path.join(model_name, "config.json")) as f:
            cfg = json.load(f)
        g, cg = cfg["talker"], cfg["code2wav"]
        dev = int(str(device).split(":")[1]) if ":" in str(device) else 0
        dt = "float16" if dtype in (torch.float16, "float16") else "bfloat16"
        eng = E.Qwen3TTSEngine(g, cg, dtype=dt, max_sessions=max_sessions, codec_max_frames=LEFT_CONTEXT_FRAMES + 16, device=dev,
                               codec_precision=codec_precision, lane=lane, lanes=lanes)
        sd = load_file(os.path.join(model_name, "model.safetensors"))
        eng.load_state_dict({k: v for k, v in sd.items() if not k.startswith("code2wav.")},
                            {k[len("code2wav."):]: v for k, v in sd.items() if k.startswith("code2wav.")})
        tok = AutoTokenizer.from_pretrained(model_name)
        return cls(eng, lambda text: tok.encode(text, add_special_tokens=False), cfg.get("speaker_id") or DEFAULT_SPEAKERS,
                   max_sessions=max_sessions, lane=lane, lanes=lanes, sampling=sampling, sampling_seed=sampling_seed)

    def share(self, lane: int, lanes: int, max_sessions: Optional[int] = None) -> "B200Qwen3TTS":
        """The same model on lane `lane` of `lanes` (default: as many session slots as this one) with the same speakers,
        tokenizer and options, on an engine that reads this model's weights (Qwen3TTSEngine.share): one weight copy per GPU."""
        n = int(max_sessions if max_sessions is not None else self.max_sessions)
        eng = self.engine.share(lane, lanes, max_sessions=n)
        return type(self)(eng, self.tokenize, self.speakers, max_sessions=n, lane=lane, lanes=lanes, **self._options)

    # ---- the calls the handler makes ------------------------------------------------------------------------------------
    def get_supported_speakers(self) -> list:
        return sorted(self.speakers)

    def warmup(self, prefill_len: int = 100) -> None:
        """One short utterance through every kernel (cudaFuncSetAttribute, cooperative-launch cold start, codec buffers)."""
        n = max(1, min(int(prefill_len), self.engine.cfg.max_text))
        for _ in self._generate([1] * n, next(iter(self.speakers.values())), chunk_size=2, max_new_tokens=2):
            pass

    def generate_custom_voice_streaming(self, text: str, speaker: str, language: Optional[str] = None, instruct: Optional[str] = None,
                                        chunk_size: int = 8, max_new_tokens: int = 1536, non_streaming_mode: Optional[bool] = True,
                                        sampling_seed: Optional[int] = None, **generation: Any) -> Iterator[tuple]:
        """generation: the qwen-tts sampling keywords (resolve_sampling), overlaid on the model's default `sampling`.
        sampling_seed: the utterance's 64-bit Philox seed (default: the next one of the model's seed generator)."""
        sampling = resolve_sampling(self.sampling, **generation)
        sid = self.speakers.get(str(speaker).lower())
        if sid is None:
            raise ValueError(f"unknown Qwen3-TTS speaker {speaker!r}; supported: {self.get_supported_speakers()}")
        if instruct:
            logger.debug("B200Qwen3TTS: `instruct` is accepted but has no slot in the built prompt layout; ignored")
        ids = list(self.tokenize(text or "Hello."))
        yield from self._generate(ids, sid, chunk_size=chunk_size, max_new_tokens=max_new_tokens, sampling=sampling, seed=sampling_seed)

    def generate_voice_clone_streaming(self, *a: Any, **k: Any) -> Iterator[tuple]:
        raise NotImplementedError("voice cloning needs the upstream speaker encoder (faster-qwen3-tts), which is absent; "
                                  "use a CustomVoice speaker")

    def generate_voice_design_streaming(self, *a: Any, **k: Any) -> Iterator[tuple]:
        raise NotImplementedError("voice design needs the upstream instruct-conditioned talker, which is absent; use a CustomVoice speaker")

    # ---- generation -----------------------------------------------------------------------------------------------------
    def _acquire_slot(self) -> int:
        with self._slot_cv:
            while not self._free:
                self._slot_cv.wait(timeout=0.05)
            return self._free.pop(0)

    def _release_slot(self, slot: int) -> None:
        with self._slot_cv:
            self._free.append(slot)
            self._slot_cv.notify()

    def _run_frames(self, key: Any, slots: list) -> list:
        """SessionBatcher callback: `key` = frames per chunk.  ONE decode_frames call for all the sessions that asked, then the
        codec decoder once per group of sessions whose chunks have the same shape (same valid frames, same history).
        -> per session (valid frames, finished, waveform on the device or None)."""
        eng, n = self.engine, int(key)
        with self._lock:
            before = [eng.frames(s) for s in slots]
            host = eng.decode_frames(slots, n).cpu().numpy()   # B x n x 16 int32: the only per-chunk D2H besides the audio
            groups: dict = {}
            out: list = [None] * len(slots)
            for i, s in enumerate(slots):
                eos = np.nonzero(host[i][:, 0] == eng.codec_eos)[0]
                valid = int(eos[0]) if len(eos) else n
                if valid < n:
                    eng.set_frames(s, before[i] + valid)
                out[i] = (valid, valid < n, None)
                if valid > 0:
                    groups.setdefault((valid, eng.history_context(s, valid, LEFT_CONTEXT_FRAMES)), []).append(i)
            for (valid, _ctx), idx in groups.items():
                wavs = eng.decode_audio_batch([slots[i] for i in idx], valid, LEFT_CONTEXT_FRAMES)
                for i, w in zip(idx, wavs):
                    out[i] = (valid, out[i][1], w)
        return out

    def _generate(self, text_ids: Sequence[int], speaker_id: int, chunk_size: int, max_new_tokens: int,
                  sampling: Optional[Mapping] = None, seed: Optional[int] = None) -> Iterator[tuple]:
        eng = self.engine
        chunk = max(1, int(chunk_size))
        budget = max(1, min(int(max_new_tokens), eng.cfg.max_positions - 16))
        ids = list(text_ids)[: eng.cfg.max_text] or [0]
        slot = self._acquire_slot()
        t0 = perf_counter()
        pending = None
        try:
            with self._lock:
                eng.prefill(slot, ids, speaker_id)
                if sampling is not None and not is_greedy(sampling):   # prefill left the slot greedy
                    if seed is None:
                        seed = self._seed_rng.getrandbits(64)
                    eng.set_sampling(slot, talker=sampling["talker"], predictor=sampling["predictor"], seed=seed)
            done = 0
            if self.batcher is None:
                while done < budget:
                    valid, finished, wav = self._run_frames(min(chunk, budget - done), [slot])[0]
                    done += valid
                    if wav is not None and wav.numel() > 0:
                        yield DeviceAudio(wav), SAMPLE_RATE, {"frames": done, "elapsed_s": perf_counter() - t0}
                    if finished:
                        break
                return
            # Shared engine: the request for chunk k + 1 leaves BEFORE chunk k is handed to the consumer.  The consumer's work on a
            # chunk (wait for its codec kernels, resample, int16, D2H: ~10 ms) would otherwise delay this session's next request
            # past the batch window, and two groups of sessions lock into alternating half-full launches (measured: mean batch
            # 7.8 of 16); with the request already queued, every session of the launch that just ended rides the next one, and the
            # engine computes chunk k + 1 while the handler threads post-process chunk k.
            pending = self.batcher.submit(min(chunk, budget), slot)
            while pending is not None:
                valid, finished, wav = pending.result()
                pending = None
                done += valid
                if not finished and done < budget:
                    pending = self.batcher.submit(min(chunk, budget - done), slot)
                if wav is not None and wav.numel() > 0:
                    yield DeviceAudio(wav), SAMPLE_RATE, {"frames": done, "elapsed_s": perf_counter() - t0}
        finally:
            if pending is not None and not pending.cancel():     # consumer stopped early: the slot is in use until the launch ends
                try:
                    pending.result()
                except Exception:  # noqa: BLE001
                    pass
            self._release_slot(slot)

    def close(self) -> None:
        if self.batcher is not None:
            self.batcher.close()
        self.engine.close()
