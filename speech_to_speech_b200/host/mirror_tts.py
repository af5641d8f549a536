"""Minimal mirror of the reference's Qwen3-TTS handler slot for machines without the upstream speech_to_speech package.

When `speech_to_speech` is importable the B200 handler subclasses the reference's own `Qwen3TTSHandler` and inherits all
of this unchanged; this mirror restates only what the hot path needs, with the same method names, argument meaning and
error behaviour (reference: S/TTS/qwen3_tts_handler.py):
  setup(should_listen, model_name, device, dtype, ..., blocksize, gen_kwargs, cancel_scope, speculative_turns)   :106-211
  process(TTSInput | EndOfResponse) -> int16[blocksize] blocks, AUDIO_RESPONSE_DONE for EndOfResponse             :812-865
  _process_custom_voice(text) -> model.generate_custom_voice_streaming(...) through _stream                     :946-978
  _estimate_max_new_tokens(text): codec-token budget (12.5 frames/s x 1.35, chunk aligned, floor 360, capped)   :615-658
  _stream(gen, label): cancel poll, resample to 16 kHz, int16, leading-silence trim with 40 ms preroll,
                       fixed-size blocks, zero-padded tail                                                      :695-749
Apple-MLX, ggml options, voice-clone caches and session voice overrides are outside the built path and not mirrored;
queued-sentence coalescing (:751-810) needs the reference's message types and is the identity here."""
from __future__ import annotations

import logging
import math
import re
import unicodedata
from time import perf_counter
from typing import Any, Iterator, Optional

import numpy as np

from . import mirror as mr

logger = logging.getLogger(__name__)

DEFAULT_MODEL = "Qwen/Qwen3-TTS-12Hz-1.7B-CustomVoice"
PIPELINE_SR = 16000
FRAMES_PER_SECOND = 12.5
_CJK = re.compile(r"[぀-ヿ㐀-䶿一-鿿가-힯豈-﫿\U00020000-\U0002fa1f]")


class MirrorQwen3TTSHandler(mr.BaseHandler):
    def setup(self, should_listen: Any = None, model_name: str = DEFAULT_MODEL, device: str = "cuda", dtype: Any = "auto",
              attn_implementation: str = "eager", backend: str = "torch", language: str = "auto", speaker: Optional[str] = "Aiden",
              instruct: Optional[str] = None, non_streaming_mode: Optional[bool] = True, streaming_chunk_size: Optional[int] = None,
              max_new_tokens: int = 1536, blocksize: int = 512, gen_kwargs: Optional[dict] = None, cancel_scope: Any = None,
              speculative_turns: Any = None, **other: Any) -> None:
        self.cancel_scope, self.speculative_turns, self.should_listen = cancel_scope, speculative_turns, should_listen
        self.requested_device = self.device = device
        self.model_name, self.language, self.speaker, self.instruct = model_name, (language or "auto"), speaker, instruct
        self.non_streaming_mode, self.max_new_tokens, self.blocksize = non_streaming_mode, max_new_tokens, blocksize
        self.gen_kwargs = gen_kwargs or {}
        self.backend = "faster_qwen3_tts"
        self.faster_backend = backend
        self.parity_mode = bool(other.get("parity_mode", False))
        self.streaming_chunk_size = max(1, int(streaming_chunk_size)) if streaming_chunk_size else 8
        self._setup_faster(model_name=model_name, dtype=dtype, attn_implementation=attn_implementation, backend=backend)
        self._initial_speaker = self.speaker
        self.warmup()

    def _setup_faster(self, model_name: str, dtype: Any, attn_implementation: str, backend: str) -> None:
        raise NotImplementedError

    def warmup(self) -> None:
        try:
            self.model.warmup(prefill_len=100)
        except Exception as e:  # the reference logs and carries on (:561-565)
            logger.warning("Qwen3-TTS backend warmup failed: %s", e)
        try:
            for _ in self._process_custom_voice("Hello, this is a warmup."):
                pass
        except Exception as e:
            logger.warning("Warmup generation failed: %s", e)

    def _model_type(self) -> str:
        inner = getattr(getattr(self.model, "model", None), "model", None)
        return getattr(inner, "tts_model_type", None) or "custom_voice"

    def _resolve_speaker(self) -> Optional[str]:
        if self.speaker:
            return self.speaker
        get = getattr(self.model, "get_supported_speakers", None)
        names = list(get() or []) if callable(get) else []
        return names[0] if names else None

    def _to_int16(self, audio: np.ndarray) -> np.ndarray:
        return np.clip(audio * 32768, -32768, 32767).astype(np.int16)

    def _resample_to_pipeline_sr(self, audio: np.ndarray, sr: int) -> np.ndarray:
        if sr == PIPELINE_SR:
            return audio
        from scipy.signal import resample_poly
        g = math.gcd(PIPELINE_SR, int(sr))
        return resample_poly(audio, up=PIPELINE_SR // g, down=int(sr) // g)

    def _prepare_audio_chunk(self, item: Any):
        if isinstance(item, tuple):
            chunk, sr, _timing = item
            return np.asarray(chunk, dtype=np.float32), sr
        audio = getattr(item, "audio", None)
        if audio is None:
            return None, None
        return np.asarray(audio, dtype=np.float32).squeeze(), getattr(item, "sample_rate", None) or PIPELINE_SR

    def _estimate_max_new_tokens(self, text: Optional[str]) -> int:
        text = (text or "").strip()
        chunk = max(1, int(getattr(self, "streaming_chunk_size", 1)))
        cap = max(1, int(getattr(self, "max_new_tokens", 1536)))
        if not text:
            return min(cap, 360)
        words = len(re.findall(r"\w+", text, flags=re.UNICODE))
        chars = len(re.sub(r"\s+", "", text))
        cjk = len(_CJK.findall(text))
        speech_s = max(words / 2.6 if words else 0.0, chars / 14.0 if chars else 0.0, cjk / 5.5 if cjk else 0.0)
        pauses_s = 0.5 * sum(unicodedata.category(ch).startswith("P") for ch in text)
        tokens = math.ceil((speech_s + pauses_s + 1.0) * FRAMES_PER_SECOND * 1.35)
        aligned = max(chunk, math.ceil(tokens / chunk) * chunk)
        return min(cap, max(360, aligned))

    def _stream(self, gen: Any, label: str) -> Iterator[np.ndarray]:
        scope = self.cancel_scope
        my_gen = scope.generation if scope else None
        t0 = perf_counter()
        emitted, first, speaking = 0, True, False
        carry = np.zeros((0,), np.int16)
        bs = self.blocksize
        for item in gen:
            if my_gen is not None and scope.is_stale(my_gen):
                logger.info("TTS generation cancelled (interruption)")
                return
            chunk, sr = self._prepare_audio_chunk(item)
            if chunk is None or sr is None or chunk.size == 0:
                continue
            if first:
                logger.info("Qwen3-TTS TTFA: %.2fs (%s)", perf_counter() - t0, label)
                first = False
            pcm = self._to_int16(self._resample_to_pipeline_sr(chunk, sr))
            if not speaking:   # skip the silent ramp-up but keep 40 ms of preroll
                loud = np.abs(pcm) > int(32768 * 0.01)
                if not loud.any():
                    continue
                pcm = pcm[max(0, int(np.argmax(loud)) - int(PIPELINE_SR * 0.040)):]
                speaking = True
            pcm = np.concatenate([carry, pcm])
            whole = (len(pcm) // bs) * bs
            for i in range(0, whole, bs):
                yield pcm[i:i + bs]
                emitted += bs
            carry = pcm[whole:]
        if len(carry):
            yield np.pad(carry, (0, bs - len(carry)))
            emitted += len(carry)
        dt = perf_counter() - t0
        logger.info("Qwen3-TTS generated %.2fs audio in %.2fs (RTF: %.2f, %s)", emitted / PIPELINE_SR, dt,
                    (emitted / PIPELINE_SR) / dt if dt > 0 else 0.0, label)

    def _process_custom_voice(self, text: str) -> Iterator[np.ndarray]:
        budget = self._estimate_max_new_tokens(text)
        speaker = self._resolve_speaker()
        if not speaker:
            raise ValueError("CustomVoice generation requires a speaker. Set qwen3_tts_speaker.")
        yield from self._stream(
            self.model.generate_custom_voice_streaming(text=text, speaker=speaker, language=self.language, instruct=self.instruct,
                                                       chunk_size=self.streaming_chunk_size, max_new_tokens=budget,
                                                       non_streaming_mode=self.non_streaming_mode),
            label="custom_voice")

    def process(self, tts_input: Any) -> Iterator[Any]:
        if isinstance(tts_input, mr.EndOfResponse):
            yield mr.AUDIO_RESPONSE_DONE
            return
        text = (getattr(tts_input, "text", "") or "").strip() or "Hello."
        try:
            first = True
            for block in self._process_custom_voice(text):
                if first:
                    stopped = getattr(tts_input, "speech_stopped_at_s", None)
                    if stopped is not None and perf_counter() - stopped >= 0:
                        logger.info("Last speech detected to first speech out: %.3fs (turn=%s rev=%s)", perf_counter() - stopped,
                                    getattr(tts_input, "turn_id", None), getattr(tts_input, "turn_revision", None))
                    first = False
                yield block
        except Exception as e:   # the reference catches generation errors inside process (:864-865)
            logger.error("Error during Qwen3-TTS generation: %s", e, exc_info=True)

    def on_session_end(self) -> None:
        self.speaker = self._initial_speaker

    def cleanup(self) -> None:
        try:
            del self.model
        except Exception as e:
            logger.warning("Cleanup error: %s", e)
