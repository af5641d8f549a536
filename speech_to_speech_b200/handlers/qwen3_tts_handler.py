"""B200Qwen3TTSHandler -- the reference's `qwen3` TTS slot with talker, code predictor, codec decoder and the per-chunk
post-processing on libs2s_b200.so.

Drop-in shape: when `speech_to_speech` is importable this is a subclass of the reference's own `Qwen3TTSHandler`
(speech_to_speech/TTS/qwen3_tts_handler.py) and inherits `setup()` with all its kwargs (:106-211),
`process` (:812-865), sentence coalescing (:751-810), `_estimate_max_new_tokens` (:615-658), `_stream` (:695-749) and the
session-voice logic unchanged; on a machine without the reference it subclasses the minimal mirror
(`host/mirror_tts.py`).  Three hooks change:

  _setup_faster(...)            builds `B200Qwen3TTS` (tts_model.py) where the reference imports faster_qwen3_tts and calls
                                `FasterQwen3TTS.from_pretrained` (:213-249).  `model_name="random:<geometry>"` gives a seeded
                                random-init model of a published geometry (no checkpoints exist offline).
  _prepare_audio_chunk(item)    keeps a device-resident chunk on the device (the reference copies to numpy, :682-693)
  _resample_to_pipeline_sr / _to_int16   one fused kernel on the device chunk (`s2s_tts_postproc`: polyphase 24 -> 16 kHz,
                                x32768, clip, int16 -- bit-exact vs scipy + numpy, tests/test_gpu_handlers.py); only int16
                                samples cross PCIe.

`gen_kwargs["max_sessions"] = N` (or setup kwarg `max_sessions`) shares ONE engine between the N pipeline units of the
process and merges the chunk requests of concurrently speaking sessions into one launch sequence (tts_model.py).
Arithmetic parity: pinned to the transformers cousin, UNPINNED vs faster-qwen3-tts (absent) -- DESIGN.md."""
from __future__ import annotations

import logging
from typing import Any, Optional

import numpy as np

from ..batcher import acquire_shared, assign_lane, release_shared
from ..tts_model import B200Qwen3TTS, DeviceAudio

logger = logging.getLogger(__name__)


def _base_class() -> Any:
    try:
        import importlib
        return importlib.import_module("speech_to_speech.TTS.qwen3_tts_handler").Qwen3TTSHandler
    except Exception:
        from ..host.mirror_tts import MirrorQwen3TTSHandler
        return MirrorQwen3TTSHandler


_Base = _base_class()


class B200Qwen3TTSHandler(_Base):  # type: ignore[misc, valid-type]
    _b200_post: Any = None
    _b200_shared_key: Optional[tuple] = None

    def setup(self, *args: Any, max_sessions: Optional[int] = None, lane: Optional[int] = None, lanes: Optional[int] = None,
              **kwargs: Any) -> None:
        gk = dict(kwargs.get("gen_kwargs") or {})
        self._b200_max_sessions = int(max_sessions if max_sessions is not None else gk.pop("max_sessions", 1))
        # SM partition: the handler instances of lane i share lane i's engine (engine.get_context); see INTEGRATION.md section 4
        self._b200_lanes = max(1, int(lanes if lanes is not None else gk.pop("lanes", 1)))
        lane = lane if lane is not None else gk.pop("lane", None)
        if lane is None:   # not pinned by the caller: units join the lanes round-robin in construction order
            lane = assign_lane(("qwen3tts", str(kwargs.get("model_name", "")), str(kwargs.get("device", "cuda"))), self._b200_lanes)
        self._b200_lane = int(lane) % self._b200_lanes
        self._b200_seed = int(gk.pop("seed", 0))
        kwargs["gen_kwargs"] = gk
        if "backend" in kwargs and kwargs["backend"] == "ggml":
            kwargs["backend"] = "torch"     # the ggml options of the reference slot do not apply; accept its default silently
        super().setup(*args, **kwargs)

    # ---- FasterQwen3TTS.from_pretrained replaced -----------------------------------------------------------------------
    def _setup_faster(self, model_name: str, dtype: Any, attn_implementation: str, backend: str) -> None:
        import torch
        device = str(getattr(self, "device", "cuda"))
        if device.startswith("cpu") or not torch.cuda.is_available():
            raise ValueError("B200Qwen3TTSHandler has no CPU path: qwen3_tts_device must be a CUDA device (sm_90a)")
        if dtype in ("auto", None):
            self.dtype = torch.bfloat16
        else:
            self.dtype = getattr(torch, dtype) if isinstance(dtype, str) else dtype
        dt = "float16" if self.dtype == torch.float16 else "bfloat16"
        dev = int(device.split(":")[1]) if ":" in device else 0
        n = max(1, self._b200_max_sessions)
        # the reference slot's `parity_mode` (qwen3_tts_arguments.py:99-101) selects the exact fp32 codec decoder
        prec = 0 if getattr(self, "parity_mode", False) else 1
        lane, lanes = getattr(self, "_b200_lane", 0), getattr(self, "_b200_lanes", 1)
        key = ("qwen3tts", model_name, dt, dev, n, prec, lane, lanes)

        def build() -> B200Qwen3TTS:
            if model_name.startswith("random:"):
                return B200Qwen3TTS.from_random(model_name.split(":", 1)[1], seed=self._b200_seed, dtype=dt, device=dev, max_sessions=n,
                                                codec_precision=prec, lane=lane, lanes=lanes)
            return B200Qwen3TTS.from_pretrained(model_name, device=device, dtype=self.dtype, attn_implementation=attn_implementation,
                                                backend=backend, max_sessions=n, codec_precision=prec, lane=lane, lanes=lanes)

        self.model = acquire_shared(key, build, lambda m: m.close())
        self._b200_shared_key = key
        self._b200_device = dev
        logger.info("Qwen3-TTS model loaded (libs2s_b200, %s, %d session slot%s)", dt, n, "" if n == 1 else "s")

    # ---- every GPU call of this handler's thread goes to its lane's stream ----------------------------------------------
    def _b200_lane_context(self):
        m = getattr(self, "model", None)
        if isinstance(m, B200Qwen3TTS):
            return m.lane_context()
        import contextlib
        return contextlib.nullcontext()

    def process(self, *args: Any, **kwargs: Any):
        with self._b200_lane_context():
            yield from super().process(*args, **kwargs)

    def warmup(self, *args: Any, **kwargs: Any):
        with self._b200_lane_context():
            return super().warmup(*args, **kwargs)

    # ---- per-chunk post-processing on the device --------------------------------------------------------------------------
    def _prepare_audio_chunk(self, item: Any):
        if isinstance(item, tuple) and isinstance(item[0], DeviceAudio):
            return item[0], item[1]
        return super()._prepare_audio_chunk(item)

    def _resample_to_pipeline_sr(self, audio: Any, sr: int):
        if isinstance(audio, DeviceAudio):
            if sr == 24000:
                if type(self)._b200_post is None:
                    from .qwen3_tts_postproc import TTSPostProcessor
                    type(self)._b200_post = TTSPostProcessor(getattr(self, "_b200_device", 0))
                return type(self)._b200_post.from_device(audio.tensor)        # int16 numpy @ 16 kHz
            audio = np.asarray(audio, dtype=np.float32)
        return super()._resample_to_pipeline_sr(audio, sr)

    def _to_int16(self, audio: np.ndarray) -> np.ndarray:
        if isinstance(audio, np.ndarray) and audio.dtype == np.int16:
            return audio
        return super()._to_int16(audio)

    def cleanup(self) -> None:
        key, self._b200_shared_key = self._b200_shared_key, None
        if key is not None:
            self.model = None
            release_shared(key)
        try:
            super().cleanup()
        except Exception:
            pass
