"""B200WhisperSTTHandler -- the reference's WhisperSTTHandler slot with the forward pass on libs2s_b200.so.

Mirrors speech_to_speech/STT/whisper_stt_handler.py: same `setup()` kwargs (:53-61), same
`process(VADAudio) -> Iterator[PartialTranscription | Transcription]` contract (:225-282) including the
language bookkeeping ("-auto" suffix, sticky last_language restricted to SUPPORTED_LANGUAGES, progressive mode).
What changes is what the handler calls: `processor(...)` + `model.generate(...)` become ONE call into the C ABI
(`s2s_whisper_transcribe`: H2D PCM, log-mel, encoder, greedy decode, D2H ids); only the BPE detokenisation
(`processor.batch_decode`, CPU, :259) stays in Python.  No CPU fallback: a non-CUDA `device` raises.

`max_batch > 1` (set it to the number of pipeline units, `--num_pipelines`) makes every handler instance of the
process with the same (model, dtype, device) share ONE engine -- one copy of the weights -- behind a SessionBatcher
(`batcher.py`): utterances of concurrent sessions that arrive within `batch_wait_ms` are transcribed by one launch."""
from __future__ import annotations

import contextlib
import logging
import re
import threading
from typing import Any, Iterator, Optional

import numpy as np

from ..host import resolve
from ..batcher import SessionBatcher, acquire_shared, assign_lane, release_shared

logger = logging.getLogger(__name__)
_api = resolve()

SUPPORTED_LANGUAGES = ["en", "fr", "es", "zh", "ja", "ko", "hi", "de", "pt", "pl", "it", "nl"]
DEFAULT_LANGUAGE = "en"
_LANGUAGE_TOKEN_RE = re.compile(r"^<\|([a-z]{2,3})\|>$")


class TokenTable:
    """Special-token ids the decoder prompt and logit processors need; from a checkpoint's generation_config
    (transformers generation_whisper.py:1455-1608 `_retrieve_init_tokens`) or synthetic for random-init models."""

    def __init__(self, sot: int, eos: int, transcribe: int, translate: int, no_timestamps: int, lang_to_id: dict[str, int],
                 suppress: list[int], begin_suppress: list[int]):
        self.sot, self.eos, self.transcribe, self.translate, self.no_timestamps = sot, eos, transcribe, translate, no_timestamps
        self.lang_to_id = dict(lang_to_id)
        self.id_to_lang = {v: k for k, v in lang_to_id.items()}
        self.suppress, self.begin_suppress = list(suppress), list(begin_suppress)

    @classmethod
    def from_generation_config(cls, gc: Any) -> "TokenTable":
        lang = {}
        for tok, idx in (getattr(gc, "lang_to_id", None) or {}).items():
            m = _LANGUAGE_TOKEN_RE.match(tok)
            if m:
                lang[m.group(1)] = int(idx)
        task = getattr(gc, "task_to_id", None) or {}
        eos = gc.eos_token_id if isinstance(gc.eos_token_id, int) else gc.eos_token_id[0]
        return cls(int(gc.decoder_start_token_id), int(eos), int(task.get("transcribe", 50359)), int(task.get("translate", 50358)),
                   int(getattr(gc, "no_timestamps_token_id", 50363)), lang, list(getattr(gc, "suppress_tokens", None) or []),
                   list(getattr(gc, "begin_suppress_tokens", None) or []))

    @classmethod
    def synthetic(cls, vocab: int) -> "TokenTable":
        if vocab >= 51865:  # multilingual Whisper layout
            langs = {c: 50259 + i for i, c in enumerate(["en", "zh", "de", "es", "ru", "ko", "fr", "ja", "pt", "tr", "pl", "ca", "nl", "ar", "sv", "it", "id", "hi"])}
            return cls(50258, 50257, 50359, 50358, 50363, langs, [1, 2, 7, 8, 9, 10, 14, 25, 50258, 50358, 50359, 50360, 50361, 50362], [220, 50257])
        base = vocab - 96
        langs = {c: base + 1 + i for i, c in enumerate(["en", "zh", "de", "es", "fr", "ja"])}
        return cls(base, vocab - 1, base + 10, base + 11, base + 12, langs, [1, 2, 7, base, base + 10, base + 11], [220, vocab - 1])


class _EngineBundle:
    """An engine with what is needed to drive it; private to one handler or shared through the batcher."""

    def __init__(self, E: Any, engine: Any, tokens: "TokenTable", decode_text: Any, max_batch: int, batch_wait_s: float,
                 lane: int = 0, lanes: int = 1, batch_gap_s: Optional[float] = None):
        self.E, self.engine, self.tokens, self.decode_text = E, engine, tokens, decode_text
        self.lane, self.lanes = lane, lanes
        self.lock = threading.Lock()  # the engine handle is used by one thread at a time (INTEGRATION.md)
        self.batcher = SessionBatcher(self._run_batch, max_batch, batch_wait_s, "s2s-stt-batcher",
                                      thread_context=self.lane_context, idle_gap_s=batch_gap_s) if max_batch > 1 else None

    def lane_context(self):
        """The lane's CUDA stream as the calling thread's current stream (engine.lane_context; a no-op for one lane)."""
        if self.lanes <= 1:
            return contextlib.nullcontext()
        return self.E.lane_context(self.engine.device, self.lane, self.lanes)

    @staticmethod
    def _key(o: Any) -> tuple:
        return (tuple(o.prefix), int(o.eos_id), int(o.max_new_tokens), tuple(o.suppress), tuple(o.begin_suppress))

    def _run_batch(self, key: tuple, audios: list) -> list:
        if key and key[0] == "auto":
            return self._run_auto_batch(key, audios)
        opts = self.E.WhisperDecodeOptions(prefix=list(key[0]), eos_id=key[1], max_new_tokens=key[2], suppress=list(key[3]),
                                           begin_suppress=list(key[4]))
        with self.lock:
            return self.engine.transcribe(audios, opts)

    def transcribe(self, audio: np.ndarray, opts: Any) -> list[int]:
        if self.batcher is not None:
            return self.batcher.call(self._key(opts), audio)
        with self.lock, self.lane_context():
            return self.engine.transcribe([audio], opts)[0]

    def detect_language(self, audio: np.ndarray, sot: int, lang_ids: list[int]) -> int:
        with self.lock, self.lane_context():
            return int(self.engine.detect_language_host(audio, sot, lang_ids))

    # auto-language mode: detection and decode share one encoder pass; concurrent sessions still share the launches.
    # spec = (sot, language ids, fallback language id, prompt tail after the language token, eos, max_new, suppress,
    # begin_suppress): hashable and identical for handlers with the same options, so their requests merge in the batcher.
    def _run_auto_batch(self, key: tuple, audios: list) -> list:
        _, sot, lang_ids, fallback, tail, eos, max_new, sup, beg = key
        known = set(lang_ids)

        def make_opts(langs: list) -> Any:
            rows = [[sot, (t if t in known else fallback)] + list(tail) for t in langs]
            return self.E.WhisperDecodeOptions(prefix=rows[0], eos_id=eos, max_new_tokens=max_new, suppress=list(sup),
                                               begin_suppress=list(beg), prefix_rows=rows)
        with self.lock, self.lane_context():
            ids, langs = self.engine.transcribe_auto(audios, sot, list(lang_ids), make_opts)
        return list(zip(ids, langs))

    def transcribe_auto(self, audio: np.ndarray, spec: tuple) -> tuple:
        key = ("auto",) + tuple(spec)
        if self.batcher is not None:
            return self.batcher.call(key, audio)
        return self._run_auto_batch(key, [audio])[0]

    def close(self) -> None:
        if self.batcher is not None:
            self.batcher.close()
        self.engine.close()


class B200WhisperSTTHandler(_api.BaseSTTHandler):
    """Speech-to-text on the H100 engine.  `model_name`: a local transformers Whisper checkpoint directory / hub id
    (weights are read once on the CPU and copied into the engine), or "random:<geometry>[:seed]" for seeded
    random-init weights at a reference geometry (tiny/small/large-v3) -- used by the tests and benches because no
    checkpoints exist offline."""

    _language_token_id_map: Optional[dict[int, str]] = None

    def setup(self, model_name: str = "distil-whisper/distil-large-v3", device: str = "cuda", torch_dtype: str = "float16",
              compile_mode: Optional[str] = None, language: Optional[str] = None, gen_kwargs: dict[str, Any] = {},
              max_batch: int = 1, batch_wait_ms: float = 6.0, lane: Optional[int] = None, lanes: int = 1, batch_gap_ms: float = 0.8) -> None:
        if not str(device).startswith("cuda"):
            raise ValueError(f"B200WhisperSTTHandler runs on CUDA (sm_90a) only, got device={device!r}; there is no CPU fallback")
        from .. import engine as E  # raises ImportError if libs2s_b200.so is not built

        self.device = device
        self.device_index = int(device.split(":")[1]) if ":" in device else 0
        self.torch_dtype = torch_dtype
        self.compile_mode = compile_mode  # accepted for config compatibility; the engine has no tracing compiler
        self.gen_kwargs = dict(gen_kwargs)
        self.start_language = language
        self.last_language = language if language != "auto" else None
        if self.last_language is not None:
            self.gen_kwargs["language"] = self.last_language
        self._E = E
        self.processor = None
        # one persistent decode launch carries up to 16 sessions; more concurrent sessions queue in the batcher
        self.max_batch = max(1, min(int(max_batch), 16))
        self.batch_wait_s = float(batch_wait_ms) / 1000.0      # upper bound; a batch leaves once arrivals pause for batch_gap_ms
        self.batch_gap_s = float(batch_gap_ms) / 1000.0 if batch_gap_ms and batch_gap_ms > 0 else None
        # SM partition: the handler instances of lane i share lane i's engine (engine.get_context; INTEGRATION.md section 4)
        self.lanes = max(1, int(lanes))
        if lane is None:   # not pinned by the caller: units join the lanes round-robin in construction order
            lane = assign_lane(("whisper", model_name, self.device_index), self.lanes)
        self.lane = int(lane) % self.lanes
        self._shared_key = None
        if self.max_batch > 1:
            self._shared_key = ("whisper", model_name, torch_dtype, self.device_index, self.max_batch, self.lane, self.lanes)
            self.bundle = acquire_shared(self._shared_key, lambda: self._load(model_name), lambda b: b.close())
        else:
            self.bundle = self._load(model_name)
        self.engine, self.tokens, self._decode_text = self.bundle.engine, self.bundle.tokens, self.bundle.decode_text
        self.processor = getattr(self.bundle, "processor", None)
        self.warmup()

    # -- loading ---------------------------------------------------------------------------------
    def _load(self, model_name: str) -> _EngineBundle:
        E = self._E
        if model_name.startswith("random:"):
            parts = model_name.split(":")
            geom = GEOMETRIES[parts[1]]
            seed = int(parts[2]) if len(parts) > 2 else 0
            engine = E.WhisperEngine(geom, dtype=self.torch_dtype, max_batch=self.max_batch, device=self.device_index,
                                     lane=self.lane, lanes=self.lanes)
            engine.init_random(seed)
            return _EngineBundle(E, engine, TokenTable.synthetic(geom["vocab"]), lambda ids: " ".join(f"<{i}>" for i in ids),
                                 self.max_batch, self.batch_wait_s, self.lane, self.lanes, self.batch_gap_s)
        from transformers import AutoModelForSpeechSeq2Seq, AutoProcessor
        processor = AutoProcessor.from_pretrained(model_name)
        hf = AutoModelForSpeechSeq2Seq.from_pretrained(model_name)
        c = hf.config
        geom = dict(d_model=c.d_model, heads=c.encoder_attention_heads, enc_layers=c.encoder_layers, dec_layers=c.decoder_layers,
                    ffn=c.encoder_ffn_dim, n_mels=c.num_mel_bins, vocab=c.vocab_size,
                    max_source_positions=c.max_source_positions, max_target_positions=c.max_target_positions)
        engine = E.WhisperEngine(geom, dtype=self.torch_dtype, max_batch=self.max_batch, device=self.device_index,
                                     lane=self.lane, lanes=self.lanes)
        engine.load_state_dict({k: v for k, v in hf.state_dict().items() if not k.startswith("proj_out")})
        tokens = TokenTable.from_generation_config(hf.generation_config)
        del hf
        bundle = _EngineBundle(E, engine, tokens,
                               lambda ids: processor.batch_decode([ids], skip_special_tokens=True, decode_with_timestamps=False)[0],
                               self.max_batch, self.batch_wait_s, self.lane, self.lanes, self.batch_gap_s)
        bundle.processor = processor   # every handler sharing the engine sees the processor, not only the one that loaded it
        return bundle

    def warmup(self) -> None:
        logger.info("Warming up %s", type(self).__name__)
        dummy = np.zeros(16000, dtype=np.float32)
        for _ in range(2):
            self._transcribe(dummy, self._forced_language() or DEFAULT_LANGUAGE)

    # -- decoding controls ------------------------------------------------------------------------
    def _forced_language(self) -> Optional[str]:
        forced = self.gen_kwargs.get("language")
        return forced if isinstance(forced, str) and forced and forced != "auto" else None

    def _prefix(self, lang_id: Optional[int]) -> list:
        """Decoder prompt of `_retrieve_init_tokens` (TF generation_whisper.py:1455-1608): multilingual checkpoints get
        [sot, language, task, notimestamps]; English-only ones (whisper-*.en, distil-*.en: no lang_to_id / task_to_id in
        the generation config) get [sot, notimestamps] -- never invented language / task tokens."""
        t = self.tokens
        tail = [] if self.gen_kwargs.get("return_timestamps") else [t.no_timestamps]
        if not t.lang_to_id or lang_id is None:
            return [t.sot] + tail
        task = t.translate if self.gen_kwargs.get("task") == "translate" else t.transcribe
        return [t.sot, int(lang_id), task] + tail

    def _options(self, language: str):
        t = self.tokens
        lang_id = t.lang_to_id.get(language, t.lang_to_id.get(DEFAULT_LANGUAGE)) if t.lang_to_id else None
        return self._E.WhisperDecodeOptions(prefix=self._prefix(lang_id), eos_id=t.eos,
                                            max_new_tokens=int(self.gen_kwargs.get("max_new_tokens", 128)),
                                            suppress=t.suppress, begin_suppress=t.begin_suppress)

    def _detect_language(self, audio: np.ndarray) -> Optional[str]:
        """Encoder + one decoder step restricted to the language tokens (reference :166-197)."""
        t = self.tokens
        if not t.lang_to_id:
            return None
        try:
            tok = self.bundle.detect_language(np.ascontiguousarray(audio[:480000], dtype=np.float32), t.sot,
                                              list(t.lang_to_id.values()))
        except Exception as e:  # the reference survives a failing detection and falls back (:188-197)
            logger.warning("Whisper language detection failed (%s); falling back to the previous language", e)
            return None
        return t.id_to_lang.get(int(tok))

    def _transcribe(self, audio: np.ndarray, language: str) -> list[int]:
        ids = self.bundle.transcribe(np.ascontiguousarray(audio, dtype=np.float32), self._options(language))
        return [i for i in ids if i != self.tokens.eos]

    # -- the slot -----------------------------------------------------------------------------------
    def process(self, vad_audio: Any) -> Iterator[Any]:
        logger.debug("infering whisper (b200)...")
        audio = np.asarray(vad_audio.audio, dtype=np.float32)
        forced = self._forced_language()
        language_code = forced
        ids = None
        if forced is None and self.tokens.lang_to_id:
            # detection and decode on one encoder pass (the reference reuses `encoder_outputs`, :236-241)
            try:
                t = self.tokens
                fallback = t.lang_to_id.get(self.last_language or DEFAULT_LANGUAGE, t.lang_to_id.get(DEFAULT_LANGUAGE))
                spec = (t.sot, tuple(t.lang_to_id.values()), fallback, tuple(self._prefix(fallback)[2:]), t.eos,
                        int(self.gen_kwargs.get("max_new_tokens", 128)), tuple(t.suppress), tuple(t.begin_suppress))
                raw, tok = self.bundle.transcribe_auto(np.ascontiguousarray(audio[:480000], dtype=np.float32), spec)
                language_code = t.id_to_lang.get(int(tok)) or self.last_language or DEFAULT_LANGUAGE
                ids = [i for i in raw if i != t.eos]
            except Exception as e:  # the reference survives a failing detection and falls back (:188-197)
                logger.warning("Whisper language detection failed (%s); falling back to the previous language", e)
                language_code = self.last_language or DEFAULT_LANGUAGE
        elif forced is None:
            language_code = self.last_language or DEFAULT_LANGUAGE
        if ids is None:
            ids = self._transcribe(audio, language_code)
        if language_code in SUPPORTED_LANGUAGES:
            self.last_language = language_code
        else:
            logger.warning("Whisper detected unsupported language: %s", language_code)
        pred_text = self._decode_text(ids)
        logger.debug("finished whisper inference")
        if self.start_language == "auto":
            language_code += "-auto"
        if getattr(vad_audio, "mode", None) == "progressive":
            yield _api.PartialTranscription(text=pred_text, turn_id=vad_audio.turn_id, turn_revision=vad_audio.turn_revision)
            return
        yield _api.Transcription(text=pred_text, language_code=language_code, turn_id=vad_audio.turn_id,
                                 turn_revision=vad_audio.turn_revision, speech_stopped_at_s=vad_audio.created_at_s)

    def cleanup(self) -> None:
        bundle = getattr(self, "bundle", None)
        if bundle is None:
            return
        self.bundle = None
        if self._shared_key is not None:
            release_shared(self._shared_key)  # the last handler of the process closes the shared engine
        else:
            bundle.close()


# Whisper geometries (transformers WhisperConfig values of the public checkpoints; SURVEY.md Appendix A)
GEOMETRIES = {
    "micro": dict(d_model=128, heads=2, enc_layers=2, dec_layers=2, ffn=512, n_mels=80, vocab=4096),
    "tiny": dict(d_model=384, heads=6, enc_layers=4, dec_layers=4, ffn=1536, n_mels=80, vocab=51865),
    "small": dict(d_model=768, heads=12, enc_layers=12, dec_layers=12, ffn=3072, n_mels=80, vocab=51865),
    "large-v3": dict(d_model=1280, heads=20, enc_layers=32, dec_layers=32, ffn=5120, n_mels=128, vocab=51866),
}
