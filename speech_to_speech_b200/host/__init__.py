"""Host-side interface layer.

`resolve()` returns the reference's own stage-runtime types when `speech_to_speech` is importable (the
drop-in case: our handlers then subclass the reference's BaseHandler / BaseSTTHandler and are driven by its
unchanged thread loop), and otherwise a minimal mirror of that interface (same names, argument meaning and
error behaviour; reference: speech_to_speech/baseHandler.py:24-187,
pipeline/messages.py:45-223) so that the handlers can be exercised on a machine that only has this repo."""
from __future__ import annotations

import importlib
import sys
import types
from dataclasses import dataclass
from typing import Any


@dataclass(frozen=True)
class HostAPI:
    source: str  # "reference" or "mirror"
    BaseHandler: Any
    BaseSTTHandler: Any
    VADAudio: Any
    Transcription: Any
    PartialTranscription: Any
    TTSInput: Any
    EndOfResponse: Any
    AUDIO_RESPONSE_DONE: Any
    PIPELINE_END: Any


_cached: HostAPI | None = None


def _stub_optional(name: str) -> None:
    """The reference's own tests stub optional deps the same way (T/test_whisper_progressive_transcription.py:49-59)."""
    if name in sys.modules:
        return
    try:
        importlib.import_module(name)
    except Exception:
        m = types.ModuleType(name)
        if name == "nltk":
            m.sent_tokenize = lambda text, language="english": [s for s in text.replace("? ", "?|").replace(". ", ".|").replace("! ", "!|").split("|") if s]
            m.download = lambda *a, **k: True
            m.data = types.SimpleNamespace(find=lambda *a, **k: True)
        sys.modules[name] = m


def resolve(prefer_reference: bool = True) -> HostAPI:
    global _cached
    if _cached is not None and (prefer_reference or _cached.source == "mirror"):
        return _cached
    if prefer_reference:
        try:
            bh = importlib.import_module("speech_to_speech.baseHandler")
            stt = importlib.import_module("speech_to_speech.STT.base_stt_handler")
            msg = importlib.import_module("speech_to_speech.pipeline.messages")
            _cached = HostAPI("reference", bh.BaseHandler, stt.BaseSTTHandler, msg.VADAudio, msg.Transcription,
                              msg.PartialTranscription, msg.TTSInput, msg.EndOfResponse, msg.AUDIO_RESPONSE_DONE,
                              msg.PIPELINE_END)
            return _cached
        except Exception:
            pass
    from . import mirror as mr
    _cached = HostAPI("mirror", mr.BaseHandler, mr.BaseSTTHandler, mr.VADAudio, mr.Transcription, mr.PartialTranscription,
                      mr.TTSInput, mr.EndOfResponse, mr.AUDIO_RESPONSE_DONE, mr.PIPELINE_END)
    return _cached
