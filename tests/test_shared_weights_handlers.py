"""CPU: the handlers' opt-in `share_weights` with fake engines.  With the flag, the first lane of a model loads the
checkpoint and every later lane's engine comes from share() on a live one; each lane keeps its own bundle; handlers close
in any order without deadlock and a closing engine is never handed out as a source.  Without it, every lane loads its own."""
import contextlib
import types
from threading import Event

import numpy as np
import pytest

from speech_to_speech_b200 import batcher


class _Fake:
    """An engine that records loads, shares and closes in `log`."""

    def __init__(self, log, lane, lanes, source=None, **caps):
        self.log, self.lane, self.lanes, self.source, self.caps, self.closed = log, lane, lanes, source, caps, False
        self.device = 0
        self.cfg = types.SimpleNamespace(max_prefill=512, max_text=64, max_positions=256)
        self.max_positions = caps.get("max_positions", 256)
        log.append(("share" if source is not None else "load", lane))

    def share(self, lane, lanes, **caps):
        assert not self.closed, "a closed engine was handed out as a weight source"
        return type(self)(self.log, lane, lanes, source=self, **caps)

    def init_random(self, seed):
        pass

    def max_decode_batch(self):
        return 4

    def max_batch(self):
        return 4

    def transcribe(self, audio, opts):
        return [[1, 2, opts.eos_id] for _ in audio]

    def close(self):
        self.closed = True
        self.log.append(("close", self.lane))


@pytest.fixture(autouse=True)
def _no_leftovers():
    yield
    assert not batcher._weight_holders, "every engine handed out must be forgotten when it closes"


# ---- LLM ------------------------------------------------------------------------------------------------------------------
def _llm_units(monkeypatch, share):
    from speech_to_speech_b200 import engine as E
    from speech_to_speech_b200.handlers import language_model_handler as LH
    log = []
    monkeypatch.setattr(E, "LlamaEngine", lambda geom, lane=0, lanes=1, **kw: _Fake(log, lane, lanes, **kw))

    def unit(lane):
        h = object.__new__(LH.B200LanguageModelHandler)
        gk = {"max_new_tokens": 8, "max_sessions": 2, "lane": lane, "lanes": 2}
        if share:
            gk["share_weights"] = True
        h._load_model("random:micro:1", "cuda:0", "bfloat16", gk)
        return h
    return log, [unit(0), unit(1), unit(0)]


@pytest.mark.parametrize("order", [(0, 1, 2), (1, 2, 0), (2, 1, 0)])
def test_llm_lanes_share_one_load(monkeypatch, order):
    log, (a0, b1, a0b) = _llm_units(monkeypatch, share=True)
    assert [k for k, _ in log] == ["load", "share"]          # the checkpoint factory ran once
    assert b1.engine.source is a0.engine and b1.engine.lane == 1
    assert b1.engine.caps == {"max_sessions": 2, "max_positions": 4096}
    assert a0.bundle is a0b.bundle and a0.bundle is not b1.bundle   # bundles stay per lane
    assert b1.bundle.tokenizer is a0.bundle.tokenizer and b1.bundle.eos_ids == a0.bundle.eos_ids
    for h in (a0, b1, a0b):
        assert "share_weights" not in h.gen_kwargs
    hs = (a0, b1, a0b)
    for i in order:
        hs[i].cleanup()
    assert a0.engine.closed and b1.engine.closed


def test_llm_a_closed_source_is_not_handed_out(monkeypatch):
    log, (a0, b1, a0b) = _llm_units(monkeypatch, share=True)
    a0.cleanup()
    a0b.cleanup()       # lane 0's engine closes; lane 1's still reads the weights
    assert a0.engine.closed
    from speech_to_speech_b200.handlers import language_model_handler as LH
    h = object.__new__(LH.B200LanguageModelHandler)
    h._load_model("random:micro:1", "cuda:0", "bfloat16", {"max_sessions": 2, "lane": 0, "lanes": 2, "share_weights": True})
    assert h.engine.source is b1.engine            # the live lane-1 engine is the source now
    assert [k for k, _ in log].count("load") == 1
    h.cleanup()
    b1.cleanup()


def test_llm_without_the_flag_every_lane_loads(monkeypatch):
    log, hs = _llm_units(monkeypatch, share=False)
    assert sorted(log) == [("load", 0), ("load", 1)]
    for h in hs:
        h.cleanup()


# ---- STT ------------------------------------------------------------------------------------------------------------------
def _stt_unit(monkeypatch, log, lane, share):
    from speech_to_speech_b200 import engine as E
    from speech_to_speech_b200.handlers import whisper_stt_handler as WH
    monkeypatch.setattr(E, "WhisperEngine", lambda geom, lane=0, lanes=1, **kw: _Fake(log, lane, lanes, **kw))
    monkeypatch.setattr(E, "lane_context", lambda *a: contextlib.nullcontext())   # no CUDA streams on the CPU
    h = object.__new__(WH.B200WhisperSTTHandler)
    h.setup(model_name="random:micro", device="cuda:0", max_batch=2, lane=lane, lanes=2, share_weights=share)
    return h


@pytest.mark.parametrize("first", [0, 1])
def test_stt_lanes_share_one_load(monkeypatch, first):
    log = []
    hs = [_stt_unit(monkeypatch, log, lane, True) for lane in (0, 1)]
    assert [k for k, _ in log] == ["load", "share"]
    assert hs[1].engine.source is hs[0].engine and hs[1].engine.caps == {"max_batch": 2}
    assert hs[0].bundle is not hs[1].bundle and hs[1].bundle.lane == 1
    assert hs[1].bundle.tokens is hs[0].bundle.tokens
    hs[first].cleanup()
    hs[1 - first].cleanup()
    assert all(h.engine.closed for h in hs)


def test_stt_without_the_flag_every_lane_loads(monkeypatch):
    log = []
    hs = [_stt_unit(monkeypatch, log, lane, False) for lane in (0, 1)]
    assert sorted(log) == [("load", 0), ("load", 1)]
    for h in hs:
        h.cleanup()


# ---- TTS ------------------------------------------------------------------------------------------------------------------
def _tts_units(monkeypatch, share):
    import torch
    from speech_to_speech_b200.handlers import qwen3_tts_handler as TH
    log = []

    class FakeModel:
        @classmethod
        def from_random(cls, geometry, lane=0, lanes=1, **kw):
            return _Fake(log, lane, lanes)

    monkeypatch.setattr(TH, "B200Qwen3TTS", FakeModel)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    seen = []
    monkeypatch.setattr(TH._Base, "setup", lambda self, *a, **kw: seen.append(kw["gen_kwargs"]))

    def unit(lane):
        h = object.__new__(TH.B200Qwen3TTSHandler)
        gk = {"lanes": 2, "lane": lane}
        if share:
            gk["share_weights"] = True
        h.setup(Event(), model_name="random:micro", device="cuda:0", max_sessions=2, gen_kwargs=gk)
        h.device = "cuda:0"
        h._setup_faster("random:micro", "bfloat16", "eager", "torch")
        return h
    hs = [unit(0), unit(1)]
    assert all("share_weights" not in g and "lanes" not in g for g in seen)
    return log, hs


@pytest.mark.parametrize("first", [0, 1])
def test_tts_lanes_share_one_load(monkeypatch, first):
    log, hs = _tts_units(monkeypatch, share=True)
    assert [k for k, _ in log] == ["load", "share"]
    assert hs[1].model.source is hs[0].model and hs[1].model.caps == {"max_sessions": 2} and hs[1].model.lane == 1
    hs[first].cleanup()
    hs[1 - first].cleanup()
    assert ("close", 0) in log and ("close", 1) in log


def test_tts_without_the_flag_every_lane_loads(monkeypatch):
    log, hs = _tts_units(monkeypatch, share=False)
    assert sorted(log) == [("load", 0), ("load", 1)]
    for h in hs:
        h.cleanup()


def test_weight_source_registry_hands_out_live_objects_only():
    made = []
    a = batcher.weight_source("k", lambda: made.append("load") or "A", lambda src: made.append(("share", src)) or "B")
    b = batcher.weight_source("k", lambda: "never", lambda src: made.append(("share", src)) or "C")
    assert (a, b) == ("A", "C") and made == ["load", ("share", "A")]
    batcher.forget_weight_source("k", a)
    d = batcher.weight_source("k", lambda: "never", lambda src: src + "D")
    assert d == "CD"
    for o in (b, d):
        batcher.forget_weight_source("k", o)
    assert np.all([k != "k" for k in batcher._weight_holders])
