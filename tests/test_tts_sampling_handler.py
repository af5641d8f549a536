"""CPU: sampling options of the TTS slot -- tts_model.resolve_sampling (qwen-tts keywords, rejections), the per-utterance seed
sequence of B200Qwen3TTS, greedy utterances that never call set_sampling, and the handler's gen_kwargs reaching the model
call through its per-handler view, on both base classes."""
import types

import pytest
import torch

from speech_to_speech_b200.tts_model import COUSIN_SAMPLING, B200Qwen3TTS, resolve_sampling
from test_tts_handler import FakeModel, _handler_module, _make, _tts_input


def test_resolution_of_the_qwen_tts_keywords():
    assert resolve_sampling(None) == {"talker": None, "predictor": None}
    c = resolve_sampling(COUSIN_SAMPLING)
    assert c["talker"] == dict(do_sample=True, temperature=0.9, top_k=50, top_p=1.0, repetition_penalty=1.05)
    assert c["predictor"] == dict(do_sample=True, temperature=1.0, top_k=50, top_p=0.8, repetition_penalty=1.0)
    r = resolve_sampling(None, do_sample=True, temperature=0.7, subtalker_dosample=True, subtalker_top_p=0.5)
    assert r["talker"] == dict(do_sample=True, temperature=0.7, top_k=0, top_p=1.0, repetition_penalty=1.0)
    assert r["predictor"] == dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.5, repetition_penalty=1.0)
    # call keywords overlay the preset; greedy settings of one model come back as None
    r = resolve_sampling(COUSIN_SAMPLING, subtalker_dosample=False, top_k=20)
    assert r["predictor"] is None and r["talker"]["top_k"] == 20 and r["talker"]["temperature"] == 0.9
    assert resolve_sampling(None, do_sample=False, repetition_penalty=1.2)["talker"] == dict(
        do_sample=False, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.2)
    assert resolve_sampling(None, do_sample=None, num_beams=1, min_p=0.0) == {"talker": None, "predictor": None}


@pytest.mark.parametrize("bad", [dict(min_p=0.1), dict(typical_p=0.9), dict(num_beams=4), dict(no_repeat_ngram_size=3),
                                 dict(subtalker_repetition_penalty=1.1), dict(min_new_tokens=5), dict(do_sample=True, temperature=0.0),
                                 dict(do_sample=True, top_p=0.0), dict(top_k=-1), dict(repetition_penalty=0.0),
                                 dict(guidance_scale=3.0)])
def test_rejections(bad):
    with pytest.raises(ValueError):
        resolve_sampling(None, **bad)


def test_rejected_presets():
    with pytest.raises(ValueError):
        resolve_sampling({"talker": dict(top_q=1)})
    with pytest.raises(ValueError):
        resolve_sampling({"predictor": dict(repetition_penalty=1.1)})


class Eng:
    """Records what B200Qwen3TTS asks of the engine (the interface of Qwen3TTSEngine)."""
    device, codec_eos = 0, 7
    cfg = types.SimpleNamespace(max_positions=4096, max_text=128)

    def __init__(self):
        self.n, self.calls = {}, []

    def max_batch(self):
        return 16

    def prefill(self, slot, ids, spk):
        self.n[slot] = 0
        self.calls.append(("prefill", slot))

    def set_sampling(self, slot, *, talker=None, predictor=None, seed=0):
        self.calls.append(("set_sampling", slot, talker, predictor, seed))

    def frames(self, s):
        return self.n[s]

    def set_frames(self, s, n):
        self.n[s] = n

    def decode_frames(self, slots, n):
        codes = torch.zeros((len(slots), n, 16), dtype=torch.int32)
        codes[:, -1, 0] = self.codec_eos
        for s in slots:
            self.n[s] += n
        return codes

    def history_context(self, s, valid, left):
        return min(left, self.n[s] - valid)

    def decode_audio_batch(self, slots, valid, left):
        return [torch.zeros(valid * 1920) for _ in slots]

    def close(self):
        pass


def _speak(model, **kw):
    return list(model.generate_custom_voice_streaming("hi", "a", chunk_size=4, max_new_tokens=8, **kw))


def test_greedy_utterances_never_call_set_sampling():
    eng = Eng()
    m = B200Qwen3TTS(eng, lambda t: [1, 2], {"a": 0})
    _speak(m)
    _speak(m, do_sample=False)
    assert [c[0] for c in eng.calls] == ["prefill", "prefill"]


def test_seed_sequence_of_a_fixed_sampling_seed():
    seeds = []
    for _ in range(2):
        eng = Eng()
        m = B200Qwen3TTS(eng, lambda t: [1, 2], {"a": 0}, sampling=COUSIN_SAMPLING, sampling_seed=7)
        for _ in range(3):
            _speak(m)
        _speak(m, do_sample=False, repetition_penalty=1.0, subtalker_dosample=False)   # greedy: no seed drawn
        _speak(m)
        calls = [c for c in eng.calls if c[0] == "set_sampling"]
        assert len(calls) == 4 and all(c[2] == resolve_sampling(COUSIN_SAMPLING)["talker"] for c in calls)
        assert all(c[3] == resolve_sampling(COUSIN_SAMPLING)["predictor"] for c in calls)
        seeds.append([c[4] for c in calls])
    assert seeds[0] == seeds[1] and len(set(seeds[0])) == 4 and all(0 <= s < 2 ** 64 for s in seeds[0])
    m = B200Qwen3TTS(Eng(), lambda t: [1, 2], {"a": 0}, sampling=COUSIN_SAMPLING, sampling_seed=8)
    _speak(m)
    assert [c[4] for c in m.engine.calls if c[0] == "set_sampling"][0] != seeds[0][0]
    # an explicit per-call seed wins; set_sampling follows the prefill of the same slot
    eng = Eng()
    m = B200Qwen3TTS(eng, lambda t: [1, 2], {"a": 0})
    _speak(m, do_sample=True, sampling_seed=1234)
    assert eng.calls[0] == ("prefill", 0) and eng.calls[1][0] == "set_sampling" and eng.calls[1][4] == 1234


def test_unsupported_keyword_fails_the_call():
    m = B200Qwen3TTS(Eng(), lambda t: [1, 2], {"a": 0})
    with pytest.raises(ValueError):
        _speak(m, min_p=0.05)


@pytest.mark.parametrize("use_reference", [True, False])
def test_handler_options_reach_the_model_call(monkeypatch, use_reference):
    mod = _handler_module(use_reference)
    fake = FakeModel([torch.zeros(512).numpy() + 0.1])
    gk = dict(do_sample=True, temperature=0.8, subtalker_top_k=20, sampling_seed=5, seed=3)
    h = _make(mod, fake, monkeypatch, speaker="Aiden", gen_kwargs=dict(gk))
    assert isinstance(h.model, mod.HandlerModelView) and h.model.wrapped is fake
    assert h.model.get_supported_speakers() == ["aiden"] and h.model.model.model.tts_model_type == "custom_voice"
    assert not {"do_sample", "temperature", "subtalker_top_k", "sampling_seed", "seed"} & set(h.gen_kwargs)
    fake.calls.clear()
    list(h.process(_tts_input(mod, "Hello there.")))
    list(h.process(_tts_input(mod, "Hello again.")))
    gens = [kw for k, kw in fake.calls if k == "gen"]
    assert len(gens) == 2
    for kw in gens:
        assert kw["do_sample"] is True and kw["temperature"] == 0.8 and kw["subtalker_top_k"] == 20
        assert kw["speaker"] == "Aiden" and kw["chunk_size"] == 8
    assert gens[0]["sampling_seed"] != gens[1]["sampling_seed"]
    import random
    r = random.Random(5)
    r.getrandbits(64)                                         # setup's warm-up utterance took the first seed
    assert [kw["sampling_seed"] for kw in gens] == [r.getrandbits(64), r.getrandbits(64)]
    h.cleanup()


@pytest.mark.parametrize("use_reference", [True, False])
def test_handler_without_options_keeps_the_shared_model_and_rejects_bad_options(monkeypatch, use_reference):
    mod = _handler_module(use_reference)
    fake = FakeModel([])
    h = _make(mod, fake, monkeypatch, speaker="Aiden")
    assert h.model is fake
    with pytest.raises(ValueError):
        _make(mod, FakeModel([]), monkeypatch, speaker="Aiden", gen_kwargs=dict(typical_p=0.5))
