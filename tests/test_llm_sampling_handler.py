"""CPU: how B200LanguageModelHandler resolves and passes its token-choice options (fake engine, no GPU):
transformers' defaults < the checkpoint's generation_config < gen_kwargs; rejection of what the kernels do not implement;
one seed per response from a generator seeded by gen_kwargs["seed"]; set_sampling reaches the slot before its prefill."""
import types

import pytest

from speech_to_speech_b200.handlers import language_model_handler as LH


def test_reference_defaults_are_greedy():
    # the reference CLI's defaults (language_model_arguments.py): do_sample=False, temperature=0.0
    s = LH.resolve_generation({"do_sample": False, "temperature": 0.0, "max_new_tokens": 128})
    assert s == dict(do_sample=False, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0, min_new_tokens=0)


def test_checkpoint_generation_config_is_honoured_when_sampling():
    from transformers import GenerationConfig
    ckpt = GenerationConfig(top_k=20, top_p=0.8, temperature=0.7)
    s = LH.resolve_generation({"do_sample": True}, ckpt)
    assert s["do_sample"] and s["top_k"] == 20 and s["top_p"] == pytest.approx(0.8) and s["temperature"] == pytest.approx(0.7)
    s = LH.resolve_generation({"do_sample": True, "temperature": 1.1, "min_new_tokens": 3}, ckpt)   # gen_kwargs win
    assert s["temperature"] == pytest.approx(1.1) and s["top_k"] == 20 and s["min_new_tokens"] == 3
    s = LH.resolve_generation({"do_sample": True})      # transformers' own default top_k=50
    assert s["top_k"] == 50 and s["top_p"] == 1.0
    assert not LH.resolve_generation({}, ckpt)["do_sample"]


@pytest.mark.parametrize("kw", [
    {"do_sample": True, "temperature": 0.0}, {"min_p": 0.05}, {"typical_p": 0.9}, {"epsilon_cutoff": 3e-4}, {"eta_cutoff": 1e-3},
    {"num_beams": 4}, {"no_repeat_ngram_size": 3}, {"do_sample": True, "top_p": 1.5}, {"repetition_penalty": 0.0},
])
def test_unsupported_options_are_rejected(kw):
    with pytest.raises(ValueError):
        LH.resolve_generation(kw)


class _Eng:
    cfg = types.SimpleNamespace(max_prefill=8)
    device = 0
    max_positions = 64

    def __init__(self):
        self.calls = []

    def reset(self, slot):
        self.calls.append(("reset", slot))

    def set_sampling(self, slot, **kw):
        self.calls.append(("set_sampling", slot, kw))

    def prefill(self, slot, ids):
        self.calls.append(("prefill", slot))
        return [0], None

    def max_decode_batch(self):
        return 4

    def close(self):
        pass


def _unit(monkeypatch, gen_kwargs):
    from speech_to_speech_b200 import engine as E
    eng = _Eng()
    monkeypatch.setattr(E, "LlamaEngine", lambda *a, **k: types.SimpleNamespace(
        init_random=lambda seed: None, **{n: getattr(eng, n) for n in ("cfg", "device", "max_positions", "reset", "set_sampling",
                                                                         "prefill", "max_decode_batch", "close")}))
    h = object.__new__(LH.B200LanguageModelHandler)
    h._load_model("random:micro:1", "cuda:0", "bfloat16", dict(gen_kwargs))
    return h, eng


def test_fixed_seed_gives_the_same_seed_sequence(monkeypatch):
    a, _ = _unit(monkeypatch, {"seed": 5, "do_sample": True})
    b, _ = _unit(monkeypatch, {"seed": 5, "do_sample": True})
    c, _ = _unit(monkeypatch, {"seed": 6, "do_sample": True})
    try:
        sa = [a.next_sampling()["seed"] for _ in range(4)]
        assert sa == [b.next_sampling()["seed"] for _ in range(4)]
        assert sa != [c.next_sampling()["seed"] for _ in range(4)]
        assert len(set(sa)) == 4 and all(0 <= s < 2 ** 64 for s in sa)
        assert "seed" not in a.gen_kwargs
        assert a.next_sampling()["eos_ids"] == [2047]       # the model's EOS ids reach the kernel (min_new_tokens)
    finally:
        for h in (a, b, c):
            h.cleanup()


def test_set_sampling_precedes_the_prefill(monkeypatch):
    h, eng = _unit(monkeypatch, {"seed": 1, "do_sample": True, "top_k": 7, "min_new_tokens": 2})
    try:
        list(h.generate_text_stream([1, 2, 3], max_new_tokens=1))
        kinds = [c[0] for c in eng.calls]
        assert kinds[:3] == ["reset", "set_sampling", "prefill"]
        kw = eng.calls[1][2]
        assert kw["do_sample"] and kw["top_k"] == 7 and kw["min_new_tokens"] == 2 and isinstance(kw["seed"], int)
    finally:
        h.cleanup()
