"""CPU: gen_kwargs["weight_dtype"] of the LLM handler reaches the engine, separates shared engines, and is validated.
The engine is a fake that records how it was built."""
import pytest

BUILT = []


class FakeEngine:
    device = 0
    max_positions = 64

    def __init__(self, geometry, **kw):
        self.kw = kw
        BUILT.append(self)

    def init_random(self, seed=0):
        pass

    def max_decode_batch(self):
        return 4

    def close(self):
        pass


@pytest.fixture
def handler_cls(monkeypatch):
    from speech_to_speech_b200 import engine as E
    from speech_to_speech_b200.handlers import language_model_handler as LH
    monkeypatch.setattr(E, "LlamaEngine", FakeEngine)
    BUILT.clear()
    return LH.B200LanguageModelHandler


def _make(cls, **gen):
    h = cls.__new__(cls)      # the base class's constructor belongs to the host pipeline; _load_model is the slot's own
    h._load_model("random:micro", "cuda:0", "bfloat16", gen)
    return h


def test_weight_dtype_reaches_the_engine_and_defaults_to_none(handler_cls):
    a = _make(handler_cls)
    b = _make(handler_cls, weight_dtype="float8_e4m3")
    try:
        assert [e.kw.get("weight_dtype") for e in BUILT] == [None, "float8_e4m3"]
        assert "weight_dtype" not in a.gen_kwargs and "weight_dtype" not in b.gen_kwargs   # not a generation option
    finally:
        a.cleanup()
        b.cleanup()


def test_weight_dtype_is_part_of_the_shared_engine_key(handler_cls):
    hs = [_make(handler_cls, max_sessions=2, lane=0, weight_dtype=w) for w in (None, "float8_e4m3", "float8_e4m3")]
    try:
        assert hs[0]._shared_key != hs[1]._shared_key == hs[2]._shared_key
        assert len(BUILT) == 2 and hs[1].engine is hs[2].engine and hs[0].engine is not hs[1].engine
    finally:
        for h in hs:
            h.cleanup()


@pytest.mark.parametrize("bad", ["int8", "float8_e5m2", "fp8", 8])
def test_unsupported_weight_dtype_raises(handler_cls, bad):
    with pytest.raises(ValueError, match="float8_e4m3"):
        _make(handler_cls, weight_dtype=bad)
    assert not BUILT
