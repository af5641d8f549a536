"""engine.get_context / lane_stream / lane_context on the CPU with a fake library: one context per (device, lane), the SM
partition each lane receives, and what one lane (the default) means."""
import contextlib
import types

import pytest


@pytest.fixture()
def E(monkeypatch):
    import torch
    from speech_to_speech_b200 import _lib, engine
    calls = []

    class FakeLib:
        def s2s_init(self, device, out):
            calls.append(("init", device))
            out._obj.value = 1000 + len(calls)
            return 0

        def s2s_set_sm_partition(self, ctx, ctas):
            calls.append(("partition", ctx.value, ctas))
            return 0
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda d: types.SimpleNamespace(multi_processor_count=132))
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: types.SimpleNamespace(kind="lane", device=device))
    monkeypatch.setattr(torch.cuda, "default_stream", lambda d=None: types.SimpleNamespace(kind="default", device=d))
    monkeypatch.setattr(engine, "_ctx_by_device", {})
    monkeypatch.setattr(engine, "_lane_streams", {})
    engine._test_calls = calls
    return engine


def test_one_context_per_device_and_lane_with_its_sm_partition(E):
    a, a2, b = E.get_context(0, 0, 2), E.get_context(0, 0, 2), E.get_context(0, 1, 2)
    assert a is a2 and a.value != b.value
    whole = E.get_context(0)
    assert whole.value not in (a.value, b.value)
    parts = [c for c in E._test_calls if c[0] == "partition"]
    assert [p[2] for p in parts] == [66, 66] and {p[1] for p in parts} == {a.value, b.value}      # 132 SMs // 2 lanes; none for one lane
    assert E.get_context(0, 2, 3) is not None and [c for c in E._test_calls if c[0] == "partition"][-1][2] == 44
    with pytest.raises(ValueError):
        E.get_context(0, 2, 2)


def test_lane_streams_and_contexts(E, monkeypatch):
    import torch
    assert E.lane_stream(0).kind == "default" and E.lane_stream(1, 0, 1).device == 1
    s0, s0b, s1 = E.lane_stream(0, 0, 2), E.lane_stream(0, 0, 2), E.lane_stream(0, 1, 2)
    assert s0 is s0b and s0 is not s1 and s0.kind == "lane"
    assert isinstance(E.lane_context(0), contextlib.nullcontext)                  # one lane: the calling thread's stream is left alone
    entered = []
    monkeypatch.setattr(torch.cuda, "stream", lambda s: entered.append(s) or contextlib.nullcontext())
    E.lane_context(0, 1, 2)
    assert entered == [s1]
