"""GPU: one copy of the weights per GPU.  An engine made by share() on lane 1 of 2 reads the weights of an engine on lane 0
(include/s2s_b200.h, shared weights) and must compute bit for bit what an engine with its own copy of the same seeded
weights computes on the same lane with the same capacities -- while the source decodes other sessions at the same time,
each lane on its own stream and host thread.  Memory is accounted through allocated_bytes (the library's own count), never
through the device's free memory, which other processes move."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from oracle import weights as W

pytestmark = pytest.mark.gpu

FP8 = "float8_e4m3"
S2S_ERR_INVALID = -1


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _concurrently(E, *jobs):
    """jobs: (lane, fn) pairs, each run on its own host thread inside its lane's stream (2 lanes) -> their results."""
    out, err = [None] * len(jobs), []

    def run(i, lane, fn):
        try:
            with E.lane_context(0, lane, 2):
                out[i] = fn()
                torch.cuda.current_stream().synchronize()
        except BaseException as e:  # noqa: BLE001 -- re-raised on the main thread
            err.append(e)
    th = [threading.Thread(target=run, args=(i, lane, fn)) for i, (lane, fn) in enumerate(jobs)]
    [t.start() for t in th]
    [t.join() for t in th]
    if err:
        raise err[0]
    return out


# ---- LLM ------------------------------------------------------------------------------------------------------------
def _llm(E, name, fmt, lane, max_sessions, max_positions, max_prefill, seed=5):
    eng = E.LlamaEngine(W.LLAMA_GEOMETRIES[name].to_dict(), max_sessions=max_sessions, max_positions=max_positions,
                        max_prefill=max_prefill, lane=lane, lanes=2, weight_dtype=fmt)
    eng.init_random(seed)
    return eng


def _llm_run(eng, B, sampled, steps=32):
    """prefill logits of slot 0, a batched prefill of slots 1..B-1, then B sessions decoding `steps` steps -> host arrays"""
    vocab = eng.geometry["vocab"]
    rng = np.random.default_rng(B * 2 + sampled)
    prompts = [rng.integers(0, vocab, 5).tolist() for _ in range(B)]
    for s in range(B):
        eng.reset(s)
        if sampled:
            eng.set_sampling(s, do_sample=True, temperature=0.9, top_k=40, top_p=0.95, repetition_penalty=1.1, seed=100 + s)
    n0, lg0 = eng.prefill(0, prompts[0], return_logits=True)
    firsts = [n0]
    if B > 1:
        firsts.append(eng.prefill_batch(list(range(1, B)), prompts[1:]))
    first = torch.cat(firsts).to(torch.int32)
    ids, lens, lg = eng.decode(list(range(B)), first, steps, return_logits=True)
    return [t.cpu().numpy() for t in (lg0, first, ids, lens, lg)]


@pytest.mark.parametrize("fmt", [None, FP8])
@pytest.mark.parametrize("name", ["micro", "qwen3-micro"])
def test_llm_sharer_equals_own_copy_while_the_source_decodes(E, name, fmt):
    src = _llm(E, name, fmt, 0, max_sessions=4, max_positions=256, max_prefill=64)
    sharer = src.share(1, 2, max_sessions=16, max_positions=192, max_prefill=96)
    own = _llm(E, name, fmt, 1, max_sessions=16, max_positions=192, max_prefill=96)
    try:
        assert sharer.weight_format() == own.weight_format() == src.weight_format()
        assert sharer.max_decode_batch() == own.max_decode_batch()
        for B in (1, 3, min(16, sharer.max_decode_batch())):
            for sampled in (False, True):
                got, _ = _concurrently(E, (1, lambda: _llm_run(sharer, B, sampled)), (0, lambda: _llm_run(src, 4, not sampled)))
                ref, _ = _concurrently(E, (1, lambda: _llm_run(own, B, sampled)), (0, lambda: _llm_run(src, 4, not sampled)))
                for g, r in zip(got, ref):
                    assert g.shape == r.shape and np.array_equal(g, r, equal_nan=True), (B, sampled)
    finally:
        for e in (src, sharer, own):
            e.close()


def test_llm_accounting_and_lifetime(E):
    own = _llm(E, "micro", None, 1, max_sessions=3, max_positions=128, max_prefill=32)
    own_state = own.device_bytes()[1] - own.device_bytes()[0]
    own.close()
    base = E.allocated_bytes()
    src = _llm(E, "micro", None, 0, max_sessions=2, max_positions=256, max_prefill=64)
    sw, st = src.device_bytes()
    assert E.allocated_bytes() - base == st
    a1 = E.allocated_bytes()
    sharer = src.share(1, 2, max_sessions=3, max_positions=128, max_prefill=32)
    w, t = sharer.device_bytes()
    assert w == sw and t - w == own_state
    assert E.allocated_bytes() - a1 == t - w
    with E.lane_context(0, 1, 2):
        before = _llm_run(sharer, 3, True)
    a2 = E.allocated_bytes()
    src.close()   # the source goes first: only its own state is released
    assert a2 - E.allocated_bytes() == st - sw
    with E.lane_context(0, 1, 2):
        after = _llm_run(sharer, 3, True)
    for g, r in zip(after, before):
        assert np.array_equal(g, r, equal_nan=True)
    sharer.close()   # the last holder: the weights go too
    assert E.allocated_bytes() == base


def _rc_all_rejected(lib, h, cfg_dtype):
    one = np.ones(4, np.float32)
    shape = (C.c_int64 * 1)(4)
    return [lib.s2s_llama_bind_tensor(h, b"model.norm.weight", one.ctypes.data_as(C.c_void_p), shape, 1, 0),
            lib.s2s_llama_init_random(h, 1), lib.s2s_llama_finalize(h), lib.s2s_llama_set_weight_format(h, cfg_dtype)]


def test_rejections(E):
    lib = E._lib.load()
    src = _llm(E, "micro", None, 0, max_sessions=2, max_positions=128, max_prefill=32)
    try:
        sharer = src.share(1, 2, max_sessions=2)
        for h in (sharer.handle, src.handle):   # the sharer, and the source while it has a live sharer
            assert _rc_all_rejected(lib, h, src.cfg.compute_dtype) == [S2S_ERR_INVALID] * 4
        assert b"other objects read these weights" in lib.s2s_last_error() or b"shared" in lib.s2s_last_error()
        with pytest.raises(E.S2SError, match="read-only"):
            sharer.init_random(1)
        sharer.close()
        src.init_random(6)        # the sharers are gone: the source can be reloaded again
        src.load_state_dict(W.make_llama_weights(W.LLAMA_GEOMETRIES["micro"], 0))
        # a source that is not finalized, and configurations that differ in more than capacities
        raw = E.LlamaEngine(W.LLAMA_GEOMETRIES["micro"].to_dict(), max_sessions=2, max_positions=128, max_prefill=32)
        with pytest.raises(E.S2SError, match="not finalized"):
            raw.share(1, 2)
        raw.close()
        for field, value in (("rope_theta", 1234.0), ("compute_dtype", E.S2S_F16), ("vocab", 4096)):
            cfg = E._lib.LlamaConfig.from_buffer_copy(src.cfg)
            setattr(cfg, field, value)
            h = C.c_void_p()
            assert lib.s2s_llama_create_shared(E.get_context(0, 1, 2), src.handle, C.byref(cfg), C.byref(h)) == S2S_ERR_INVALID
            assert field.encode() in lib.s2s_last_error()
    finally:
        src.close()


# ---- Whisper --------------------------------------------------------------------------------------------------------
def _whisper(E, lane, max_batch, seed=3):
    eng = E.WhisperEngine(W.WHISPER_GEOMETRIES["micro"].to_dict(), dtype="float16", max_batch=max_batch, lane=lane, lanes=2)
    eng.init_random(seed)
    return eng


def _whisper_run(E, eng, B):
    auds = [W.synthetic_audio(10 + b, 48000 + 16000 * b) for b in range(B)]
    opts = E.WhisperDecodeOptions(prefix=[4000, 4001, 4002, 4003], eos_id=4095, max_new_tokens=24, suppress=[1, 2, 7],
                                  begin_suppress=[220, 4095])
    pcm = torch.zeros((B, max(len(a) for a in auds)), dtype=torch.float32, device="cuda")
    for b, a in enumerate(auds):
        pcm[b, : len(a)] = torch.from_numpy(a).cuda()
    eng.logmel(pcm, [len(a) for a in auds])
    enc = eng.encode(B, return_output=True).cpu().numpy()
    return enc, eng.transcribe(auds, opts)


def test_whisper_sharer_equals_own_copy(E):
    src = _whisper(E, 0, max_batch=3)
    sharer = src.share(1, 2, max_batch=4)
    own = _whisper(E, 1, max_batch=4)
    try:
        w, t = sharer.device_bytes()
        assert w == src.device_bytes()[0] == own.device_bytes()[0] and t - w == own.device_bytes()[1] - own.device_bytes()[0]
        for B in (1, 3):   # one session: the cluster kernel; three: the cooperative kernel
            (genc, gids), _ = _concurrently(E, (1, lambda: _whisper_run(E, sharer, B)), (0, lambda: _whisper_run(E, src, 3)))
            (renc, rids), _ = _concurrently(E, (1, lambda: _whisper_run(E, own, B)), (0, lambda: _whisper_run(E, src, 3)))
            assert np.array_equal(genc, renc) and gids == rids
        cfg = E._lib.WhisperConfig.from_buffer_copy(src.cfg)
        cfg.dec_layers += 1
        h = C.c_void_p()
        lib = E._lib.load()
        assert lib.s2s_whisper_create_shared(E.get_context(0, 1, 2), src.handle, C.byref(cfg), C.byref(h)) == S2S_ERR_INVALID
        assert b"dec_layers" in lib.s2s_last_error()
        assert lib.s2s_whisper_init_random(src.handle, 1) == S2S_ERR_INVALID
    finally:
        for e in (sharer, src, own):
            e.close()


# ---- Qwen3-TTS ------------------------------------------------------------------------------------------------------
def _tts(E, lane, max_sessions, seed=7):
    from speech_to_speech_b200.tts_model import CODEC_GEOMETRIES, TTS_GEOMETRIES
    eng = E.Qwen3TTSEngine(TTS_GEOMETRIES["micro"], CODEC_GEOMETRIES["micro"], max_sessions=max_sessions, max_positions=128,
                           max_text=64, lane=lane, lanes=2)
    eng.init_random(seed)
    return eng


def _tts_run(eng, B, sampling):
    rng = np.random.default_rng(B)
    for s in range(B):
        eng.prefill(s, rng.integers(0, 400, 6 + s).tolist(), 2301)
        if sampling is not None:
            eng.set_sampling(s, talker=sampling["talker"], predictor=sampling["predictor"], seed=50 + s)
    codes = eng.decode_frames(list(range(B)), 8)
    wavs = eng.decode_audio_batch(list(range(B)), 8)
    return codes.cpu().numpy(), [w.cpu().numpy() for w in wavs]


@pytest.mark.parametrize("sampled", [False, True])
def test_tts_sharer_equals_own_copy(E, sampled):
    from speech_to_speech_b200.tts_model import COUSIN_SAMPLING
    sampling = COUSIN_SAMPLING if sampled else None
    src = _tts(E, 0, max_sessions=4)
    sharer = src.share(1, 2, max_sessions=3)
    own = _tts(E, 1, max_sessions=3)
    try:
        w, t = sharer.device_bytes()
        ow, ot = own.device_bytes()
        assert w == src.device_bytes()[0] == ow and t - w == ot - ow
        (gc, gw), _ = _concurrently(E, (1, lambda: _tts_run(sharer, 3, sampling)), (0, lambda: _tts_run(src, 4, COUSIN_SAMPLING)))
        (rc, rw), _ = _concurrently(E, (1, lambda: _tts_run(own, 3, sampling)), (0, lambda: _tts_run(src, 4, COUSIN_SAMPLING)))
        assert np.array_equal(gc, rc)
        assert len(gw) == len(rw) and all(np.array_equal(a, b) for a, b in zip(gw, rw))
        cfg = E._lib.Qwen3TTSConfig.from_buffer_copy(src.cfg)
        cfg.codec.precision = 1 - cfg.codec.precision
        h = C.c_void_p()
        lib = E._lib.load()
        assert lib.s2s_qwen3tts_create_shared(E.get_context(0, 1, 2), src.handle, C.byref(cfg), C.byref(h)) == S2S_ERR_INVALID
        assert b"precision" in lib.s2s_last_error()
        assert lib.s2s_qwen3tts_finalize(sharer.handle) == S2S_ERR_INVALID
    finally:
        for e in (src, sharer, own):   # the source first: the sharer's weights outlive it
            e.close()


def test_tts_accounting_returns_to_baseline(E):
    base = E.allocated_bytes()
    src = _tts(E, 0, max_sessions=2)
    sw, st = src.device_bytes()
    assert E.allocated_bytes() - base == st
    sharer = src.share(1, 2, max_sessions=4)
    w, t = sharer.device_bytes()
    assert w == sw and E.allocated_bytes() - base == st + (t - w)
    src.close()
    assert E.allocated_bytes() - base == t - w + w
    sharer.close()
    assert E.allocated_bytes() == base


# ---- the real geometry: one Llama-3-8B store for two 66-CTA lanes ------------------------------------------------------
def test_llama3_8b_two_lanes_share_one_store(E):
    g = W.LLAMA_GEOMETRIES["llama-3-8b"].to_dict()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("two 66-CTA lanes need a 132-SM H100")
    src = E.LlamaEngine(g, max_sessions=16, max_positions=1024, max_prefill=64, lane=0, lanes=2)
    src.init_random(1)
    sharer = src.share(1, 2)
    own = E.LlamaEngine(g, max_sessions=16, max_positions=1024, max_prefill=64, lane=1, lanes=2)   # never loaded: state only
    try:
        assert src.max_decode_batch() == 16 and sharer.max_decode_batch() == 16
        w, t = sharer.device_bytes()
        assert w == src.device_bytes()[0]
        ow, ot = own.device_bytes()
        own.close()
        assert t - w == ot - ow

        def step(eng):
            for s in range(16):
                eng.reset(s)
            first = eng.prefill_batch(list(range(16)), [[1 + s, 2, 3] for s in range(16)])
            return eng.decode(list(range(16)), first, 2)[0].cpu().numpy()
        a, b = _concurrently(E, (0, lambda: step(src)), (1, lambda: step(sharer)))
        assert np.array_equal(a, b)   # same weights, same prompts
    finally:
        for e in (src, sharer, own):
            e.close()
