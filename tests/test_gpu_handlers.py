"""GPU: the handlers end to end on an H100 (mirror runtime when the reference tree is absent), and the TTS
post-processing kernel against scipy (bit-exact int16)."""
from queue import Queue
from threading import Event, Thread

import numpy as np
import pytest
import torch

from oracle import weights as W, whisper_ref as WR, llama_ref as LR, tts_post_ref as T

pytestmark = pytest.mark.gpu


def test_whisper_handler_random_model_through_stage_loop():
    from speech_to_speech_b200.host import resolve
    from speech_to_speech_b200.handlers.whisper_stt_handler import B200WhisperSTTHandler
    api = resolve()
    qi, qo, stop = Queue(), Queue(), Event()
    h = B200WhisperSTTHandler(stop, queue_in=qi, queue_out=qo,
                              setup_kwargs={"model_name": "random:tiny:3", "device": "cuda", "torch_dtype": "float16",
                                            "language": "en", "gen_kwargs": {"max_new_tokens": 12, "task": "transcribe"}})
    th = Thread(target=h.run)
    th.start()
    audio = W.synthetic_audio(4, 48000)
    item = api.VADAudio(audio=audio, mode="final", turn_id="a", turn_revision=1)
    qi.put(item)
    out = qo.get(timeout=60)
    assert isinstance(out, api.Transcription) and out.language_code == "en" and out.turn_id == "a"
    assert out.speech_stopped_at_s == item.created_at_s
    ids = [int(t.strip("<>")) for t in out.text.split()]
    assert 1 <= len(ids) <= 12 and all(0 <= i < 51865 for i in ids)
    # same utterance twice -> identical ids (deterministic), progressive mode -> PartialTranscription
    qi.put(api.VADAudio(audio=audio, mode="progressive", turn_id="a", turn_revision=2))
    out2 = qo.get(timeout=60)
    assert isinstance(out2, api.PartialTranscription) and out2.text == out.text
    qi.put(api.PIPELINE_END)
    assert qo.get(timeout=10) == api.PIPELINE_END
    th.join(timeout=10)


def test_concurrent_sessions_share_one_engine_and_match_the_single_session_path():
    """6 pipeline units (handler instances) with max_batch=8: one shared engine, their utterances ride one launch;
    every session's ids equal what the one-session handler produces for the same audio."""
    from speech_to_speech_b200.host import resolve
    from speech_to_speech_b200.handlers.whisper_stt_handler import B200WhisperSTTHandler
    api = resolve()
    kw = {"model_name": "random:tiny:3", "device": "cuda", "torch_dtype": "float16", "language": "en",
          "gen_kwargs": {"max_new_tokens": 10, "task": "transcribe"}}
    single = B200WhisperSTTHandler(Event(), queue_in=Queue(), queue_out=Queue(), setup_kwargs=dict(kw))
    auds = [W.synthetic_audio(40 + i, 32000 + 16000 * (i % 3)) for i in range(6)]
    want = [list(single.process(api.VADAudio(audio=a, mode="final")))[0].text for a in auds]
    single.cleanup()
    units = [B200WhisperSTTHandler(Event(), queue_in=Queue(), queue_out=Queue(),
                                   setup_kwargs=dict(kw, max_batch=8, batch_wait_ms=200.0)) for _ in range(6)]
    assert all(u.bundle is units[0].bundle for u in units)  # ONE engine, one copy of the weights
    got = {}

    def session(i):
        got[i] = list(units[i].process(api.VADAudio(audio=auds[i], mode="final")))[0].text

    before = units[0].bundle.batcher.batches_run
    ths = [Thread(target=session, args=(i,)) for i in range(6)]
    [t.start() for t in ths]
    [t.join(120) for t in ths]
    assert [got[i] for i in range(6)] == want
    b = units[0].bundle.batcher
    assert b.largest_batch >= 2 and b.batches_run - before < 6
    for u in units:
        u.cleanup()


def test_whisper_handler_auto_language_reports_detected_code():
    from speech_to_speech_b200.host import resolve
    from speech_to_speech_b200.handlers.whisper_stt_handler import B200WhisperSTTHandler
    api = resolve()
    h = B200WhisperSTTHandler(Event(), queue_in=Queue(), queue_out=Queue(),
                              setup_kwargs={"model_name": "random:tiny:3", "device": "cuda", "language": "auto",
                                            "gen_kwargs": {"max_new_tokens": 4}})
    out = list(h.process(api.VADAudio(audio=W.synthetic_audio(5, 32000), mode="final")))[0]
    assert out.language_code.endswith("-auto") and out.language_code[:-5] in h.tokens.lang_to_id


def test_llm_token_streamer_matches_oracle_ids():
    from speech_to_speech_b200 import engine as E
    from speech_to_speech_b200.handlers.language_model_handler import TokenStreamer
    g = W.LLAMA_GEOMETRIES["micro"]
    w = W.make_llama_weights(g, 0)
    eng = E.LlamaEngine(g.to_dict(), dtype="float16", max_positions=256, max_prefill=16)
    eng.load_state_dict(w)
    prompt = np.random.default_rng(11).integers(0, g.vocab, 37)
    ref, lg = LR.greedy_generate(w, g, prompt, 20, return_logits=True)
    srt = np.sort(lg, axis=1)
    safe = (srt[:, -1] - srt[:, -2]) > 0.05
    k = int(np.argmin(safe)) if (~safe).any() else len(ref)
    st = TokenStreamer(eng, lambda ids: "".join(f"<{i}> " for i in ids), [g.vocab + 5], chunk=6)
    text = "".join(st.stream(prompt.tolist(), 20))
    assert st.generated[:k] == ref[:k] and len(st.generated) == 20
    assert text == "".join(f"<{i}> " for i in st.generated)


def test_llm_handlers_share_one_engine_and_merge_decode_chunks():
    """3 pipeline units with gen_kwargs max_sessions=3: ONE engine (one weight copy, 3 KV slots); the decode chunks of the
    concurrent sessions ride multi-session launches; results are reproducible and start like the single-session path."""
    from speech_to_speech_b200.handlers.language_model_handler import B200LanguageModelHandler

    def make(**kw):
        h = object.__new__(B200LanguageModelHandler)
        h._load_model("random:micro:5", "cuda", "float16", dict({"max_new_tokens": 24, "stream_chunk_tokens": 6, "max_positions": 256}, **kw))
        return h

    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, 2048, 9 + 5 * i).tolist() for i in range(3)]
    single = make()
    want = []
    for p in prompts:
        "".join(single.generate_text_stream(p, 24))
        want.append(list(single.streamer.generated))
    single.cleanup()
    units = [make(max_sessions=3, batch_wait_ms=200.0) for _ in range(3)]
    assert all(u.bundle is units[0].bundle for u in units) and sorted(u.slot for u in units) == [0, 1, 2]
    runs = []
    for _ in range(2):
        got = {}

        def session(i):
            "".join(units[i].generate_text_stream(prompts[i], 24))
            got[i] = list(units[i].streamer.generated)

        ths = [Thread(target=session, args=(i,)) for i in range(3)]
        [t.start() for t in ths]
        [t.join(120) for t in ths]
        runs.append([got[i] for i in range(3)])
    assert runs[0] == runs[1]                                     # same launches -> same ids
    for i in range(3):
        assert len(runs[0][i]) >= 4 and runs[0][i][:4] == want[i][:4]
    assert units[0].bundle.batcher.largest_batch >= 2
    for u in units:
        u.cleanup()


@pytest.mark.parametrize("n", [1, 2, 3, 100, 1919, 1920, 15360, 48001])
def test_tts_postproc_is_bit_exact_vs_scipy(n):
    from speech_to_speech_b200.handlers.qwen3_tts_postproc import TTSPostProcessor
    rng = np.random.default_rng(n)
    t = np.arange(n) / 24000.0
    x = (0.6 * np.sin(2 * np.pi * 220 * t) * np.minimum(1.0, t * 20) + 0.02 * rng.standard_normal(n)).astype(np.float32)
    x[::97] *= 3.0  # some samples clip
    got = TTSPostProcessor(0)(x)
    ref = T.postproc(x)
    assert got.dtype == np.int16 and got.shape == ref.shape
    assert np.array_equal(got, ref)


def test_tts_stream_blocks_with_gpu_postproc_match_reference_logic():
    """Leading-silence trim + 512-sample re-blocking (reference _stream) on top of the GPU resample/int16."""
    from speech_to_speech_b200.handlers.qwen3_tts_postproc import TTSPostProcessor
    post = TTSPostProcessor(0)
    rng = np.random.default_rng(0)
    chunks = [np.zeros(15360, np.float32), (0.001 * rng.standard_normal(15360)).astype(np.float32)]
    chunks += [(0.3 * np.sin(np.arange(15360) * 0.03 + i)).astype(np.float32) for i in range(3)]
    ref = T.stream_blocks(chunks, 512)
    found, leftover, out = False, np.array([], np.int16), []
    for c in chunks:
        a = post(c)
        if not found:
            above = np.abs(a) > int(32768 * 0.01)
            if not above.any():
                continue
            a = a[max(0, int(np.argmax(above)) - 640):]
            found = True
        a = np.concatenate([leftover, a])
        k = (len(a) // 512) * 512
        out += [a[i:i + 512] for i in range(0, k, 512)]
        leftover = a[k:]
    if len(leftover):
        out.append(np.pad(leftover, (0, 512 - len(leftover))))
    assert len(out) == len(ref) and all(np.array_equal(a, b) for a, b in zip(out, ref))
