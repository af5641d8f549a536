"""GPU parity tests (H100) of the TTS talker + code predictor (csrc/qwen3tts.cu) through the C ABI: codebook ids
bit-exact against the numpy oracle (oracle/qwen3tts_ref.py) and the golden codes generated from the transformers
cousin; sessions batched in one launch equal the single-session results.  Unpinned vs faster-qwen3-tts (absent)."""
import os

import numpy as np
import pytest
import torch

from oracle import code2wav_ref as C, qwen3tts_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _engine(E, dtype="float16", **kw):
    g, cg = R.GEOMETRIES["micro"], C.GEOMETRIES["micro"]
    cg = C.Code2WavGeometry(**{**cg.to_dict(), "quantizers": g.n_groups, "codebook_size": g.predictor.vocab,
                               "upsample_rates": tuple(cg.upsample_rates), "upsampling_ratios": tuple(cg.upsampling_ratios)})
    w, cw = R.make_weights(g, 0), C.make_weights(cg, 0)
    eng = E.Qwen3TTSEngine(g.to_dict(), cg.to_dict(), dtype=dtype, max_positions=128, max_text=64, codec_precision=0, **kw)
    eng.load_state_dict(w, cw)
    return g, cg, w, cw, eng


# logits tolerances of the 16-bit engines (the same figures as tests/test_gpu_llama.py); a decision is "safe" when the oracle's
# top-1 margin exceeds 4x the tolerance.  Random-init heads give margins of O(1), so most -- not all -- decisions are safe.
TOL = {"float16": 2.5e-2, "bfloat16": 0.2}


def _margins(t_logits, p_logits):
    """[F] talker margins and [F, G-1] predictor margins (top-1 minus top-2 of the processed logits)."""
    def m(x):
        s = np.sort(np.where(np.isfinite(x), x, -1e30), axis=-1)
        return s[..., -1] - s[..., -2]
    return m(t_logits), m(p_logits)


def _check_forced(eng, slot_codes, slots, tol, min_safe_frac):
    """Teacher-forced run along the oracle's codes: every one of the 16 x F decisions is compared where it is safe.
    slot_codes: list of (codes [F, G], talker_logits [>=F, V], predictor_logits [F, G-1, Vp]) per slot."""
    F = min(len(c[0]) for c in slot_codes)
    forced = torch.tensor(np.stack([c[0][:F] for c in slot_codes]), dtype=torch.int32, device="cuda")
    got = eng.decode_frames(slots, F, forced=forced).cpu().numpy()
    n_safe = n_all = 0
    for i, (codes, tl, pl) in enumerate(slot_codes):
        mt, mp = _margins(tl[:F], pl[:F])
        safe = np.concatenate([mt[:, None], mp], axis=1) > 4 * tol       # [F, G]
        assert np.array_equal(got[i][safe], codes[:F][safe]), (i, np.argwhere(safe & (got[i] != codes[:F]))[:4])
        n_safe += int(safe.sum()); n_all += safe.size
    assert n_safe >= min_safe_frac * n_all, (n_safe, n_all)
    return got


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_codes_match_transformers_golden(E, golden_dir, dtype):
    """Codes and margins from the transformers cousin (tests/golden/qwen3tts_micro.npz): teacher-forced along the golden
    codes every safe decision is bit-exact; the free run equals the golden codes up to the first unsafe decision."""
    g, cg, w, cw, eng = _engine(E, dtype)
    G = np.load(os.path.join(golden_dir, "qwen3tts_micro.npz"))
    gold, tl, pl = G["codes"], G["talker_logits"], G["predictor_top2"]   # the margins need only each row's top two
    F = len(gold)
    eng.prefill(0, G["text_ids"].tolist(), int(G["speaker"]))
    _check_forced(eng, [(gold, tl, pl)], [0], TOL[dtype], 0.6 if dtype == "float16" else 0.2)
    mt, mp = _margins(tl[:F], pl[:F])
    safe = (np.concatenate([mt[:, None], mp], axis=1) > 4 * TOL[dtype]).all(axis=1)
    k = int(np.argmin(safe)) if (~safe).any() else F
    eng.prefill(0, G["text_ids"].tolist(), int(G["speaker"]))
    free = eng.decode_frames([0], F)[0].cpu().numpy()
    assert np.array_equal(free[:k], gold[:k])
    if k < F:   # the first unsafe frame may differ only in its unsafe codebooks' suffix: its first code is safe or equal
        assert free[k, 0] == gold[k, 0] or mt[k] <= 4 * TOL[dtype]


def test_batched_sessions_equal_oracle_and_single_runs(E):
    g, cg, w, cw, eng = _engine(E, "float16", max_sessions=4)
    rng = np.random.default_rng(3)
    texts = [rng.integers(0, 400, n).tolist() for n in (1, 3, 9, 17)]
    speakers = [2301, 2302, 2301, 2400]
    F = 7
    refs = [R.generate(w, g, t, s, F, return_logits=True) for t, s in zip(texts, speakers)]
    for slot, (t, s) in enumerate(zip(texts, speakers)):
        eng.prefill(slot, t, s)
    _check_forced(eng, refs, [0, 1, 2, 3], TOL["float16"], 0.6)
    # free run of the four sessions in one launch sequence == each session alone (same kernels, batch of 1): bit-exact
    for slot, (t, s) in enumerate(zip(texts, speakers)):
        eng.prefill(slot, t, s)
    got = eng.decode_frames([0, 1, 2, 3], F).cpu().numpy()
    for slot, (t, s) in enumerate(zip(texts, speakers)):
        eng.prefill(slot, t, s)
        alone = eng.decode_frames([slot], F)[0].cpu().numpy()
        mt, mp = _margins(refs[slot][1][:F], refs[slot][2][:F])
        safe = (np.concatenate([mt[:, None], mp], axis=1) > 4 * TOL["float16"]).all(axis=1)
        k = int(np.argmin(safe)) if (~safe).any() else F
        assert np.array_equal(got[slot][:k], refs[slot][0][:k]) and np.array_equal(alone[:k], refs[slot][0][:k]), slot
    # frames continue across calls (state lives in the library): 3 + 4 frames == 7 frames in one call
    for slot, (t, s) in enumerate(zip(texts, speakers)):
        eng.prefill(slot, t, s)
    a = eng.decode_frames([3, 1], 3).cpu().numpy()
    b = eng.decode_frames([3, 1], 4).cpu().numpy()
    eng.prefill(3, texts[3], speakers[3]); eng.prefill(1, texts[1], speakers[1])
    whole = eng.decode_frames([3, 1], 7).cpu().numpy()
    assert np.array_equal(np.concatenate([a, b], 1), whole)
    assert eng.frames(3) == 7 and eng.frames(1) == 7 and eng.frames(0) == 0   # slot 0 was re-prefilled and not decoded since


def test_persistent_launch_equals_per_phase_launches(E, monkeypatch):
    outs = []
    for dbg in ("0", "1"):
        monkeypatch.setenv("S2S_DEBUG_PHASES", dbg)
        g, cg, w, cw, eng = _engine(E, "bfloat16")
        eng.prefill(0, [5, 6, 7, 8], 2301)
        outs.append(eng.decode_frames([0], 5).cpu().numpy().copy())
        eng.close()
    assert np.array_equal(outs[0], outs[1])


def test_streaming_audio_matches_the_oracle_chunked_decode(E):
    """8-frame chunks behind 25 frames of history (the reference handler's chunk_size, S/TTS/qwen3_tts_handler.py:49):
    the concatenated chunks equal the oracle's chunked_decode of the oracle's codes."""
    g, cg, w, cw, eng = _engine(E, "float16")
    text, F, chunk, left = [11, 12, 13, 14, 15], 20, 8, 25
    codes_ref = R.generate(w, g, text, 2301, F)
    assert len(codes_ref) == F
    wav_ref = C.chunked_decode(cw, cg, codes_ref.T, chunk_size=chunk, left_context=left)
    eng.prefill(0, text, 2301)
    outs, done = [], 0
    while done < F:   # teacher-forced along the oracle's codes: the library keeps the forced codes, the codec decodes those
        n = min(chunk, F - done)
        forced = torch.tensor(codes_ref[None, done:done + n], dtype=torch.int32, device="cuda")
        eng.decode_frames([0], n, forced=forced)
        outs.append(eng.decode_audio(0, n, left).cpu().numpy())
        done += n
    got = np.concatenate(outs)
    assert got.shape == wav_ref.shape
    assert np.abs(got - wav_ref).max() < 1e-3


def test_batched_audio_decode_equals_per_session_decode(E):
    """Three speaking sessions with chunks of the same shape through ONE codec launch sequence == each alone, bit for bit
    (every output row depends on its own sequence only), in both codec precisions."""
    for prec in (0, 1):
        g, cg = R.GEOMETRIES["micro"], C.GEOMETRIES["micro"]
        cg = C.Code2WavGeometry(**{**cg.to_dict(), "quantizers": g.n_groups, "codebook_size": g.predictor.vocab,
                                   "upsample_rates": tuple(cg.upsample_rates), "upsampling_ratios": tuple(cg.upsampling_ratios)})
        eng = E.Qwen3TTSEngine(g.to_dict(), cg.to_dict(), dtype="float16", max_sessions=3, max_positions=128, max_text=64,
                               codec_precision=prec)
        eng.load_state_dict(R.make_weights(g, 0), C.make_weights(cg, 0))
        for slot, text in enumerate(([1, 2, 3], [9, 8], [4, 4, 4, 4])):
            eng.prefill(slot, text, 2301)
        for n in (8, 8, 5):     # history 0, 8, 16 frames behind the chunk
            eng.decode_frames([0, 1, 2], n)
            together = [w.cpu().numpy().copy() for w in eng.decode_audio_batch([0, 1, 2], n, 25)]
            for slot in range(3):
                alone = eng.decode_audio(slot, n, 25).cpu().numpy()
                assert np.array_equal(alone, together[slot]), (prec, n, slot)
        eng.close()
