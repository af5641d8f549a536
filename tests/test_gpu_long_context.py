"""GPU tests (H100) of the engines at their cache limits, against the numpy oracles.

Llama family at max_positions = 4096 with prefill chunks of 512 (the LLM handler's defaults): what the kernel-level
attention tests (test_gpu_attention.py) cannot see -- RoPE at high positions, the KV append, the Qwen3 own-key path, split
plans that change in the middle of a launch, sessions of very different lengths in one launch, and the engine's position
bookkeeping.  Logit tolerances are those of test_gpu_llama.py (fp16 2.5e-2, bf16 0.2).

Whisper at max_target_positions = 448 (n_prefix + max_new = 448): the decoder's self-attention phase is its own code
(whisper_decode.cu: a split plan per key-block count, and the thread-block-cluster kernel's record merge at one session),
run here over all 14 key blocks, at one session (cluster kernel) and three.  Logit tolerance that of test_gpu_whisper.py
(2e-3)."""
import functools

import numpy as np
import pytest
import torch

from oracle import weights as W, llama_ref as R, whisper_ref as WR

pytestmark = pytest.mark.gpu
TOL = {"float16": 2.5e-2, "bfloat16": 0.2}
MAX_POS, CHUNK = 4096, 512
S2S_ERR_INVALID = -1


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@functools.lru_cache(maxsize=None)
def _weights(name):
    g = W.LLAMA_GEOMETRIES[name]
    return g, W.make_llama_weights(g, 0)


@functools.lru_cache(maxsize=None)
def _oracle(name, n_prompt, n_feed, seed):
    """A random prompt of n_prompt ids, then n_feed greedy ids fed one by one.  -> (prompt, prompt logits [n_prompt, V],
    ids [n_feed + 1] (ids[0] = the prompt's choice), logits [n_feed + 1, V] (row i predicts ids[i]))."""
    g, w = _weights(name)
    prompt = np.random.default_rng(seed).integers(0, g.vocab, n_prompt)
    cache = R.KVCache(g)
    pre = R.forward(w, g, prompt, cache)
    ids, lg = [int(np.argmax(pre[-1]))], [pre[-1]]
    for _ in range(n_feed):
        row = R.forward(w, g, np.asarray([ids[-1]]), cache)[-1]
        ids.append(int(np.argmax(row)))
        lg.append(row)
    return prompt, pre, np.asarray(ids), np.stack(lg)


def _engine(E, name, dtype, sessions=1, **kw):
    g, w = _weights(name)
    eng = E.LlamaEngine(g.to_dict(), dtype=dtype, max_sessions=sessions, max_positions=MAX_POS, max_prefill=CHUNK, **kw)
    eng.load_state_dict(w)
    return eng


def _prefill_chunks(eng, slot, prompt, pre, tol):
    """The handler's chunked prefill; the last row of every chunk against the oracle."""
    for o in range(0, len(prompt), CHUNK):
        n = min(CHUNK, len(prompt) - o)
        _, lg = eng.prefill(slot, prompt[o: o + n].tolist(), return_logits=True)
        err = np.abs(lg[-1].cpu().numpy() - pre[o + n - 1]).max()
        assert err < tol, f"prefill chunk at {o}: max |err| {err:.3g}"


def _decode_forced(eng, slots, ids, lgs, a, b, tol):
    """Feed ids[s][a:b] of every session in one launch (teacher-forced); logits against the oracle rows a+1 .. b."""
    first = torch.tensor([int(x[a]) for x in ids], dtype=torch.int32, device="cuda")
    forced = torch.tensor(np.stack([x[a + 1: b + 1] for x in ids]), dtype=torch.int32, device="cuda")
    _, _, logits = eng.decode(slots, first, b - a, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()
    for s in range(len(slots)):
        err = np.abs(lg[:, s] - lgs[s][a + 1: b + 1]).max(axis=1)
        assert err.max() < tol, f"session {s}: step {a + int(err.argmax())}: max |err| {err.max():.3g}"
    return lg


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", ["micro", "qwen3-micro"])
def test_long_prompt_then_decode_to_the_last_position(E, name, dtype):
    """3600-token prompt in 512-token chunks, then teacher-forced decode in three launches until the cache holds exactly
    max_positions keys; one step more is refused and leaves the engine usable: the slot, reset, serves a short prompt
    again (nothing of its 4096 stale rows may be read)."""
    tol = TOL[dtype]
    n_prompt, n_feed = 3600, MAX_POS - 3600
    prompt, pre, ids, lgs = _oracle(name, n_prompt, n_feed, 1)
    eng = _engine(E, name, dtype)
    _prefill_chunks(eng, 0, prompt, pre, tol)
    for a, b in ((0, 200), (200, 400), (400, n_feed)):
        _decode_forced(eng, [0], [ids], [lgs], a, b, tol)
    from speech_to_speech_b200._lib import S2SError
    with pytest.raises(S2SError, match=rf"\({S2S_ERR_INVALID}\).*exceed max_positions"):   # check() reports "(rc)"
        eng.decode([0], torch.tensor([int(ids[n_feed])], dtype=torch.int32, device="cuda"), 1)
    eng.reset(0)
    p2, pre2, ids2, lgs2 = _oracle(name, 40, 8, 2)
    _prefill_chunks(eng, 0, p2, pre2, tol)
    _decode_forced(eng, [0], [ids2], [lgs2], 0, 8, tol)


@pytest.mark.parametrize("lanes", [1, 2])
def test_sessions_of_3900_700_33_and_5_tokens_in_one_launch(E, lanes):
    """Four sessions of very different lengths decode together (the split plan follows the longest; the shorter sessions
    get empty splits), on the whole grid and on one of two lanes (66 CTAs)."""
    lens, n_feed, tol = (3900, 700, 33, 5), 6, TOL["float16"]
    runs = [_oracle("micro", n, n_feed, 10 + i) for i, n in enumerate(lens)]
    with E.lane_context(0, 0, lanes):
        eng = _engine(E, "micro", "float16", sessions=len(lens), lane=0, lanes=lanes)
        for s, (prompt, pre, _, _) in enumerate(runs):
            _prefill_chunks(eng, s, prompt, pre, tol)
        _decode_forced(eng, list(range(len(lens))), [r[2] for r in runs], [r[3] for r in runs], 0, n_feed, tol)
        torch.cuda.current_stream().synchronize()
        eng.close()


def test_qwen3_long_context_persistent_equals_debug_phases(E, monkeypatch):
    """Qwen3 at ~3900 positions next to a short session: the persistent launch and the one-launch-per-phase debug mode
    agree bit for bit, and both match the oracle."""
    lens, n_feed, tol = (3900, 70), 5, TOL["float16"]
    runs = [_oracle("qwen3-micro", n, n_feed, 20 + i) for i, n in enumerate(lens)]
    outs = []
    for dbg in ("0", "1"):
        monkeypatch.setenv("S2S_DEBUG_PHASES", dbg)
        eng = _engine(E, "qwen3-micro", "float16", sessions=2)
        for s, (prompt, pre, _, _) in enumerate(runs):
            _prefill_chunks(eng, s, prompt, pre, tol)
        outs.append(_decode_forced(eng, [0, 1], [r[2] for r in runs], [r[3] for r in runs], 0, n_feed, tol).copy())
        eng.close()
    assert np.array_equal(outs[0], outs[1])


WHISPER_TOL = 2e-3
WHISPER_PREFIX, WHISPER_SUPPRESS = [4000, 4001, 4002, 4003], [1, 2, 7, 8, 9, 10, 14, 25, 4000, 4001]


@pytest.mark.parametrize("B", [1, 3])
def test_whisper_decode_to_max_target_positions(E, monkeypatch, B):
    """Whisper micro, n_prefix + max_new = max_target_positions = 448, teacher-forced along the oracle's greedy tokens on
    the engine's own encoder output: logits of all 444 steps against whisper_ref, the forced run's argmax equal to the
    oracle's wherever its top-1 margin exceeds 4x the tolerance.  B = 1 runs the cluster kernel, B = 3 the 8-phase kernel."""
    monkeypatch.setenv("S2S_WHISPER_CLUSTER", "1")
    g = W.WHISPER_GEOMETRIES["micro"]
    w = W.make_whisper_weights(g, 0)
    max_new = g.max_target_positions - len(WHISPER_PREFIX)
    eng = E.WhisperEngine(g.to_dict(), dtype="float16", max_batch=B)
    eng.load_state_dict(w)
    auds = [W.synthetic_audio(40 + b, 160000) for b in range(B)]
    eng.logmel(torch.from_numpy(np.stack(auds)).cuda(), [len(a) for a in auds])
    enc = eng.encode(B, return_output=True).cpu().numpy()
    opts = E.WhisperDecodeOptions(prefix=WHISPER_PREFIX, eos_id=-1, max_new_tokens=max_new, suppress=WHISPER_SUPPRESS,
                                  begin_suppress=[220, g.vocab - 1])
    refs = [WR.greedy_decode(w, g, enc[b], WHISPER_PREFIX, max_new, -1, WHISPER_SUPPRESS, [220, g.vocab - 1],
                             return_logits=True) for b in range(B)]
    forced = torch.tensor([r[0] for r in refs], dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode(B, opts, forced=forced, return_logits=True)
    ids, lg = ids.cpu().numpy(), logits.cpu().numpy()
    assert (lens.cpu().numpy() == max_new).all()
    for b, (ref_ids, lg_ref) in enumerate(refs):
        fin = np.isfinite(lg_ref)
        assert (np.isfinite(lg[:, b]) == fin).all(), f"session {b}: suppressed ids differ"
        err = np.where(fin, np.abs(np.nan_to_num(lg[:, b] - lg_ref, posinf=0, neginf=0)), 0).max(axis=1)
        assert err.max() < WHISPER_TOL, f"session {b}: step {int(err.argmax())}: max |err| {err.max():.3g}"
        srt = np.sort(lg_ref, axis=1)
        safe = (srt[:, -1] - srt[:, -2]) > 4 * WHISPER_TOL
        print(f"\nwhisper B={B} session {b}: max |err| {err.max():.2e}, {int(safe.sum())} of {max_new} ids checked")
        assert safe.sum() >= max_new // 2 and (ids[b][safe] == np.asarray(ref_ids)[safe]).all(), f"session {b}"
    eng.close()
