"""numpy restatement of sampled Qwen3-TTS decoding (test infrastructure for tests/test_*tts_sampling*.py).

The token choice is oracle/sampling_ref.py's (transformers' logits-processor order: repetition penalty, then temperature,
top-k, top-p and a Gumbel-max draw), extended by the third Philox counter word the device uses, `stream`:
u(seed, position, id, stream) is the first raw output of numpy.random.Philox(key=seed, counter=[id, position, stream, 0]).
The LLM and the Qwen3-TTS talker draw from stream 0 (oracle/sampling_ref.py's stream); the code predictor, whose positions
repeat every frame, from stream 1 + the frame's index since prefill.

The frame loop is oracle/qwen3tts_ref.py's (prompt, talker and code-predictor arithmetic reused from there) with each
decision made by `choose`:
  talker     first code of frame f at talker position 9 + f (the 9 prompt rows occupy 0..8), stream 0, suppressed ids -inf,
             repetition penalty over the first codes of the frames kept so far -- the cousin calls talker.generate without
             input_ids (modeling_qwen3_omni_moe.py:4064-4068), so the prompt's codec ids are not penalised;
  predictor  code i (1..n_groups-1) of frame f at predictor position i + 1 ([talker hidden, code0] occupy 0 and 1),
             stream 1 + f, no repetition penalty.
tests/test_oracle_tts_sampling.py pins the processors against the transformers cousin driven with its own sampling
arguments (talker T 0.9 / top-k 50 / top-p 1.0 / penalty 1.05, predictor top-k 50 / top-p 0.8 at T 1.0)."""
from __future__ import annotations

import numpy as np

from oracle import llama_ref as L
from oracle import qwen3tts_ref as R
from oracle import sampling_ref as S


# ------------------------------------------------------------------------------------------------ the token choice
def uniforms(seed: int, position: int, n: int, stream: int = 0) -> np.ndarray:
    """u for token ids 0..n-1: consecutive ids are consecutive Philox counters, so one generator yields all."""
    g = np.random.Philox(key=int(seed) & ((1 << 64) - 1), counter=[0, int(position), int(stream), 0])
    raw = g.random_raw(4 * n)[::4]
    return (raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def uniform_one(seed: int, position: int, token: int, stream: int = 0) -> float:
    raw = np.random.Philox(key=int(seed) & ((1 << 64) - 1), counter=[int(token), int(position), int(stream), 0]).random_raw()
    return float(int(raw) >> 11) * (1.0 / 9007199254740992.0)


def choose(z, position, seed=0, seen=(), penalty=1.0, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, stream=0):
    """-> (token, processed row, scores): sampling_ref.choose with the draw taken from `stream`."""
    w = S.process(z, seen, penalty, (), False, do_sample, temperature, top_k, top_p)
    if not do_sample:
        s = w.astype(np.float64)
    else:
        with np.errstate(divide="ignore"):
            s = w.astype(np.float64) - np.log(-np.log(uniforms(seed, position, w.shape[0], stream)))
    return int(np.argmax(s)), w, s


def margin(z, position, **kw) -> float:
    """sampling_ref.margin for `choose`: the winner gap of the scores and, when sampling, the distance of the top-k value
    and of the top-p cumulative mass to their cut-offs."""
    tok, w, s = choose(z, position, **kw)
    fin = np.sort(s[np.isfinite(s)])[::-1]
    gaps = [fin[0] - fin[1] if fin.shape[0] > 1 else np.inf]
    if kw.get("do_sample"):
        base = S.process(z, kw.get("seen", ()), kw.get("penalty", 1.0), (), False, True, kw.get("temperature", 1.0))
        v = np.sort(base.astype(np.float64))[::-1]
        k = kw.get("top_k", 0)
        if 0 < k < v.shape[0]:
            gaps += [v[k - 1] - v[k]] if v[k - 1] != v[k] else []
            v = v[v >= v[k - 1]]
        tp = kw.get("top_p", 1.0)
        if tp < 1.0:
            p = np.exp(v - v[0]); p /= p.sum()
            gaps.append(float(np.min(np.abs(np.cumsum(p) - tp))))
    return float(min(gaps))


def choose_kw(cfg) -> dict:
    """`choose` keywords of a talker / predictor sampling dict (the keywords of Qwen3TTSEngine.set_sampling; None = greedy)."""
    cfg = dict(cfg or {})
    return dict(penalty=cfg.get("repetition_penalty", 1.0), do_sample=bool(cfg.get("do_sample", False)),
                temperature=cfg.get("temperature", 1.0), top_k=cfg.get("top_k", 0), top_p=cfg.get("top_p", 1.0))


def talker_position(f: int) -> int:
    return 9 + f


def predictor_position(i: int) -> int:
    return i + 1


# ------------------------------------------------------------------------------------------------ the frame loop
def _residual_codes(w, g, past_hidden, code0, select, forced):
    """qwen3tts_ref.predict_residual_codes with select(i, logits) -> code i + 1 and optional forced feedback."""
    wv, gg = R.predictor_view(w), g.predictor
    cache = L.KVCache(gg)
    e0 = w["model.codec_embedding.weight"][code0]
    _, xn = R._decoder(wv, gg, np.stack([past_hidden, e0]).astype(np.float32), cache)
    codes, acc, rows = [], e0.astype(np.float32).copy(), []
    h = xn[-1]
    for i in range(g.n_groups - 1):
        logits = (h @ w[f"code_predictor.lm_head.{i}.weight"].T).astype(np.float32)
        c = int(select(i, logits))
        codes.append(c)
        rows.append(logits)
        if forced is not None:
            c = int(forced[i])
        e = w[f"code_predictor.model.codec_embedding.{i}.weight"][c].astype(np.float32)
        acc = acc + e
        if i + 1 < g.n_groups - 1:
            _, xn = R._decoder(wv, gg, e[None], cache)
            h = xn[-1]
    return codes, acc, np.stack(rows)


def _run(w, g, text_ids, speaker_id, max_frames, sampling, seed, forced, record):
    wv, gg = R.talker_view(w), g.talker
    sampling = sampling or {}
    tkw, pkw = choose_kw(sampling.get("talker")), choose_kw(sampling.get("predictor"))
    embeds, trailing, pad = R.build_prompt(w, g, text_ids, speaker_id)
    mask = np.zeros(gg.vocab, bool)
    mask[R.suppress_ids(g)] = True
    cache = L.KVCache(gg)
    logits, xn = R._decoder(wv, gg, embeds, cache)
    frames, seen = [], []
    for f in range(max_frames):
        lg = np.where(mask, -np.inf, logits[-1]).astype(np.float32)
        pos = talker_position(f)
        code0 = choose(lg, pos, seed=seed, seen=list(seen), **tkw)[0]
        record.append(dict(frame=f, group=0, row=lg, position=pos, stream=0, seen=frozenset(seen), choice=code0, kw=tkw))
        if forced is None and code0 == g.codec_eos:
            break
        kept0 = code0 if forced is None else int(forced[f][0])

        def select(i, row, f=f):
            c = choose(row, predictor_position(i + 1), seed=seed, stream=1 + f, **pkw)[0]
            record.append(dict(frame=f, group=i + 1, row=row, position=predictor_position(i + 1), stream=1 + f, seen=frozenset(),
                               choice=c, kw=pkw))
            return c
        res = _residual_codes(w, g, xn[-1], kept0, select, None if forced is None else forced[f][1:])
        frames.append([code0] + res[0])
        seen.append(kept0)
        nxt = res[1] + (trailing[f] if f < len(trailing) else pad)
        if f + 1 < max_frames:
            logits, xn = R._decoder(wv, gg, nxt[None].astype(np.float32), cache)
    return np.asarray(frames, np.int32).reshape(len(frames), g.n_groups)


def generate(w, g, text_ids, speaker_id: int, max_frames: int, sampling=None, seed: int = 0) -> np.ndarray:
    """Sampled talker loop -> codes [F, n_groups] (frames up to, not including, the one whose first code is codec_eos).
    sampling: {"talker": dict | None, "predictor": dict | None} with Qwen3TTSEngine.set_sampling's keywords."""
    return _run(w, g, text_ids, speaker_id, max_frames, sampling, seed, None, [])


def replay(w, g, text_ids, speaker_id: int, forced_codes, sampling=None, seed: int = 0) -> list:
    """Teacher-forced run along forced_codes [F, n_groups] (what the device's decode_frames(forced=...) feeds and keeps).
    -> one dict per decision, in order: frame, group (0 = talker), the fp32 row it was chosen from (talker: suppressed ids
    -inf), position, stream, seen (the talker's penalty set: the forced first codes of the earlier frames), choice, and kw
    (the remaining `choose` keywords)."""
    record: list = []
    _run(w, g, text_ids, speaker_id, len(forced_codes), sampling, seed, np.asarray(forced_codes), record)
    return record
