"""numpy restatement of the LLM token choice (speech_to_speech_b200/csrc/sampling.cuh), in transformers' logits-processor
order (generation/utils.py _get_logits_processor): repetition penalty, min_new_tokens EOS mask, then only when sampling
temperature, top-k, top-p and a Gumbel-max draw.  The processed values are float32 like transformers'; the top-p softmax and
the draw are float64.  The uniforms come from numpy.random.Philox itself: u(seed, position, id) is the first raw output of
Philox(key=seed, counter=[id, position, 0, 0]), mapped to [0, 1) as numpy's random() does."""
from __future__ import annotations

import numpy as np


def process(z, seen=(), penalty=1.0, eos_ids=(), mask_eos=False, do_sample=False, temperature=1.0, top_k=0, top_p=1.0):
    """The processed (greedy) or warped (sampling) float32 row; removed entries are -inf."""
    z = np.array(z, dtype=np.float32, copy=True)
    V = z.shape[0]
    if penalty != 1.0 and len(seen):
        idx = np.unique(np.asarray(list(seen), dtype=np.int64))
        s = z[idx]
        z[idx] = np.where(s < 0, s * np.float32(penalty), s / np.float32(penalty))
    if mask_eos and len(eos_ids):
        z[np.asarray(list(eos_ids), dtype=np.int64)] = -np.inf
    if not do_sample:
        return z
    z = z / np.float32(temperature)
    if 0 < top_k < V:
        kth = np.sort(z)[::-1][top_k - 1]
        z = np.where(z < kth, np.float32(-np.inf), z)
    if top_p < 1.0:
        order = np.argsort(-z.astype(np.float64), kind="stable")    # descending
        zs = z[order].astype(np.float64)
        p = np.exp(zs - zs[0])
        p /= p.sum()
        excl = np.concatenate([[0.0], np.cumsum(p)[:-1]])           # mass strictly above each entry
        keep = excl < top_p
        # ties with the last kept value are kept as well (the kernel's threshold is a value)
        thr = zs[keep][-1]
        z = np.where(z.astype(np.float64) < thr, np.float32(-np.inf), z)
    return z


def uniforms(seed: int, position: int, n: int) -> np.ndarray:
    """u for token ids 0..n-1 at `position`: consecutive ids are consecutive Philox counters, so one generator yields all."""
    g = np.random.Philox(key=int(seed) & ((1 << 64) - 1), counter=[0, int(position), 0, 0])
    raw = g.random_raw(4 * n)[::4]
    return (raw >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def uniform_one(seed: int, position: int, token: int) -> float:
    raw = np.random.Philox(key=int(seed) & ((1 << 64) - 1), counter=[int(token), int(position), 0, 0]).random_raw()
    return float(int(raw) >> 11) * (1.0 / 9007199254740992.0)


def gumbel_scores(z: np.ndarray, seed: int, position: int) -> np.ndarray:
    u = uniforms(seed, position, z.shape[0])
    with np.errstate(divide="ignore"):
        return z.astype(np.float64) - np.log(-np.log(u))


def choose(z, position, seed=0, seen=(), penalty=1.0, eos_ids=(), min_new_tokens=0, n_generated=0, do_sample=False,
           temperature=1.0, top_k=0, top_p=1.0):
    """-> (token, processed row, scores): scores are the processed row (greedy) or the Gumbel scores (sampling)."""
    w = process(z, seen, penalty, eos_ids, n_generated < min_new_tokens, do_sample, temperature, top_k, top_p)
    s = gumbel_scores(w, seed, position) if do_sample else w.astype(np.float64)
    return int(np.argmax(s)), w, s


def margin(z, position, **kw) -> float:
    """Smallest gap a float rounding would have to bridge to change the choice: the winner gap of the scores and, when
    sampling, the distance of the top-k value and of the top-p cumulative mass to their cut-offs."""
    tok, w, s = choose(z, position, **kw)
    fin = np.sort(s[np.isfinite(s)])[::-1]
    gaps = [fin[0] - fin[1] if fin.shape[0] > 1 else np.inf]
    if kw.get("do_sample"):
        base = process(z, kw.get("seen", ()), kw.get("penalty", 1.0), kw.get("eos_ids", ()),
                       kw.get("n_generated", 0) < kw.get("min_new_tokens", 0), True, kw.get("temperature", 1.0))
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
