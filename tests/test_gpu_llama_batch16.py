"""GPU: 16 Llama-3-8B-shaped sessions in ONE decode launch (the third shared-memory tier of llama_decode_plan: no fp32
statistics copy, RMSNorm rows read from L2 into registers).  The launch keeps the reduction orders of an 8-session launch
(assoc_b), so every session's ids and logits are bit-identical to the same sessions decoded as 8 + 8 -- greedy, sampled,
and on two concurrent lanes -- and match the oracle.  The attention split plan follows the launch's longest session, so
both halves of every batch here hold a session of the longest prompt."""
import os
import threading

import numpy as np
import pytest
import torch

from oracle import weights as W, llama_ref as R

pytestmark = pytest.mark.gpu
TOL = {"float16": 2.5e-2, "bfloat16": 0.2}       # tests/test_gpu_llama.py
LENS = [150, 12, 40, 133, 70, 5, 99, 31, 150, 20, 64, 131, 7, 88, 145, 33]   # > 128: five key blocks at the first step
STEPS = 12
SAMPLED = {1: dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.9, seed=11),
           4: dict(do_sample=True, temperature=1.1, top_k=0, top_p=0.7, seed=12),
           9: dict(do_sample=True, temperature=0.7, top_k=20, top_p=1.0, repetition_penalty=1.2, seed=13),
           6: dict(repetition_penalty=1.3), 14: dict(do_sample=True, temperature=1.0, top_k=50, top_p=0.95, seed=14)}


@pytest.fixture(scope="module")
def geo():
    g = W.LLAMA_GEOMETRIES["llama-3-8b-2l"]
    w = W.make_llama_weights(g, 0)
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, g.vocab, n) for n in LENS]
    return g, w, prompts


def _engine(geo, dtype, lane=0, lanes=1):
    from speech_to_speech_b200 import engine as E
    g, w, _ = geo
    eng = E.LlamaEngine(g.to_dict(), dtype=dtype, max_sessions=16, max_positions=256, max_prefill=256, lane=lane, lanes=lanes)
    eng.load_state_dict(w)
    return eng


def _prefill(eng, prompts, sampling=None):
    firsts = []
    for s, p in enumerate(prompts):
        eng.reset(s)
        if sampling and s in sampling:
            eng.set_sampling(s, **sampling[s])
        firsts.append(int(eng.prefill(s, p.tolist())[0][0]))
    return torch.tensor(firsts, dtype=torch.int32, device="cuda")


def _decode(eng, slots, first, forced=None):
    f = None if forced is None else forced.contiguous()
    ids, _, lg = eng.decode(slots, first.contiguous(), STEPS, forced=f, return_logits=True)
    return ids.cpu().numpy(), lg.cpu().numpy()


def _one_vs_halves(eng, prompts, sampling=None):
    """(ids, logits) of one 16-session launch and of the same sessions decoded as 8 + 8, each after a fresh prefill"""
    first = _prefill(eng, prompts, sampling)
    one = _decode(eng, list(range(16)), first)
    first = _prefill(eng, prompts, sampling)
    a = _decode(eng, list(range(8)), first[:8])
    b = _decode(eng, list(range(8, 16)), first[8:])
    halves = (np.concatenate([a[0], b[0]], axis=0), np.concatenate([a[1], b[1]], axis=1))
    return one, halves


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_sixteen_sessions_equal_eight_plus_eight(geo, dtype):
    eng = _engine(geo, dtype)
    try:
        assert eng.max_decode_batch() == 16
        one, halves = _one_vs_halves(eng, geo[2])
        assert np.array_equal(one[0], halves[0]) and np.array_equal(one[1], halves[1])
        one, halves = _one_vs_halves(eng, geo[2], SAMPLED)
        assert np.array_equal(one[0], halves[0]) and np.array_equal(one[1], halves[1])
    finally:
        eng.close()


ORACLE_SESSIONS = (0, 3, 5, 8, 11, 14)   # both halves, the longest and the shortest prompts
N_ORACLE = 4


@pytest.fixture(scope="module")
def refs(geo):
    g, w, prompts = geo
    return {s: R.greedy_generate(w, g, prompts[s], N_ORACLE, return_logits=True) for s in ORACLE_SESSIONS}


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_sixteen_sessions_match_oracle(geo, refs, dtype):
    """teacher-forced along the oracle's greedy ids (the other sessions along arbitrary ids): the logits of sessions from both
    halves within the tolerance of tests/test_gpu_llama.py"""
    eng = _engine(geo, dtype)
    try:
        first = _prefill(eng, geo[2]).cpu().numpy()
        forced = np.zeros((16, N_ORACLE - 1), dtype=np.int32)
        for s, r in refs.items():
            first[s], forced[s] = r[0][0], r[0][1:]
        _, _, lg = eng.decode(list(range(16)), torch.from_numpy(first).cuda(), N_ORACLE - 1, forced=torch.from_numpy(forced).cuda(),
                              return_logits=True)
        lg = lg.cpu().numpy()
    finally:
        eng.close()
    for s, r in refs.items():
        assert np.abs(lg[:, s] - r[1][1:]).max() < TOL[dtype], s


def test_sixteen_sessions_two_lanes(geo):
    """both SM partitions decode 16 sessions at once (66 CTAs each on an H100), each equal to its own 8 + 8"""
    prompts = geo[2]
    from speech_to_speech_b200 import engine as E
    lanes = [_engine(geo, "bfloat16", lane=i, lanes=2) for i in range(2)]
    got = {}
    try:
        assert all(e.max_decode_batch() == 16 for e in lanes)

        def run(i):
            with E.lane_context(0, i, 2):
                got[i] = _one_vs_halves(lanes[i], prompts, SAMPLED if i else None)
                torch.cuda.current_stream().synchronize()
        th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        [t.start() for t in th]
        [t.join() for t in th]
    finally:
        for e in lanes:
            e.close()
    for i in range(2):
        one, halves = got[i]
        assert np.array_equal(one[0], halves[0]) and np.array_equal(one[1], halves[1]), i


def test_sixteen_sessions_persistent_equals_debug_phases(geo):
    """the cooperative launch (grid barriers, look-ahead across them) against one launch per phase, bit for bit"""
    out = []
    for dbg in ("0", "1"):
        os.environ["S2S_DEBUG_PHASES"] = dbg
        try:
            eng = _engine(geo, "bfloat16")
        finally:
            os.environ.pop("S2S_DEBUG_PHASES", None)
        try:
            first = _prefill(eng, geo[2], SAMPLED)
            out.append(_decode(eng, list(range(16)), first))
        finally:
            eng.close()
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
