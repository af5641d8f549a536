"""GPU: FP8 E4M3 weight-only decode of the Llama family.  With power-of-two row scales the dequantised weights dq(q(W)) are
bfloat16 numbers and the scale commutes with the fp32 accumulation, so an FP8 engine bound to W must equal, bit for bit, a
bfloat16 engine bound to dq(q(W)) (oracle/fp8_ref.py) -- prefill logits, decode ids and decode logits, greedy and sampled --
and both must match the numpy oracle on those weights.  Geometries: tiny Llama and tiny Qwen3 (qk_norm); "mini", whose
lm_head has whole main rounds and a K-split tail on a full grid; and a one-layer Llama-3-8B-shaped model with a small
vocabulary, whose down-projection operand is staged in K-chunks from 5 sessions on."""
import numpy as np
import pytest
import torch

from oracle import fp8_ref as F, weights as W, llama_ref as R

pytestmark = pytest.mark.gpu
TOL = 0.2                                            # bfloat16, tests/test_gpu_llama.py
STEPS = 32
LENS = [37, 5, 64, 12, 50, 9, 33, 21, 64, 7, 45, 18, 3, 60, 29, 14]
GEOMETRIES = dict(W.LLAMA_GEOMETRIES)
GEOMETRIES["8b-wide-1l"] = W.LlamaGeometry(4096, 1, 32, 8, 128, 14336, 2048)
SAMPLED = {0: dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.9, seed=21),
           2: dict(do_sample=True, temperature=1.1, top_k=0, top_p=0.7, repetition_penalty=1.2, seed=22),
           5: dict(repetition_penalty=1.3)}


@pytest.fixture(scope="module", params=["micro", "qwen3-micro", "mini", "8b-wide-1l"])
def pair(request):
    """(geometry, W, dq(q(W)), prompts, FP8 engine bound to W, bfloat16 engine bound to dq(q(W)))"""
    from speech_to_speech_b200 import engine as E
    g = GEOMETRIES[request.param]
    w = W.make_llama_weights(g, 3)
    wd = F.dq_state_dict(w, g)
    rng = np.random.default_rng(9)
    prompts = [rng.integers(0, g.vocab, n) for n in LENS]
    kw = dict(dtype="bfloat16", max_sessions=16, max_positions=128, max_prefill=64)
    a = E.LlamaEngine(g.to_dict(), weight_dtype="float8_e4m3", **kw)
    b = E.LlamaEngine(g.to_dict(), **kw)
    try:
        a.load_state_dict(w)
        b.load_state_dict(wd)
        yield g, w, wd, prompts, a, b
    finally:
        a.close()
        b.close()


def _prefill(eng, prompts, sampling=None):
    firsts, logits = [], []
    for s, p in enumerate(prompts):
        eng.reset(s)
        eng.set_sampling(s, **(sampling or {}).get(s, {}))
        nxt, lg = eng.prefill(s, p.tolist(), return_logits=True)
        firsts.append(int(nxt[0]))
        logits.append(lg[-1].cpu().numpy())
    return torch.tensor(firsts, dtype=torch.int32, device="cuda"), np.stack(logits)


def _run(eng, prompts, sampling=None, steps=STEPS):
    first, pl = _prefill(eng, prompts, sampling)
    ids, _, lg = eng.decode(list(range(len(prompts))), first, steps, return_logits=True)
    return first.cpu().numpy(), pl, ids.cpu().numpy(), lg.cpu().numpy()


@pytest.mark.parametrize("B", [1, 3, 8, 16])
def test_fp8_engine_equals_bf16_engine_on_dequantised_weights(pair, B):
    g, _, _, prompts, a, b = pair
    from speech_to_speech_b200 import _lib
    assert a.weight_format() == _lib.S2S_FP8_E4M3 and b.weight_format() == _lib.S2S_BF16
    assert a.max_decode_batch() == b.max_decode_batch() >= B
    ra, rb = _run(a, prompts[:B]), _run(b, prompts[:B])
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[2], rb[2])                          # ids
    assert np.array_equal(ra[1].view(np.uint32), rb[1].view(np.uint32)), "prefill logits"        # the row-major dq(Q)
    assert np.array_equal(ra[3].view(np.uint32), rb[3].view(np.uint32)), "decode logits"         # the FP8 stream


def test_fp8_engine_matches_oracle_on_dequantised_weights(pair):
    """guards against both engines being wrong together: the numpy forward pass over dq(q(W))"""
    g, _, wd, prompts, a, _ = pair
    if g.d_model > 1024:
        pytest.skip("the numpy oracle is run on the small geometries")
    n = 6
    sessions = (0, 1, 2)
    refs = {s: R.greedy_generate(wd, g, prompts[s], n, return_logits=True) for s in sessions}
    first, pl = _prefill(a, prompts[:3])
    first = first.cpu().numpy()
    forced = np.zeros((3, n - 1), dtype=np.int32)
    for s, r in refs.items():
        assert np.abs(pl[s] - r[1][0]).max() < TOL
        top2 = np.sort(r[1][0])[-2:]
        if top2[1] - top2[0] > 4 * TOL:
            assert first[s] == r[0][0]
        first[s], forced[s] = r[0][0], r[0][1:]
    ids, _, lg = a.decode([0, 1, 2], torch.from_numpy(first).cuda(), n - 1, forced=torch.from_numpy(forced).cuda(), return_logits=True)
    ids, lg = ids.cpu().numpy(), lg.cpu().numpy()
    for s, r in refs.items():
        assert np.abs(lg[:, s] - r[1][1:]).max() < TOL, s
        for i in range(n - 1):
            top2 = np.sort(r[1][1 + i])[-2:]
            if top2[1] - top2[0] > 4 * TOL:
                assert ids[s, i] == r[0][1 + i], (s, i)


def test_fp8_batch_invariance_and_sampling(pair):
    g, _, _, prompts, a, b = pair
    alone = _run(a, prompts[:1])
    among = _run(a, prompts)
    assert np.array_equal(alone[2][0], among[2][0])          # a session's ids do not depend on its neighbours
    sa, sb = _run(a, prompts[:8], SAMPLED), _run(b, prompts[:8], SAMPLED)
    assert np.array_equal(sa[0], sb[0]) and np.array_equal(sa[2], sb[2])
    assert np.array_equal(sa[3].view(np.uint32), sb[3].view(np.uint32))
    assert not np.array_equal(sa[2][0], among[2][0])         # the sampled session did leave the greedy path


def test_fp8_interface():
    from speech_to_speech_b200 import _lib, engine as E
    from speech_to_speech_b200._lib import S2SError
    g = GEOMETRIES["micro"]
    kw = dict(max_sessions=1, max_positions=64, max_prefill=16)
    with pytest.raises(ValueError, match="float8_e4m3"):
        E.LlamaEngine(g.to_dict(), weight_dtype="int8", **kw)
    with pytest.raises(S2SError):                            # dq(Q) can leave fp16's range
        E.LlamaEngine(g.to_dict(), dtype="float16", weight_dtype="float8_e4m3", **kw)
    with pytest.raises(S2SError):                            # multi-table models (TTS code predictor) stay 16-bit
        E.LlamaEngine(dict(g.to_dict(), n_tables=2), weight_dtype="float8_e4m3", **kw)
    eng = E.LlamaEngine(g.to_dict(), dtype="float16", **kw)
    try:
        lib = eng.lib
        assert eng.weight_format() == _lib.S2S_F16
        assert lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_FP8_E4M3) == -4     # S2S_ERR_UNSUPPORTED
        assert lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_F16) == 0
        eng.init_random(1)
        assert lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_F16) == -1          # S2S_ERR_INVALID: finalized
    finally:
        eng.close()
    eng = E.LlamaEngine(g.to_dict(), weight_dtype="float8_e4m3", **kw)
    try:
        eng.init_random(1)
        assert eng.weight_format() == _lib.S2S_FP8_E4M3
        assert eng.lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_BF16) == -1
        out = eng.generate([1, 2, 3], 8)
        assert len(out) == 8
    finally:
        eng.close()


def test_fp8_llama_3_8b_geometry_decodes_16_sessions_per_lane():
    """the FP8 ring slots are no larger than the 16-bit ones: the plan of a 66-CTA lane still carries 16 sessions"""
    from speech_to_speech_b200 import engine as E
    eng = E.LlamaEngine(GEOMETRIES["8b-wide-1l"].to_dict(), weight_dtype="float8_e4m3", max_sessions=16, max_positions=64,
                        max_prefill=16, lane=1, lanes=2)
    try:
        assert eng.max_decode_batch() == 16
    finally:
        eng.close()
