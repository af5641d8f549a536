"""GPU parity tests (H100) for the Llama-family path through the C ABI, against the numpy oracle and the
transformers goldens.  bf16 weights/operands, fp32 accumulate/residual: logits tolerance 3e-2 (values O(1));
token ids exact wherever the oracle's top-1 margin exceeds 4x that tolerance."""
import os

import numpy as np
import pytest
import torch

from oracle import weights as W, llama_ref as R

pytestmark = pytest.mark.gpu
# fp16 operands validate the algorithm tightly; bf16 (the Llama storage type) has 3 fewer mantissa bits and the
# sharp random-init attention amplifies it: measured max |err| 0.09 on logits of std 0.65 (mini), fp16 0.010.
TOL = {"float16": 2.5e-2, "bfloat16": 0.2}
LOGIT_TOL = TOL["bfloat16"]


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _engine(E, name, dtype="bfloat16", **kw):
    g = W.LLAMA_GEOMETRIES[name]
    w = W.make_llama_weights(g, 0)
    eng = E.LlamaEngine(g.to_dict(), dtype=dtype, max_positions=256, max_prefill=128, **kw)
    eng.load_state_dict(w)
    return g, w, eng


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", ["micro", "mini"])
def test_prefill_logits_match_golden(E, golden_dir, name, dtype):
    g, w, eng = _engine(E, name, dtype)
    LOGIT_TOL = TOL[dtype]
    G = np.load(os.path.join(golden_dir, f"llama_{name}.npz"))
    nxt, logits = eng.prefill(0, G["prompt"].tolist(), return_logits=True)
    lg = logits.cpu().numpy()
    assert np.abs(lg[-1][G["col_idx"]] - G["prefill_last_cols"]).max() < LOGIT_TOL
    assert np.abs(lg[len(G["prompt"]) // 2][G["col_idx"]] - G["prefill_mid_cols"]).max() < LOGIT_TOL
    if G["top_val"][0, 0] - G["top_val"][0, 1] > 4 * LOGIT_TOL:
        assert int(nxt[0]) == int(G["gen_ids"][0])


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", ["micro", "mini"])
def test_decode_ids_and_logits_match_golden(E, golden_dir, name, dtype):
    g, w, eng = _engine(E, name, dtype)
    LOGIT_TOL = TOL[dtype]
    G = np.load(os.path.join(golden_dir, f"llama_{name}.npz"))
    gold = G["gen_ids"]
    n = len(gold)
    eng.prefill(0, G["prompt"].tolist())
    first = torch.tensor([int(gold[0])], dtype=torch.int32, device="cuda")
    forced = torch.from_numpy(np.ascontiguousarray(gold[None, 1:])).cuda().int()
    ids, lens, logits = eng.decode([0], first, n - 1, forced=forced, return_logits=True)
    ids = ids[0].cpu().numpy()
    lg = logits[:, 0].cpu().numpy()
    tv = np.take_along_axis(lg, G["top_idx"][1:], 1)
    assert np.abs(tv - G["top_val"][1:]).max() < LOGIT_TOL
    margin = G["top_val"][1:, 0] - G["top_val"][1:, 1]
    safe = margin > 4 * LOGIT_TOL
    assert (ids[safe] == gold[1:][safe]).all()


def test_generate_end_to_end_and_chunked_prefill(E, golden_dir):
    g, w, eng = _engine(E, "micro")
    G = np.load(os.path.join(golden_dir, "llama_micro.npz"))
    gold = G["gen_ids"]
    margin = G["top_val"][:, 0] - G["top_val"][:, 1]
    safe = margin > 4 * LOGIT_TOL
    k = int(np.argmin(safe)) if (~safe).any() else len(gold)
    out = eng.generate(G["prompt"].tolist(), len(gold))
    assert out[:k] == gold[:k].tolist()
    # the same prompt through prefill chunks of 7 tokens
    eng2 = E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_positions=256, max_prefill=7)
    eng2.load_state_dict(w)
    out2 = eng2.generate(G["prompt"].tolist(), len(gold))
    assert out2[:k] == gold[:k].tolist()


def test_two_sessions_of_different_length_decode_together(E):
    g, w, eng = _engine(E, "micro", max_sessions=2)
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, g.vocab, 9), rng.integers(0, g.vocab, 70)]
    refs, firsts = [], []
    for p in prompts:
        ids, lg = R.greedy_generate(w, g, p, 7, return_logits=True)
        refs.append((ids, lg))
    for s, p in enumerate(prompts):
        nxt, _ = eng.prefill(s, p.tolist())
        firsts.append(refs[s][0][0])
    first = torch.tensor(firsts, dtype=torch.int32, device="cuda")
    forced = torch.tensor([r[0][1:] for r in refs], dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode([0, 1], first, 6, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()
    for s in range(2):
        assert np.abs(lg[:, s] - refs[s][1][1:]).max() < LOGIT_TOL


def test_ten_sessions_decode_together(E):
    """10 sessions in one persistent launch (sessions 8, 9 sit in the upper half of the tensor-core tile)."""
    nb = 10
    g, w, eng = _engine(E, "micro", dtype="float16", max_sessions=nb)
    rng = np.random.default_rng(11)
    prompts = [rng.integers(0, g.vocab, 5 + 6 * s) for s in range(nb)]
    refs = [R.greedy_generate(w, g, p, 5, return_logits=True) for p in prompts]
    for s, p in enumerate(prompts):
        eng.prefill(s, p.tolist())
    first = torch.tensor([r[0][0] for r in refs], dtype=torch.int32, device="cuda")
    forced = torch.tensor([r[0][1:] for r in refs], dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode(list(range(nb)), first, 4, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()
    for s in range(nb):
        assert np.abs(lg[:, s] - refs[s][1][1:]).max() < TOL["float16"], s


def test_eos_stops_generation(E, golden_dir):
    g, w, eng = _engine(E, "micro")
    G = np.load(os.path.join(golden_dir, "llama_micro.npz"))
    gold = G["gen_ids"]
    eos = int(gold[3])
    first = int(np.argmax(gold == eos))
    out = eng.generate(G["prompt"].tolist(), len(gold), eos_id=eos)
    assert out == gold[: first + 1].tolist()


def test_llama3_8b_layer_geometry_two_layers(E):
    """Exact Llama-3-8B layer shapes (d 4096, 32/8 heads, ffn 14336, vocab 128256), 2 layers: decode logits vs oracle."""
    g = W.LLAMA_GEOMETRIES["llama-3-8b-2l"]
    w = W.make_llama_weights(g, 0)
    eng = E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_positions=128, max_prefill=64)
    eng.load_state_dict(w)
    prompt = np.random.default_rng(9).integers(0, g.vocab, 40)
    ref_ids, ref_lg = R.greedy_generate(w, g, prompt, 3, return_logits=True)
    nxt, logits = eng.prefill(0, prompt.tolist(), return_logits=True)
    assert np.abs(logits[-1].cpu().numpy() - ref_lg[0]).max() < LOGIT_TOL
    first = torch.tensor([ref_ids[0]], dtype=torch.int32, device="cuda")
    forced = torch.tensor([ref_ids[1:]], dtype=torch.int32, device="cuda")
    ids, lens, lg = eng.decode([0], first, 2, forced=forced, return_logits=True)
    assert np.abs(lg[:, 0].cpu().numpy() - ref_lg[1:]).max() < LOGIT_TOL


# ---- Qwen3 family (qk_norm): the reference's DEFAULT LLM is Qwen/Qwen3-4B-Instruct-2507 (language_model_base_arguments.py:6-9)
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_qwen3_qk_norm_prefill_and_decode_match_golden(E, golden_dir, dtype):
    """Per-head RMSNorm(head_dim) on q and k before RoPE (transformers modeling_qwen3.py Qwen3Attention), golden pinned
    to Qwen3ForCausalLM: prefill logits, teacher-forced decode logits, ids where the margin allows."""
    g, w, eng = _engine(E, "qwen3-micro", dtype)
    tol = TOL[dtype]
    G = np.load(os.path.join(golden_dir, "llama_qwen3-micro.npz"))
    gold = G["gen_ids"]
    nxt, logits = eng.prefill(0, G["prompt"].tolist(), return_logits=True)
    lg = logits.cpu().numpy()
    assert np.abs(lg[-1][G["col_idx"]] - G["prefill_last_cols"]).max() < tol
    assert np.abs(lg[len(G["prompt"]) // 2][G["col_idx"]] - G["prefill_mid_cols"]).max() < tol
    first = torch.tensor([int(gold[0])], dtype=torch.int32, device="cuda")
    forced = torch.from_numpy(np.ascontiguousarray(gold[None, 1:])).cuda().int()
    ids, lens, dlog = eng.decode([0], first, len(gold) - 1, forced=forced, return_logits=True)
    dl = dlog[:, 0].cpu().numpy()
    tv = np.take_along_axis(dl, G["top_idx"][1:], 1)
    assert np.abs(tv - G["top_val"][1:]).max() < tol
    safe = (G["top_val"][1:, 0] - G["top_val"][1:, 1]) > 4 * tol
    assert (ids[0].cpu().numpy()[safe] == gold[1:][safe]).all()


def test_qwen3_decode_matches_debug_phases_and_oracle_batch(E, monkeypatch):
    """Qwen3 geometry, 3 sessions of different lengths in one launch vs the oracle; the persistent launch and the
    one-launch-per-phase debug mode must agree bit for bit (the grid barrier is the only difference)."""
    g = W.LLAMA_GEOMETRIES["qwen3-micro"]
    w = W.make_llama_weights(g, 0)
    rng = np.random.default_rng(21)
    prompts = [rng.integers(0, g.vocab, n) for n in (5, 33, 70)]
    refs = [R.greedy_generate(w, g, p, 6, return_logits=True) for p in prompts]
    outs = []
    for dbg in ("0", "1"):
        monkeypatch.setenv("S2S_DEBUG_PHASES", dbg)
        eng = E.LlamaEngine(g.to_dict(), dtype="float16", max_sessions=3, max_positions=128, max_prefill=128)
        eng.load_state_dict(w)
        for s, p in enumerate(prompts):
            eng.prefill(s, p.tolist())
        first = torch.tensor([r[0][0] for r in refs], dtype=torch.int32, device="cuda")
        forced = torch.tensor([r[0][1:] for r in refs], dtype=torch.int32, device="cuda")
        ids, lens, logits = eng.decode([0, 1, 2], first, 5, forced=forced, return_logits=True)
        outs.append((ids.cpu().numpy().copy(), logits.cpu().numpy().copy()))
        eng.close()
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    for s in range(3):
        assert np.abs(outs[0][1][:, s] - refs[s][1][1:]).max() < TOL["float16"], s


def test_llama3_8b_geometry_eight_sessions_k_chunked_down_projection(E):
    """Llama-3-8B layer shapes, 2 layers, EIGHT sessions of different lengths in one launch: beyond 4 sessions the ffn-wide
    (14336) down-projection operand is staged in K-chunks of 4096 columns and the RMSNorm statistics copy in row groups
    (llama_decode_plan).  fp16 operands for a tight tolerance; every session's logits against the oracle, and the chunked
    launch against the same sessions decoded 4 + 4 through the unchunked path."""
    g = W.LLAMA_GEOMETRIES["llama-3-8b-2l"]
    w = W.make_llama_weights(g, 0)
    eng = E.LlamaEngine(g.to_dict(), dtype="float16", max_sessions=8, max_positions=128, max_prefill=64)
    eng.load_state_dict(w)
    assert eng.max_decode_batch() >= 8
    rng = np.random.default_rng(31)
    prompts = [rng.integers(0, g.vocab, 4 + 5 * s) for s in range(8)]
    refs = [R.greedy_generate(w, g, p, 4, return_logits=True) for p in prompts]
    first = torch.tensor([r[0][0] for r in refs], dtype=torch.int32, device="cuda")
    forced = torch.tensor([r[0][1:] for r in refs], dtype=torch.int32, device="cuda")

    def prefill_all():
        for s, p in enumerate(prompts):
            eng.reset(s)
            eng.prefill(s, p.tolist())
    prefill_all()
    ids8, _, lg8 = eng.decode(list(range(8)), first, 3, forced=forced, return_logits=True)
    lg8 = lg8.cpu().numpy()
    for s in range(8):
        assert np.abs(lg8[:, s] - refs[s][1][1:]).max() < TOL["float16"], s
    prefill_all()
    _, _, a = eng.decode([0, 1, 2, 3], first[:4].contiguous(), 3, forced=forced[:4].contiguous(), return_logits=True)
    _, _, b = eng.decode([4, 5, 6, 7], first[4:].contiguous(), 3, forced=forced[4:].contiguous(), return_logits=True)
    lg44 = np.concatenate([a.cpu().numpy(), b.cpu().numpy()], axis=1)
    assert np.abs(lg8 - lg44).max() < 5e-3     # same sums, different association across the K-chunks (measured 2.1e-3)


def test_batched_prefill_matches_oracle_and_sequential_prefill(E):
    """s2s_llama_prefill_batch: four prompts of different lengths prefilled in one pass over the weights (one of them appended to
    a session that already holds 9 tokens) -- next ids equal the sequential prefill's, and the decode that follows matches the
    oracle's logits for every session (the KV rows written by the batched pass are the ones a sequential pass writes)."""
    g, w, eng = _engine(E, "micro", max_sessions=8)
    rng = np.random.default_rng(21)
    prompts = [rng.integers(0, g.vocab, n) for n in (15, 30, 5, 17)]
    refs = [R.greedy_generate(w, g, p, 6, return_logits=True) for p in prompts]
    # sequential reference on slots 4..7
    seq_next = [int(eng.prefill(4 + s, p.tolist())[0][0]) for s, p in enumerate(prompts)]
    # batched: session 0 already holds the first 9 tokens of its prompt, the batch appends the remaining 6
    eng.prefill(0, prompts[0][:9].tolist())
    nxt = eng.prefill_batch([0, 1, 2, 3], [prompts[0][9:].tolist()] + [p.tolist() for p in prompts[1:]]).cpu().tolist()
    for s in range(4):
        margin = refs[s][1][0]
        top2 = np.sort(margin)[-2:]
        if top2[1] - top2[0] > 4 * LOGIT_TOL:
            assert nxt[s] == seq_next[s] == int(refs[s][0][0]), s
    first = torch.tensor([r[0][0] for r in refs], dtype=torch.int32, device="cuda")
    forced = torch.tensor([r[0][1:] for r in refs], dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode([0, 1, 2, 3], first, 5, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()
    ids2, lens2, logits2 = eng.decode([4, 5, 6, 7], first, 5, forced=forced, return_logits=True)
    lg2 = logits2.cpu().numpy()
    for s in range(4):
        assert np.abs(lg[:, s] - refs[s][1][1:]).max() < LOGIT_TOL, s
        # against the sequentially prefilled twin: same kernels, same cache contents up to the GEMM tile shape
        assert np.abs(lg[:, s] - lg2[:, s]).max() < 2e-2, s
