"""GPU: the device token choice (csrc/sampling.cuh) in prefill and decode against oracle/sampling_ref.py applied to the kernel's
own logits_out, in launches that mix greedy, penalised-greedy and sampled sessions.  Ids must be exact wherever the decision
margin (Gumbel winner gap, top-k and top-p boundaries) exceeds 1e-4; a session is followed up to its first step below that."""
import threading

import numpy as np
import pytest
import torch

from oracle import sampling_ref as R

pytestmark = pytest.mark.gpu

SAFE = 1e-4
GEOMS = {
    "micro": dict(d_model=256, layers=2, heads=2, kv_heads=1, head_dim=128, ffn=512, vocab=2048),
    "llama-3-8b": dict(d_model=4096, layers=32, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256,
                       rope_theta=500000.0, rms_eps=1e-5),
}
CONFIGS = [
    dict(),                                                          # greedy
    dict(repetition_penalty=1.3),                                    # penalised greedy
    dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9),
    dict(do_sample=True, top_k=0, top_p=0.9),
    dict(do_sample=True, temperature=1.5, top_k=5, repetition_penalty=1.1),
    dict(do_sample=True, temperature=1.0),                           # the whole vocabulary survives
    dict(min_new_tokens=16),                                         # EOS ids filled in per session
    dict(do_sample=True, temperature=0.8, top_p=0.5, min_new_tokens=16),
]


def _engine(name, max_sessions, lane=0, lanes=1):
    from speech_to_speech_b200 import engine as E
    eng = E.LlamaEngine(GEOMS[name], dtype="bfloat16", max_sessions=max_sessions, max_positions=256, max_prefill=64, lane=lane, lanes=lanes)
    eng.init_random(11)
    return eng


@pytest.fixture(scope="module", params=["micro", "llama-3-8b"])
def eng(request):
    e = _engine(request.param, 16)
    yield e
    e.close()
    torch.cuda.empty_cache()


def _plan(eng, B, rng):
    V = eng.geometry["vocab"]
    out = []
    for b in range(B):
        cfg = dict(CONFIGS[b % len(CONFIGS)])
        prompt = rng.integers(0, V, size=int(rng.integers(3, 20))).tolist()
        if cfg.get("min_new_tokens"):
            cfg["eos_ids"] = []   # the top raw candidates of the prompt, set after the prefill logits are known
        out.append((b, cfg, prompt, 1000 + 17 * b))
    return out


def _prefill_all(eng, plan, kernel_cfgs=True, eos_from=None):
    firsts, prefill_logits = [], []
    for slot, cfg, prompt, seed in plan:
        eng.reset(slot)
        c = dict(cfg) if kernel_cfgs else {}
        if eos_from is not None and "eos_ids" in c:
            c["eos_ids"] = eos_from[slot]
        eng.set_sampling(slot, seed=seed, **c)
        nxt, lg = eng.prefill(slot, prompt, return_logits=True)
        firsts.append(int(nxt[0]))
        prefill_logits.append(lg[-1].float().cpu().numpy())
    return firsts, prefill_logits


def _eos_ids(eng, plan):
    """For the min_new_tokens sessions: the 8 most likely raw ids after the prompt, so that EOS would win at once."""
    out = {}
    for slot, cfg, prompt, seed in plan:
        eng.reset(slot)
        eng.set_sampling(slot)
        _, lg = eng.prefill(slot, prompt, return_logits=True)
        out[slot] = np.argsort(-lg[-1].float().cpu().numpy())[:8].tolist()
    return out


def _kw(cfg, seed, seen, n_generated, eos):
    return dict(seed=seed, seen=list(seen), penalty=cfg.get("repetition_penalty", 1.0), eos_ids=eos.get("eos", []),
                min_new_tokens=cfg.get("min_new_tokens", 0), n_generated=n_generated, do_sample=cfg.get("do_sample", False),
                temperature=cfg.get("temperature", 1.0), top_k=cfg.get("top_k", 0), top_p=cfg.get("top_p", 1.0))


def _check_session(cfg, seed, prompt, first, pre_row, ids, logits, eos):
    """-> number of decisions checked; asserts every safe decision equals the oracle's."""
    n = len(prompt)
    seen = set(prompt)
    kw = _kw(cfg, seed, seen, 0, eos)
    checked = 0
    if R.margin(pre_row, n, **kw) > SAFE:
        assert first == R.choose(pre_row, n, **kw)[0]
        checked += 1
    else:
        return checked
    seen.add(first)
    for s in range(ids.shape[0]):
        kw = _kw(cfg, seed, seen, s + 1, eos)
        if R.margin(logits[s], n + s + 1, **kw) <= SAFE:
            break
        assert int(ids[s]) == R.choose(logits[s], n + s + 1, **kw)[0], f"step {s} cfg {cfg}"
        checked += 1
        seen.add(int(ids[s]))
    return checked


def test_mixed_launch_matches_the_oracle_and_keeps_greedy_bit_identical(eng):
    B = eng.max_decode_batch()
    rng = np.random.default_rng(5)
    plan = _plan(eng, B, rng)
    eos = _eos_ids(eng, plan)
    firsts, pre = _prefill_all(eng, plan, eos_from=eos)
    first_t = torch.tensor(firsts, dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode([p[0] for p in plan], first_t, 32, return_logits=True)
    ids = ids.cpu().numpy()
    lg = logits.float().cpu().numpy()
    total = 0
    for b, (slot, cfg, prompt, seed) in enumerate(plan):
        e = {"eos": eos[slot]} if "eos_ids" in cfg else {}
        total += _check_session(cfg, seed, prompt, firsts[b], pre[b], ids[b], lg[:, b], e)
        if cfg.get("min_new_tokens"):   # no EOS before min_new_tokens tokens: the prefill's token and decode steps 0..14
            assert firsts[b] not in eos[slot] and not set(ids[b, :15].tolist()) & set(eos[slot])
    assert total >= B * 8, f"only {total} decisions were safely checkable"
    # the same launch with every session greedy: the greedy sessions' ids and logits do not move
    g_first, _ = _prefill_all(eng, plan, kernel_cfgs=False)
    g_ids, _, g_logits = eng.decode([p[0] for p in plan], torch.tensor(g_first, dtype=torch.int32, device="cuda"), 32, return_logits=True)
    for b, (slot, cfg, prompt, seed) in enumerate(plan):
        if not cfg:
            assert g_first[b] == firsts[b]
            assert np.array_equal(g_ids[b].cpu().numpy(), ids[b])
            assert torch.equal(g_logits[:, b], logits[:, b])


def test_penalty_sees_exactly_the_prompt_and_the_fed_ids_after_a_chunked_prefill(eng):
    """A prompt longer than max_prefill is prefilled in chunks; the token chosen after each intermediate chunk is discarded
    and must not join the repetition-penalty set: the oracle's seen set is the prompt plus the fed ids, nothing else."""
    cap = int(eng.cfg.max_prefill)
    rng = np.random.default_rng(21)
    V = eng.geometry["vocab"]
    cfgs = [dict(repetition_penalty=3.0), dict(do_sample=True, temperature=0.7, top_k=50, repetition_penalty=2.0)]
    checked = 0
    for slot, cfg in enumerate(cfgs):
        prompt = rng.integers(0, V, size=2 * cap + 22).tolist()
        eng.reset(slot)
        eng.set_sampling(slot, seed=77 + slot, **cfg)
        for o in range(0, len(prompt), cap):
            nxt, lg = eng.prefill(slot, prompt[o:o + cap], return_logits=True)
        first = int(nxt[0])
        ids, _, logits = eng.decode([slot], nxt, 24, return_logits=True)
        checked += _check_session(cfg, 77 + slot, prompt, first, lg[-1].float().cpu().numpy(), ids[0].cpu().numpy(),
                                  logits[:, 0].float().cpu().numpy(), {})
    assert checked >= 16


def test_batched_prefill_matches_the_oracle(eng):
    """s2s_llama_prefill_batch chooses every session's token like s2s_llama_prefill; its rows differ from the single-session
    prefill only by the GEMM tile shape, so decisions are compared where the margin exceeds 1e-2."""
    B = min(eng.max_decode_batch(), 8)
    plan = _plan(eng, B, np.random.default_rng(13))
    plan = [(s, {k: v for k, v in c.items() if k != "eos_ids"}, p[:7], seed) for s, c, p, seed in plan]
    _, rows = _prefill_all(eng, plan)
    for slot, cfg, prompt, seed in plan:
        eng.reset(slot)
        eng.set_sampling(slot, seed=seed, **cfg)
    got = eng.prefill_batch([p[0] for p in plan], [p[2] for p in plan]).tolist()
    checked = 0
    for b, (slot, cfg, prompt, seed) in enumerate(plan):
        kw = _kw(cfg, seed, set(prompt), 0, {})
        if R.margin(rows[b], len(prompt), **kw) > 1e-2:
            assert got[b] == R.choose(rows[b], len(prompt), **kw)[0], cfg
            checked += 1
    assert checked >= B // 2


def test_one_long_launch_equals_short_launches(eng):
    B = min(eng.max_decode_batch(), 6)
    plan = _plan(eng, B, np.random.default_rng(9))[:B]
    plan = [(s, {k: v for k, v in c.items() if k != "eos_ids"}, p, seed) for s, c, p, seed in plan]
    slots = [p[0] for p in plan]
    firsts, _ = _prefill_all(eng, plan)
    long_ids, _ = eng.decode(slots, torch.tensor(firsts, dtype=torch.int32, device="cuda"), 32)
    firsts2, _ = _prefill_all(eng, plan)
    assert firsts2 == firsts
    cur, parts = torch.tensor(firsts2, dtype=torch.int32, device="cuda"), []
    for _ in range(8):
        ids, _ = eng.decode(slots, cur, 4)
        parts.append(ids)
        cur = ids[:, -1].contiguous()
    assert torch.equal(torch.cat(parts, dim=1), long_ids)


def test_two_lanes_match_one_lane():
    plan = _plan(_Geom("micro"), 4, np.random.default_rng(3))
    plan = [(s, {k: v for k, v in c.items() if k != "eos_ids"}, p, seed) for s, c, p, seed in plan]
    one = _engine("micro", 4)
    try:
        firsts, pre = _prefill_all(one, plan)
        ids1, _, lg1 = one.decode([0, 1, 2, 3], torch.tensor(firsts, dtype=torch.int32, device="cuda"), 24, return_logits=True)
        ids1, lg1 = ids1.cpu().numpy(), lg1.float().cpu().numpy()
    finally:
        one.close()
    from speech_to_speech_b200 import engine as E
    lanes = [_engine("micro", 4, lane=i, lanes=2) for i in range(2)]
    got = {}
    try:
        def run(i):
            eng = lanes[i]
            mine = plan[2 * i: 2 * i + 2]
            with E.lane_context(0, i, 2):
                f, _ = _prefill_all(eng, mine)
                ids, _ = eng.decode([p[0] for p in mine], torch.tensor(f, dtype=torch.int32, device="cuda"), 24)
                torch.cuda.current_stream().synchronize()
            for j, p in enumerate(mine):
                got[p[0]] = (f[j], ids[j].cpu().numpy())
        th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        [t.start() for t in th]
        [t.join() for t in th]
    finally:
        for e in lanes:
            e.close()
    compared = 0
    for b, (slot, cfg, prompt, seed) in enumerate(plan):
        f, ids = got[slot]
        n, seen = len(prompt), set(prompt)
        if R.margin(pre[b], n, **_kw(cfg, seed, seen, 0, {})) <= SAFE:
            continue
        assert f == firsts[b]
        seen.add(f)
        for s in range(24):
            if R.margin(lg1[s, b], n + s + 1, **_kw(cfg, seed, seen, s + 1, {})) <= SAFE:
                break
            assert int(ids[s]) == int(ids1[b, s])
            seen.add(int(ids[s]))
            compared += 1
    assert compared >= 16


class _Geom:
    def __init__(self, name):
        self.geometry = GEOMS[name]


def test_handler_with_a_fixed_seed_reproduces_its_text_alone_and_shared():
    from speech_to_speech_b200.handlers import language_model_handler as LH

    def unit(seed):
        h = object.__new__(LH.B200LanguageModelHandler)
        h._load_model("random:micro:3", "cuda:0", "bfloat16",
                      {"max_new_tokens": 24, "max_sessions": 2, "do_sample": True, "temperature": 0.9, "top_k": 40, "top_p": 0.95,
                       "repetition_penalty": 1.1, "seed": seed})
        return h
    prompt = [5, 6, 7, 8, 9, 10]
    a = unit(7)
    try:
        alone = "".join(a.generate_text_stream(prompt, max_new_tokens=24))
    finally:
        a.cleanup()
    a2, b2 = unit(7), unit(8)
    out = {}
    try:
        def go(name, h):
            out[name] = "".join(h.generate_text_stream(prompt, max_new_tokens=24))
        th = [threading.Thread(target=go, args=("a", a2)), threading.Thread(target=go, args=("b", b2))]
        [t.start() for t in th]
        [t.join() for t in th]
    finally:
        a2.cleanup()
        b2.cleanup()
    assert alone and out["a"] == alone
    assert out["b"] != alone          # another seed draws another reply
