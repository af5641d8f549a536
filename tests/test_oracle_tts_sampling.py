"""CPU: the sampled Qwen3-TTS token choice of tests/tts_sampling_ref.py (on oracle/qwen3tts_ref.py + oracle/sampling_ref.py) against the transformers cousin
(Qwen3OmniMoeTalkerForConditionalGeneration at the micro geometry with make_weights weights, built the way
tests/golden/make_golden.py builds it) driven with the cousin's own sampling arguments: the processor lists of the talker
and of the code predictor are recorded, and every processed row must equal sampling_ref.process of the raw row with the
oracle's settings -- penalty domain = the generated first codes only, suppressed ids, T, top-k, top-p.  Also: the
stream word of the Philox counter."""
import numpy as np
import pytest
import torch

import tts_sampling_ref as T
from oracle import qwen3tts_ref as R, sampling_ref as S
from speech_to_speech_b200.tts_model import COUSIN_SAMPLING


def _cousin(g, w):
    from transformers.models.qwen3_omni_moe.configuration_qwen3_omni_moe import Qwen3OmniMoeTalkerConfig
    from transformers.models.qwen3_omni_moe import modeling_qwen3_omni_moe as M
    t, c = g.talker, g.predictor
    sec = [t.head_dim // 8, t.head_dim // 8 + t.head_dim // 16, 0]
    sec[2] = t.head_dim // 2 - sec[0] - sec[1]
    tc = dict(vocab_size=t.vocab, hidden_size=t.d_model, intermediate_size=t.ffn, num_hidden_layers=t.layers,
              num_attention_heads=t.heads, num_key_value_heads=t.kv_heads, head_dim=t.head_dim, rms_norm_eps=t.rms_eps,
              num_experts=2, num_experts_per_tok=1, moe_intermediate_size=64, shared_expert_intermediate_size=64,
              rope_parameters=dict(rope_type="default", rope_theta=t.rope_theta, mrope_section=sec, mrope_interleaved=True))
    cp = dict(vocab_size=c.vocab, hidden_size=c.d_model, intermediate_size=c.ffn, num_hidden_layers=c.layers,
              num_attention_heads=c.heads, num_key_value_heads=c.kv_heads, head_dim=c.head_dim, rms_norm_eps=c.rms_eps,
              num_code_groups=g.n_groups, rope_parameters={"rope_type": "default", "rope_theta": c.rope_theta})
    cfg = Qwen3OmniMoeTalkerConfig(text_config=tc, code_predictor_config=cp, num_code_groups=g.n_groups,
                                   thinker_hidden_size=g.text_hidden, codec_eos_token_id=g.codec_eos,
                                   codec_nothink_id=g.codec_nothink, codec_think_bos_id=g.codec_think_bos,
                                   codec_think_eos_id=g.codec_think_eos, codec_pad_id=g.codec_pad, codec_bos_id=g.codec_bos,
                                   speaker_id={"aiden": 2301}, spatial_merge_size=2)
    m = M.Qwen3OmniMoeTalkerForConditionalGeneration(cfg).eval()
    for layer in m.model.layers:   # the dense talker MLP (oracle/qwen3tts_ref.py)
        layer.mlp = M.Qwen3OmniMoeTalkerTextMLP(cfg.text_config, intermediate_size=t.ffn)
    sd = m.state_dict()
    m.load_state_dict({k: (sd[k] if k.startswith("hidden_projection.") else torch.from_numpy(w[k])) for k in sd})
    return M, cfg, m


def _record(model, log):
    """Wrap the logits-processor list `model.generate` builds: every call logs (input ids, raw scores, processed scores)."""
    from transformers import LogitsProcessorList
    orig = model._get_logits_processor

    class Rec(LogitsProcessorList):
        def __call__(self, input_ids, scores, **kw):
            out = super().__call__(input_ids, scores.clone(), **kw)
            log.append((input_ids[0].tolist(), scores[0].float().numpy().copy(), out[0].float().numpy().copy()))
            return out

    model._get_logits_processor = lambda *a, **k: Rec(orig(*a, **k))


@pytest.fixture(scope="module")
def cousin_run():
    g = R.GEOMETRIES["micro"]
    w = R.make_weights(g, 0)
    M, cfg, m = _cousin(g, w)
    talker_log, pred_log = [], []
    _record(m, talker_log)
    _record(m.code_predictor, pred_log)
    emb = torch.from_numpy(w["text_embedding.weight"])
    ids = torch.tensor([[g.im_start, g.assistant, g.newline, 5, 6, 7, 8]])

    class Host:   # the attributes _get_talker_assistant_parts reads from the top-level model
        pass
    host = Host()
    host.talker = m
    host.config = type("C", (), {"talker_config": cfg, "tts_pad_token_id": g.tts_pad})()
    suppress = R.suppress_ids(g)
    tk = COUSIN_SAMPLING["talker"]
    torch.manual_seed(0)
    with torch.no_grad():
        bos_e, eos_e, pad_e = m.text_projection(emb[torch.tensor([[g.tts_bos, g.tts_eos, g.tts_pad]])]).chunk(3, dim=1)
        embeds, in_ids, trailing = M.Qwen3OmniMoeForConditionalGeneration._get_talker_assistant_parts(
            host, 0, ids.shape[1], 2301, emb[ids], pad_e, bos_e, eos_e)
        # the cousin's talker call (TF:4064-4068, 3905-3909): inputs_embeds without input_ids, its sampling arguments
        res = m.generate(inputs_embeds=embeds, trailing_text_hidden=trailing, tts_pad_embed=pad_e, talker_input_ids=in_ids,
                         max_new_tokens=6, do_sample=True, top_k=tk["top_k"], top_p=tk["top_p"], temperature=tk["temperature"],
                         repetition_penalty=tk["repetition_penalty"], eos_token_id=g.codec_eos, suppress_tokens=suppress,
                         output_hidden_states=True, return_dict_in_generate=True, pad_token_id=g.codec_pad,
                         attention_mask=torch.ones_like(in_ids))
    return g, m, talker_log, pred_log, res.sequences[0].tolist(), suppress


def test_talker_processors_penalise_the_generated_first_codes_only(cousin_run):
    g, m, talker_log, _, seq, suppress = cousin_run
    assert len(talker_log) >= 2
    tkw = T.choose_kw(COUSIN_SAMPLING["talker"])
    for step, (ids, raw, want) in enumerate(talker_log):
        assert ids == seq[:step]                               # generate's sequence holds the generated code0s only
        row = raw.copy()
        row[suppress] = -np.inf                                # what the device stores: suppressed ids -inf (EPI_LOGITS)
        got = S.process(row, seen=ids, eos_ids=(), **{k: v for k, v in tkw.items()})
        np.testing.assert_array_equal(np.isinf(got), np.isinf(want))
        np.testing.assert_array_equal(got[np.isfinite(got)], want[np.isfinite(want)])


def test_predictor_processors_are_top_k_50_top_p_0_8_at_temperature_1(cousin_run):
    g, m, _, pred_log, _, _ = cousin_run
    assert m.code_predictor.generation_config.temperature in (None, 1.0)   # the predictor's own default: T = 1
    assert len(pred_log) >= g.n_groups - 1
    pkw = T.choose_kw(COUSIN_SAMPLING["predictor"])
    assert pkw["temperature"] == 1.0 and pkw["top_k"] == 50 and pkw["top_p"] == 0.8 and pkw["penalty"] == 1.0
    for ids, raw, want in pred_log:
        got = S.process(raw, **pkw)
        np.testing.assert_array_equal(np.isinf(got), np.isinf(want))
        np.testing.assert_array_equal(got[np.isfinite(got)], want[np.isfinite(want)])


def _kernel_philox(seed, c0, c1, c2):
    """The rounds of csrc/sampling.cuh samp_philox, in Python integers."""
    M0, M1, W0, W1, MASK = 0xD2E7470EE14C6C93, 0xCA5A826395121157, 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B, (1 << 64) - 1
    x0, x1, x2, x3, k0, k1 = c0, c1, c2, 0, seed, 0
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * x0, M1 * x2
        x0, x1, x2, x3 = ((p1 >> 64) ^ x1 ^ k0) & MASK, p1 & MASK, ((p0 >> 64) ^ x3 ^ k1) & MASK, p0 & MASK
    return x0


@pytest.mark.parametrize("seed,pos,stream", [(0, 2, 1), (123456789, 9, 17), ((1 << 64) - 1, 3, 1536)])
def test_stream_word_is_the_third_philox_counter(seed, pos, stream):
    u = T.uniforms(seed, pos, 200, stream)
    u0 = T.uniforms(seed, pos, 200)
    for tok in (0, 1, 77, 199):
        raw = int(np.random.Philox(key=seed, counter=[tok, pos, stream, 0]).random_raw())
        assert raw == _kernel_philox(seed, tok + 1, pos, stream)
        assert u[tok] == T.uniform_one(seed, pos, tok, stream) == (raw >> 11) / 2.0 ** 53
        raw0 = int(np.random.Philox(key=seed, counter=[tok, pos, 0, 0]).random_raw())   # stream 0: the LLM's stream
        assert u0[tok] == T.uniforms(seed, pos, 200, 0)[tok] == (raw0 >> 11) / 2.0 ** 53
    assert not np.array_equal(u, u0)
    np.testing.assert_array_equal(u0, S.uniforms(seed, pos, 200))                  # stream 0 = oracle/sampling_ref.py's stream
    z = np.random.default_rng(pos).standard_normal(200).astype(np.float32)
    kw = dict(do_sample=True, temperature=0.9, top_k=50, top_p=0.8)
    assert T.choose(z, pos, seed=seed, **kw)[0] == S.choose(z, pos, seed=seed, **kw)[0]


def test_oracle_sampled_generation_counters_and_replay():
    """generate(sampling=...) chooses every code with (talker position, stream 0, seen code0s) / (predictor position,
    stream 1 + frame); the teacher-forced replay along its own codes reports the same decisions."""
    g = R.GEOMETRIES["micro"]
    w = R.make_weights(g, 0)
    codes = T.generate(w, g, [5, 6, 7], 2301, 4, sampling=COUSIN_SAMPLING, seed=99)
    greedy = R.generate(w, g, [5, 6, 7], 2301, 4)
    np.testing.assert_array_equal(T.generate(w, g, [5, 6, 7], 2301, 4), greedy)   # no sampling: the pinned greedy oracle
    assert codes.shape[1] == g.n_groups and not np.array_equal(codes, greedy[: len(codes)])
    rec = T.replay(w, g, [5, 6, 7], 2301, codes, sampling=COUSIN_SAMPLING, seed=99)
    assert len(rec) == codes.size
    for d in rec:
        assert d["choice"] == codes[d["frame"], d["group"]]
        if d["group"] == 0:
            assert d["stream"] == 0 and d["position"] == 9 + d["frame"] and d["seen"] == frozenset(codes[: d["frame"], 0].tolist())
        else:
            assert d["stream"] == 1 + d["frame"] and d["position"] == d["group"] + 1
    np.testing.assert_array_equal(T.generate(w, g, [5, 6, 7], 2301, 4, sampling=COUSIN_SAMPLING, seed=99), codes)
