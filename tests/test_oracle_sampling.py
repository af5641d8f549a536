"""CPU: oracle/sampling_ref.py against transformers and numpy.
(a) the processed / warped rows equal what the processor list of transformers' _get_logits_processor makes of them;
(b) the uniforms are numpy.random.Philox's stream, and a plain restatement of the kernel's Philox4x64-10 rounds agrees;
(c) the Gumbel draws follow the softmax of the warped row (chi-square over fixed counters: deterministic)."""
import numpy as np
import pytest
import torch

from oracle import sampling_ref as R

V = 64


@pytest.fixture(scope="module")
def tiny_llama():
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=V, hidden_size=16, intermediate_size=32, num_hidden_layers=1, num_attention_heads=2,
                      num_key_value_heads=1, max_position_embeddings=64)
    return LlamaForCausalLM(cfg)


def _hf_row(model, z, prompt, n_generated, **gen):
    from transformers import GenerationConfig
    gc = GenerationConfig(**gen)
    model._prepare_special_tokens(gc, kwargs_has_attention_mask=True, device="cpu")
    procs = model._get_logits_processor(generation_config=gc, input_ids_seq_length=len(prompt), encoder_input_ids=None,
                                        logits_processor=None, device="cpu", model_kwargs={})
    rng = np.random.default_rng(len(prompt) + n_generated)
    ids = list(prompt) + rng.integers(0, V, size=n_generated).tolist()
    out = procs(torch.tensor([ids]), torch.tensor(z, dtype=torch.float32)[None].clone())
    return out[0].numpy(), ids


CASES = [
    dict(),
    dict(repetition_penalty=1.3),
    dict(do_sample=True, temperature=0.7, top_k=10, top_p=0.9),
    dict(do_sample=True, temperature=1.3, top_k=0, top_p=0.5),
    dict(do_sample=True, top_k=200),                                  # top_k > vocab: off
    dict(do_sample=True, top_k=0, top_p=1e-6),                        # only the top id survives
    dict(do_sample=True, top_k=0, top_p=1.0),
    dict(do_sample=True, temperature=0.5, top_k=7, repetition_penalty=0.8),
    dict(min_new_tokens=4, eos_token_id=[3, 9]),
    dict(do_sample=True, top_k=5, min_new_tokens=2, eos_token_id=5, repetition_penalty=1.2),
]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("n_generated", [0, 3])
def test_processed_rows_match_transformers(tiny_llama, case, n_generated):
    gen = dict(CASES[case])
    rng = np.random.default_rng(case * 7 + n_generated)
    z = rng.standard_normal(V).astype(np.float32) * 3.0
    z[::5] = -np.abs(z[::5])                 # negative logits of seen ids are multiplied by the penalty
    prompt = rng.integers(0, V, size=6).tolist()
    want, ids = _hf_row(tiny_llama, z, prompt, n_generated, **gen)
    eos = gen.pop("eos_token_id", [])
    eos = [eos] if isinstance(eos, int) else eos
    got = R.process(z, seen=ids, penalty=gen.get("repetition_penalty", 1.0), eos_ids=eos,
                    mask_eos=n_generated < gen.get("min_new_tokens", 0), do_sample=gen.get("do_sample", False),
                    temperature=gen.get("temperature", 1.0), top_k=gen.get("top_k", 0), top_p=gen.get("top_p", 1.0))
    np.testing.assert_array_equal(np.isinf(got), np.isinf(want))
    np.testing.assert_array_equal(got[np.isfinite(got)], want[np.isfinite(want)])


def test_top_k_keeps_ties_with_the_kth_value(tiny_llama):
    z = np.zeros(V, dtype=np.float32)
    z[:3] = 5.0
    z[3:9] = 2.0                             # the 4th..9th largest tie
    want, _ = _hf_row(tiny_llama, z, [1], 0, do_sample=True, top_k=5)
    got = R.process(z, do_sample=True, top_k=5)
    assert np.isfinite(got).sum() == 9
    np.testing.assert_array_equal(got, want)


def _kernel_philox(seed, c0, c1):
    """The rounds of csrc/sampling.cuh samp_philox, in Python integers."""
    M0, M1, W0, W1, MASK = 0xD2E7470EE14C6C93, 0xCA5A826395121157, 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B, (1 << 64) - 1
    x0, x1, x2, x3, k0, k1 = c0, c1, 0, 0, seed, 0
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * x0, M1 * x2
        x0, x1, x2, x3 = ((p1 >> 64) ^ x1 ^ k0) & MASK, p1 & MASK, ((p0 >> 64) ^ x3 ^ k1) & MASK, p0 & MASK
    return x0


@pytest.mark.parametrize("seed,pos", [(0, 0), (123456789, 77), ((1 << 64) - 1, 4095)])
def test_uniforms_are_numpys_philox_stream(seed, pos):
    u = R.uniforms(seed, pos, 300)
    for tok in (0, 1, 17, 299):
        raw = int(np.random.Philox(key=seed, counter=[tok, pos, 0, 0]).random_raw())
        assert raw == _kernel_philox(seed, tok + 1, pos)
        assert u[tok] == R.uniform_one(seed, pos, tok) == (raw >> 11) / 2.0 ** 53
    assert 0.0 <= u.min() and u.max() < 1.0


def test_gumbel_draws_follow_the_softmax():
    rng = np.random.default_rng(0)
    z = (rng.standard_normal(16) * 1.5).astype(np.float32)
    kw = dict(do_sample=True, temperature=0.8, top_k=12, top_p=0.95)
    w = R.process(z, **kw)
    p = np.exp(w.astype(np.float64) - w.max())
    p /= p.sum()
    n = 24000
    counts = np.zeros(16)
    for pos in range(n):                     # one draw per position: a fixed set of counters
        counts[R.choose(z, pos, seed=42, **kw)[0]] += 1
    assert counts[p == 0].sum() == 0
    from scipy.stats import chi2
    live = p > 0
    stat = float(((counts[live] - n * p[live]) ** 2 / (n * p[live])).sum())
    assert stat < chi2.ppf(0.999, live.sum() - 1), (stat, counts, n * p)
