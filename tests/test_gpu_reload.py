"""GPU: reloading weights into an existing engine.  For weights A and B, `load(A); load(B)` and `init_random(); load(B)` must
give bit for bit what a fresh engine loaded with B gives -- every engine: codec decoder (both precisions), Qwen3-TTS (codes
and audio), Whisper (float16, bfloat16) and Llama (bfloat16, FP8 weights).  A partial reload (one tensor rebound) must equal
a fresh engine bound to the merged weights: for the codec, one SnakeBeta alpha (transformed at finalize, exactly once); for
FP8 Llama, one projection, so every other matrix is quantised again from its own dequantised values; for Whisper, the k rows
of a shared tiled q/k/v matrix and the tiled token embedding (its lookup and the tied logits), each written by the bind
alone."""
import numpy as np
import pytest
import torch

from oracle import code2wav_ref as C, qwen3tts_ref as Q, weights as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _assert_reloads(make, load, run, wa, wb, partial=None):
    """make() -> engine; load(eng, weights); run(eng) -> tuple of numpy arrays.  partial = (name, value) of one tensor."""
    fresh = make()
    load(fresh, wb)
    want = run(fresh)
    other = make()
    load(other, wa)
    assert any(not _same(x, y) for x, y in zip(run(other), want)), "weights A and B give the same output: the test sees nothing"
    load(other, wb)
    assert all(_same(x, y) for x, y in zip(run(other), want)), "load(A); load(B) differs from a fresh engine loaded with B"
    rnd = make()
    rnd.init_random(7)
    load(rnd, wb)
    assert all(_same(x, y) for x, y in zip(run(rnd), want)), "init_random(); load(B) differs from a fresh engine loaded with B"
    if partial is not None:
        name, value = partial
        merged = make()
        load(merged, {**wa, name: value})
        part = make()
        load(part, wa)
        load(part, {name: value})
        assert all(_same(x, y) for x, y in zip(run(part), run(merged))), f"rebinding only {name} differs from the merged weights"


@pytest.mark.parametrize("precision", [0, 1])
def test_codec_reload(E, precision):
    g = C.GEOMETRIES["micro"]
    codes = torch.from_numpy(np.random.default_rng(3).integers(0, g.codebook_size, (20, g.quantizers)).astype(np.int32)).cuda()
    wb = C.make_weights(g, 1)

    def run(eng):
        return eng.decode(codes, 0).cpu().numpy(), eng.decode(codes[4:18].contiguous(), 6).cpu().numpy()

    _assert_reloads(lambda: E.CodecEngine(g.to_dict(), max_frames=24, precision=precision), lambda e, w: e.load_state_dict(w),
                    run, C.make_weights(g, 0), wb, partial=("decoder.1.block.0.alpha", wb["decoder.1.block.0.alpha"]))


def test_qwen3tts_reload(E):
    g, cg = Q.GEOMETRIES["micro"], C.GEOMETRIES["micro"]
    cg = C.Code2WavGeometry(**{**cg.to_dict(), "quantizers": g.n_groups, "codebook_size": g.predictor.vocab,
                               "upsample_rates": tuple(cg.upsample_rates), "upsampling_ratios": tuple(cg.upsampling_ratios)})
    wa, wb = (Q.make_weights(g, 0), C.make_weights(cg, 0)), (Q.make_weights(g, 1), C.make_weights(cg, 1))

    def run(eng):
        eng.prefill(0, [5, 6, 7, 8, 9], 2301)
        codes = eng.decode_frames([0], 6).cpu().numpy()
        return codes, eng.decode_audio(0, 6, 25).cpu().numpy()

    _assert_reloads(lambda: E.Qwen3TTSEngine(g.to_dict(), cg.to_dict(), dtype="bfloat16", max_sessions=1, max_positions=128,
                                             max_text=64),
                    lambda e, w: e.load_state_dict(*w), run, wa, wb)


@pytest.mark.parametrize("name", ["model.decoder.layers.1.self_attn.k_proj.weight", "model.decoder.embed_tokens.weight"],
                         ids=["k_proj", "embed_tokens"])
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_whisper_reload(E, dtype, name):
    g = W.WHISPER_GEOMETRIES["micro"]
    wb = W.make_whisper_weights(g, 1)
    audio = W.synthetic_audio(0, 160000)
    eos = 4095
    opts = E.WhisperDecodeOptions(prefix=[4000, 4001, 4002, 4003], eos_id=eos, max_new_tokens=8, suppress=[1, 2],
                                  begin_suppress=[220, eos])

    def run(eng):
        eng.logmel(torch.from_numpy(audio)[None].cuda().contiguous(), [len(audio)])
        enc = eng.encode(1, return_output=True)
        ids, lens, logits = eng.decode(1, opts, return_logits=True)
        return enc.cpu().numpy(), ids.cpu().numpy(), logits.cpu().numpy()

    _assert_reloads(lambda: E.WhisperEngine(g.to_dict(), dtype=dtype), lambda e, w: e.load_state_dict(w), run,
                    W.make_whisper_weights(g, 0), wb, partial=(name, wb[name]))


@pytest.mark.parametrize("weight_dtype", [None, "float8_e4m3"], ids=["bf16", "fp8"])
def test_llama_reload(E, weight_dtype):
    g = W.LLAMA_GEOMETRIES["micro"]
    prompt = np.random.default_rng(4).integers(0, g.vocab, 23).tolist()
    wb = W.make_llama_weights(g, 1)
    name = "model.layers.0.mlp.down_proj.weight"

    def run(eng):
        eng.reset(0)
        first, logits = eng.prefill(0, prompt, return_logits=True)
        ids, _, dl = eng.decode([0], first, 12, return_logits=True)
        return logits.cpu().numpy(), ids.cpu().numpy(), dl.cpu().numpy()

    _assert_reloads(lambda: E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_positions=128, max_prefill=64, weight_dtype=weight_dtype),
                    lambda e, w: e.load_state_dict(w), run, W.make_llama_weights(g, 0), wb, partial=(name, wb[name]))
