"""GPU: sampled Qwen3-TTS decoding (talker and code predictor, csrc/qwen3tts.cu + csrc/sampling.cuh) against
tests/tts_sampling_ref.py applied to the kernel's own captured rows, with the counters of include/s2s_b200.h
s2s_qwen3tts_set_sampling: talker stream 0 at its talker position, predictor stream 1 + frame index at its predictor
position, and the talker's penalty set = the first codes kept since prefill."""
import numpy as np
import pytest
import torch

import tts_sampling_ref as T
from oracle import code2wav_ref as C, qwen3tts_ref as R, sampling_ref as S
from speech_to_speech_b200.tts_model import COUSIN_SAMPLING

pytestmark = pytest.mark.gpu

SAFE = 1e-4
TOL = {"float16": 2.5e-2, "bfloat16": 0.2}   # logits tolerances of the 16-bit engines (tests/test_gpu_qwen3tts.py)
CONFIGS = [
    COUSIN_SAMPLING,
    {"talker": dict(repetition_penalty=1.3), "predictor": None},                      # penalised greedy talker
    {"talker": None, "predictor": dict(do_sample=True, temperature=1.0, top_k=50, top_p=0.8)},
    {"talker": None, "predictor": None},                                              # greedy
]


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _micro(E, dtype, max_sessions=4):
    g, cg = R.GEOMETRIES["micro"], C.GEOMETRIES["micro"]
    cg = C.Code2WavGeometry(**{**cg.to_dict(), "quantizers": g.n_groups, "codebook_size": g.predictor.vocab,
                               "upsample_rates": tuple(cg.upsample_rates), "upsampling_ratios": tuple(cg.upsampling_ratios)})
    w, cw = R.make_weights(g, 0), C.make_weights(cg, 0)
    eng = E.Qwen3TTSEngine(g.to_dict(), cg.to_dict(), dtype=dtype, max_sessions=max_sessions, max_positions=128, max_text=64,
                           codec_precision=0)
    eng.load_state_dict(w, cw)
    return g, w, eng


def _start(eng, slot, text, speaker, cfg, seed):
    eng.prefill(slot, text, speaker)
    if cfg["talker"] is not None or cfg["predictor"] is not None:
        eng.set_sampling(slot, talker=cfg["talker"], predictor=cfg["predictor"], seed=seed)


def _check_decisions(codes, tl, pl, cfg, seed, seen0=(), forced=None):
    """codes [F, G] of one session, its rows tl [F, V] and pl [F, G, Vp]; -> (safe, total).  Asserts every safe decision."""
    tkw, pkw = T.choose_kw(cfg["talker"]), T.choose_kw(cfg["predictor"])
    kept = forced if forced is not None else codes
    seen = list(seen0)
    safe = total = 0
    for f in range(codes.shape[0]):
        pos = T.talker_position(f)
        total += 1
        if T.margin(tl[f], pos, seed=seed, seen=seen, **tkw) > SAFE:
            assert int(codes[f, 0]) == T.choose(tl[f], pos, seed=seed, seen=seen, **tkw)[0], ("talker", f)
            safe += 1
        for i in range(1, codes.shape[1]):
            p = T.predictor_position(i)
            total += 1
            if T.margin(pl[f, i], p, seed=seed, stream=1 + f, **pkw) > SAFE:
                assert int(codes[f, i]) == T.choose(pl[f, i], p, seed=seed, stream=1 + f, **pkw)[0], ("predictor", f, i)
                safe += 1
        seen.append(int(kept[f, 0]))
    return safe, total


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_mixed_launch_matches_the_oracle_on_the_kernel_rows_and_keeps_greedy_bit_identical(E, dtype):
    g, w, eng = _micro(E, dtype)
    rng = np.random.default_rng(1)
    texts = [rng.integers(0, 400, n).tolist() for n in (2, 5, 9, 3)]
    spk, F = [2301, 2302, 2303, 2301], 10
    for slot in range(4):
        _start(eng, slot, texts[slot], spk[slot], CONFIGS[slot], 100 + slot)
    codes, tl, pl = eng.decode_frames([0, 1, 2, 3], F, return_logits=True)
    codes, tl, pl = codes.cpu().numpy(), tl.cpu().numpy(), pl.cpu().numpy()
    safe = total = 0
    for b in range(4):
        s, t = _check_decisions(codes[b], tl[:, b], pl[:, :, b], CONFIGS[b], 100 + b)
        safe, total = safe + s, total + t
    print(f"{dtype}: {safe} of {total} decisions safe ({safe / total:.1%})")
    assert safe >= 0.9 * total, (safe, total)
    # the greedy session equals itself in a greedy-only launch, bit for bit
    eng.prefill(3, texts[3], spk[3])
    alone = eng.decode_frames([3], F).cpu().numpy()
    assert np.array_equal(alone[0], codes[3])
    # the sampled sessions did sample: their codes differ from a greedy run of the same prompt
    eng.prefill(0, texts[0], spk[0])
    assert not np.array_equal(eng.decode_frames([0], F).cpu().numpy()[0], codes[0])


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_teacher_forced_along_the_oracle_sampled_codes(E, dtype):
    """The fp32 oracle samples with the cousin preset; forced along its codes, every decision that is safe by 4 x TOL plus
    the sampling margin equals the oracle's -- the talker's penalty set holds the forced first codes."""
    g, w, eng = _micro(E, dtype, max_sessions=1)
    text, spk, seed, F = [7, 8, 9, 10, 11], 2302, 4242, 8
    ref = T.generate(w, g, text, spk, F, sampling=COUSIN_SAMPLING, seed=seed)
    assert len(ref) >= 4
    rec = T.replay(w, g, text, spk, ref, sampling=COUSIN_SAMPLING, seed=seed)
    _start(eng, 0, text, spk, COUSIN_SAMPLING, seed)
    forced = torch.tensor(ref[None], dtype=torch.int32, device="cuda")
    got, tl, pl = eng.decode_frames([0], len(ref), forced=forced, return_logits=True)
    got, tl, pl = got[0].cpu().numpy(), tl.cpu().numpy()[:, 0], pl.cpu().numpy()[:, :, 0]
    # the kernel's rows under teacher forcing are the oracle's rows within the logits tolerance
    err = max(float(np.nanmax(np.abs(np.where(np.isfinite(d["row"]), (tl[d["frame"]] if d["group"] == 0 else pl[d["frame"], d["group"]])
                                              - d["row"], 0.0)))) for d in rec)
    print(f"{dtype}: max |row - oracle row| {err:.3g}")
    assert err < 4 * TOL[dtype], err
    n_safe = 0
    for d in rec:
        # the decision survives a logits error of TOL when its margin (Gumbel winner gap, top-k value gap, top-p mass gap)
        # exceeds 4 x TOL
        if T.margin(d["row"], d["position"], seed=seed, seen=list(d["seen"]), stream=d["stream"], **d["kw"]) > 4 * TOL[dtype]:
            assert got[d["frame"], d["group"]] == d["choice"], (d["frame"], d["group"])
            n_safe += 1
    # few sampled decisions have a margin above 4 x TOL (the Gumbel gaps are O(1) in logit units and the top-p 0.8 mass gap
    # is a probability), so the exact check is the one below, on the kernel's own rows
    print(f"{dtype}: {n_safe} of {len(rec)} forced decisions safe against the fp32 oracle")
    # on the kernel's own rows every decision is exact, with the forced first codes as the talker's penalty set
    s_, t_ = _check_decisions(got, tl, pl, COUSIN_SAMPLING, seed, forced=ref)
    assert s_ >= 0.9 * t_, (s_, t_)


def test_invariance_seeds_and_reprefill(E):
    g, w, eng = _micro(E, "bfloat16")
    rng = np.random.default_rng(2)
    texts = [rng.integers(0, 400, n).tolist() for n in (4, 6, 2, 8)]
    cfg, F = COUSIN_SAMPLING, 7
    _start(eng, 0, texts[0], 2301, cfg, 77)
    alone = eng.decode_frames([0], F).cpu().numpy()[0]
    for slot in range(4):
        _start(eng, slot, texts[slot], 2301 + slot % 3, cfg, 77 if slot == 0 else 900 + slot)
    batch = eng.decode_frames([2, 0, 3, 1], F).cpu().numpy()
    assert np.array_equal(batch[1], alone)                       # alone == in a batch of 4 (another batch position)
    _start(eng, 0, texts[0], 2301, cfg, 77)
    split = np.concatenate([eng.decode_frames([0], 3).cpu().numpy()[0], eng.decode_frames([0], 4).cpu().numpy()[0]])
    assert np.array_equal(split, alone)                          # 3 + 4 frames == 7 frames
    _start(eng, 0, texts[0], 2301, cfg, 77)                      # re-prefill with the same seed: no stale seen id survives
    assert np.array_equal(eng.decode_frames([0], F).cpu().numpy()[0], alone)
    _start(eng, 0, texts[0], 2301, cfg, 78)
    assert not np.array_equal(eng.decode_frames([0], F).cpu().numpy()[0], alone)


def test_predictor_support_over_64_seeds(E):
    """Every predictor code of a fixed frame lies in the top-50 and top-p 0.8 set of its own row, over 64 seeds."""
    g, w, eng = _micro(E, "bfloat16", max_sessions=16)
    B = eng.max_batch()
    cfg = {"talker": None, "predictor": dict(do_sample=True, top_k=50, top_p=0.8)}
    pkw = T.choose_kw(cfg["predictor"])
    outside = checked = 0
    seeds = list(range(5000, 5064))
    for lo in range(0, 64, B):
        batch = seeds[lo:lo + B]
        for slot, seed in enumerate(batch):
            _start(eng, slot, [3, 4, 5], 2301, cfg, seed)
        codes, _, pl = eng.decode_frames(list(range(len(batch))), 1, return_logits=True)
        codes, pl = codes.cpu().numpy(), pl.cpu().numpy()
        for b in range(len(batch)):
            for i in range(1, g.n_groups):
                allowed = np.isfinite(S.process(pl[0, i, b], **pkw))
                checked += 1
                outside += int(not allowed[codes[b, 0, i]])
    assert checked == 64 * (g.n_groups - 1) and outside == 0


def test_12hz_geometry_max_batch_cousin_preset_matches_the_oracle_rows(E):
    from speech_to_speech_b200.tts_model import CODEC_GEOMETRIES, TTS_GEOMETRIES
    eng = E.Qwen3TTSEngine(TTS_GEOMETRIES["qwen3-tts-12hz"], CODEC_GEOMETRIES["qwen3-tts-12hz"], dtype="bfloat16",
                           max_sessions=16, max_positions=128, max_text=32, codec_max_frames=41)
    eng.init_random(11)
    B, F = eng.max_batch(), 8
    rng = np.random.default_rng(4)
    for slot in range(B):
        _start(eng, slot, rng.integers(0, 1000, 6).tolist(), 2301, COUSIN_SAMPLING, 31 + slot)
    codes, tl, pl = eng.decode_frames(list(range(B)), F, return_logits=True)
    codes, tl, pl = codes.cpu().numpy(), tl.cpu().numpy(), pl.cpu().numpy()
    safe = total = 0
    for b in range(B):
        s, t = _check_decisions(codes[b], tl[:, b], pl[:, :, b], COUSIN_SAMPLING, 31 + b)
        safe, total = safe + s, total + t
    print(f"12 Hz, B={B}: {safe} of {total} decisions safe ({safe / total:.1%})")
    assert safe >= 0.9 * total
    eng.close()


def test_model_object_is_reproducible_with_a_fixed_sampling_seed():
    from speech_to_speech_b200.tts_model import B200Qwen3TTS
    outs = []
    for _ in range(2):
        m = B200Qwen3TTS.from_random("micro", seed=3, dtype="bfloat16", max_positions=128, max_text=32,
                                     sampling=COUSIN_SAMPLING, sampling_seed=7)
        codes, decode = [], m.engine.decode_frames

        def record(slots, n, **kw):
            out = decode(slots, n, **kw)
            codes.append(out.cpu().numpy().copy())
            return out
        m.engine.decode_frames = record
        chunks = [np.asarray(a).copy() for a, _, _ in m.generate_custom_voice_streaming("hello there", "aiden", chunk_size=4,
                                                                                        max_new_tokens=12)]
        outs.append((np.concatenate(chunks) if chunks else np.zeros(0), np.concatenate(codes, axis=1)))
        m.close()
    assert outs[0][1].size > 0 and np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][0], outs[1][0])
