"""GPU parity tests (H100): the CUDA path, called through the C ABI, against the numpy oracle and the
transformers-generated golden vectors.

Tolerances (stated, per BASELINE.json north_star "token ids bit-exact, logits/mel within a stated fp tolerance"):
  log-mel            |err| <= 1e-4   (fp32 DFT vs fp64 FFT; values in [-1.5, 1.5])
  encoder output     |err| <= 5e-3   (fp16 GEMM operands, fp32 accumulate / residual; values O(1))
  logits             |err| <= 2e-3
  token ids          exact wherever the oracle's top-1 margin exceeds 4x the logits tolerance (random-init
                     logits are nearly flat, SURVEY.md section 7 "hard parts"); free-running ids must equal the
                     golden ids up to the first sub-margin step.
"""
import os

import numpy as np
import pytest
import torch

from oracle import weights as W, whisper_ref as R

pytestmark = pytest.mark.gpu

MEL_TOL, ENC_TOL, LOGIT_TOL = 1e-4, 5e-3, 2e-3


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _engine(E, name, max_batch=1, dtype="float16"):
    g = W.WHISPER_GEOMETRIES[name]
    w = W.make_whisper_weights(g, 0)
    eng = E.WhisperEngine(g.to_dict(), dtype=dtype, max_batch=max_batch)
    eng.load_state_dict(w)
    return g, w, eng


def _opts(E, G, max_new=None):
    return E.WhisperDecodeOptions(prefix=G["prefix"].tolist(), eos_id=int(G["eos"]),
                                  max_new_tokens=int(max_new or G["max_new"]), suppress=G["suppress"].tolist(),
                                  begin_suppress=G["begin_suppress"].tolist())


# ------------------------------------------------------------------------------------------ log-mel
@pytest.mark.parametrize("seed,n", [(0, 160000), (2, 480000), (3, 12345), (4, 500000), (5, 0), (6, 200), (7, 479999)])
def test_logmel_matches_oracle(E, seed, n):
    g, w, eng = _engine(E, "micro")
    audio = W.synthetic_audio(seed, n) if n else np.zeros(0, np.float32)
    ref = R.log_mel_spectrogram(audio, g.n_mels)
    pcm = torch.zeros((1, max(n, 8)), dtype=torch.float32, device="cuda")
    pcm[0, :n] = torch.from_numpy(audio)
    mel = eng.logmel(pcm, [n], return_mel=True)[0].cpu().numpy()
    assert np.abs(mel - ref).max() < MEL_TOL


def test_logmel_ragged_batch_and_128_mels(E):
    g = W.WHISPER_GEOMETRIES["micro"]
    geo = g.to_dict() | {"n_mels": 128}
    eng = E.WhisperEngine(geo, max_batch=3)
    lens = [160000, 40000, 480000]
    pcm = torch.zeros((3, 480000), dtype=torch.float32, device="cuda")
    auds = [W.synthetic_audio(10 + i, n) for i, n in enumerate(lens)]
    for i, a in enumerate(auds):
        pcm[i, : len(a)] = torch.from_numpy(a)
    mel = eng.logmel(pcm, lens, return_mel=True).cpu().numpy()
    for i, a in enumerate(auds):
        assert np.abs(mel[i] - R.log_mel_spectrogram(a, 128)).max() < MEL_TOL


def test_logmel_matches_transformers_golden(E, golden_dir):
    g, w, eng = _engine(E, "tiny")
    G = np.load(os.path.join(golden_dir, "whisper_tiny.npz"))
    audio = W.synthetic_audio(int(G["audio_seed"]), int(G["n_samples"]))
    mel = eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)], return_mel=True)[0].cpu().numpy()
    assert np.abs(mel[:, G["frame_idx"]] - G["mel_frames"]).max() < MEL_TOL


# ------------------------------------------------------------------------------------------ encoder / decoder
@pytest.mark.parametrize("name", ["micro", "tiny"])
def test_encoder_matches_transformers_golden(E, golden_dir, name):
    g, w, eng = _engine(E, name)
    G = np.load(os.path.join(golden_dir, f"whisper_{name}.npz"))
    audio = W.synthetic_audio(int(G["audio_seed"]), int(G["n_samples"]))
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    out = eng.encode(1, return_output=True)[0].cpu().numpy()
    assert np.isfinite(out).all()
    assert np.abs(out[G["row_idx"]] - G["enc_rows"]).max() < ENC_TOL


def test_encoder_accepts_external_mel(E, golden_dir):
    g, w, eng = _engine(E, "micro")
    audio = W.synthetic_audio(0, 160000)
    mel = R.log_mel_spectrogram(audio, g.n_mels)
    ref = R.encoder_forward(w, g, mel)
    out = eng.encode(1, mel=torch.from_numpy(mel)[None].cuda().contiguous(), return_output=True)[0].cpu().numpy()
    assert np.abs(out - ref).max() < ENC_TOL


@pytest.mark.parametrize("name", ["micro", "tiny"])
def test_decode_ids_and_logits_match_golden(E, golden_dir, name):
    g, w, eng = _engine(E, name)
    G = np.load(os.path.join(golden_dir, f"whisper_{name}.npz"))
    audio = W.synthetic_audio(int(G["audio_seed"]), int(G["n_samples"]))
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    eng.encode(1)
    opts = _opts(E, G)
    gold = G["gen_ids"]
    n = len(gold)
    forced = torch.from_numpy(np.ascontiguousarray(gold[None])).cuda().int()
    ids, lens, logits = eng.decode(1, opts, forced=forced, return_logits=True)
    ids = ids[0].cpu().numpy()
    lg = logits[:, 0].cpu().numpy()
    tv = np.take_along_axis(lg[:n], G["top_idx"][:n], 1)
    assert np.abs(tv - G["top_val"][:n]).max() < LOGIT_TOL
    assert np.isneginf(lg[0][G["suppress"]]).all() and np.isneginf(lg[0][G["begin_suppress"]]).all()
    assert np.isneginf(lg[1][G["suppress"]]).all() and np.isfinite(lg[1][G["begin_suppress"][0]])
    margin = G["top_val"][:n, 0] - G["top_val"][:n, 1]
    safe = margin > 4 * LOGIT_TOL
    assert safe.sum() >= n // 2
    assert (ids[:n][safe] == gold[safe]).all()
    # free-running greedy: identical up to the first sub-margin step
    ids2, lens2 = eng.decode(1, opts)
    ids2 = ids2[0].cpu().numpy()
    first_unsafe = int(np.argmin(safe)) if (~safe).any() else n
    assert (ids2[:first_unsafe] == gold[:first_unsafe]).all()


def test_decode_cooperative_equals_phase_by_phase(E, golden_dir, monkeypatch):
    """The persistent kernel (grid barriers) and the one-launch-per-phase debug path must agree bit for bit."""
    G = np.load(os.path.join(golden_dir, "whisper_micro.npz"))
    audio = W.synthetic_audio(0, 160000)
    outs = []
    for dbg in ("0", "1"):
        monkeypatch.setenv("S2S_DEBUG_PHASES", dbg)
        g, w, eng = _engine(E, "micro")
        eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
        eng.encode(1)
        ids, lens, logits = eng.decode(1, _opts(E, G, 6), return_logits=True)
        outs.append((ids.cpu().numpy(), logits.cpu().numpy()))
    assert (outs[0][0] == outs[1][0]).all()
    assert np.array_equal(outs[0][1], outs[1][1])


def test_batched_ragged_transcribe_matches_oracle(E, golden_dir):
    """3 utterances of different length in one call == each utterance alone == oracle (margin-aware)."""
    g, w, eng = _engine(E, "micro", max_batch=3)
    G = np.load(os.path.join(golden_dir, "whisper_micro.npz"))
    opts = _opts(E, G, 10)
    auds = [W.synthetic_audio(0, 160000), W.synthetic_audio(21, 48000), W.synthetic_audio(22, 480000)]
    batch = eng.transcribe(auds, opts)
    for i, a in enumerate(auds):
        single = eng.transcribe([a], opts)[0]
        assert single == batch[i]
        enc = R.encoder_forward(w, g, R.log_mel_spectrogram(a, g.n_mels))
        ref, lg = R.greedy_decode(w, g, enc, opts.prefix, 10, opts.eos_id, list(opts.suppress), list(opts.begin_suppress),
                                  return_logits=True)
        srt = np.sort(lg, axis=1)
        safe = (srt[:, -1] - srt[:, -2]) > 4 * LOGIT_TOL
        k = int(np.argmin(safe)) if (~safe).any() else len(ref)
        assert batch[i][:k] == ref[:k]


def test_eleven_sessions_in_one_launch_match_oracle(E, golden_dir):
    """11 sessions per persistent launch (sessions 8..10 use the upper half of the tensor-core tile): forced decode,
    per-session logits against the oracle."""
    nb = 11
    g, w, eng = _engine(E, "micro", max_batch=nb)
    G = np.load(os.path.join(golden_dir, "whisper_micro.npz"))
    opts = _opts(E, G, 5)
    auds = [W.synthetic_audio(100 + i, 160000 if i % 3 else 64000) for i in range(nb)]
    pcm = np.zeros((nb, 480000), np.float32)
    for i, a in enumerate(auds):
        pcm[i, : len(a)] = a
    eng.logmel(torch.from_numpy(pcm).cuda(), [len(a) for a in auds])
    eng.encode(nb)
    refs = []
    for a in auds:
        enc = R.encoder_forward(w, g, R.log_mel_spectrogram(a, g.n_mels))
        refs.append(R.greedy_decode(w, g, enc, opts.prefix, 5, opts.eos_id, list(opts.suppress), list(opts.begin_suppress),
                                    return_logits=True))
    forced = torch.tensor(np.stack([np.asarray(r[0][:5]) for r in refs]), dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode(nb, opts, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()  # [steps, B, vocab]
    for i, (ref_ids, ref_lg) in enumerate(refs):
        fin = np.isfinite(ref_lg)
        assert (np.isfinite(lg[:, i]) == fin).all()
        assert np.abs(lg[:, i][fin] - ref_lg[fin]).max() < LOGIT_TOL, i


def test_eos_stops_row_and_pads(E, golden_dir):
    """Make the golden's 3rd generated token the EOS id: decoding must stop there (len 3) and pad with EOS."""
    g, w, eng = _engine(E, "micro")
    G = np.load(os.path.join(golden_dir, "whisper_micro.npz"))
    audio = W.synthetic_audio(0, 160000)
    gold = G["gen_ids"]
    eos = int(gold[2])
    first = int(np.argmax(gold == eos))
    opts = E.WhisperDecodeOptions(prefix=G["prefix"].tolist(), eos_id=eos, max_new_tokens=12,
                                  suppress=G["suppress"].tolist(), begin_suppress=[220])
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    eng.encode(1)
    ids, lens = eng.decode(1, opts)
    ids = ids[0].cpu().numpy()
    assert int(lens[0]) == first + 1
    assert (ids[: first + 1] == gold[: first + 1]).all() and (ids[first + 1 :] == eos).all()


def test_detect_language_matches_oracle(E, golden_dir):
    g, w, eng = _engine(E, "micro")
    audio = W.synthetic_audio(0, 160000)
    enc = R.encoder_forward(w, g, R.log_mel_spectrogram(audio, g.n_mels))
    lang = [5, 17, 33, 250, 1000, 2047]
    ref = R.detect_language(w, g, enc, 4000, lang)
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    eng.encode(1)
    got = int(eng.detect_language(1, 4000, lang)[0])
    assert got == ref


def test_small_geometry_encoder_and_short_decode(E):
    """Whisper-small geometry (the bench configuration): encoder vs oracle + 4 teacher-forced steps."""
    g, w, eng = _engine(E, "small")
    audio = W.synthetic_audio(3, 160000)
    mel = R.log_mel_spectrogram(audio, g.n_mels)
    enc_ref = R.encoder_forward(w, g, mel)
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    out = eng.encode(1, return_output=True)[0].cpu().numpy()
    assert np.abs(out - enc_ref).max() < 2 * ENC_TOL
    prefix, eos = [50258, 50259, 50359, 50363], 50257
    ref_ids, lg_ref = R.greedy_decode(w, g, enc_ref, prefix, 4, eos, [1, 2], [220, eos], return_logits=True)
    opts = E.WhisperDecodeOptions(prefix=prefix, eos_id=eos, max_new_tokens=4, suppress=[1, 2], begin_suppress=[220, eos])
    forced = torch.tensor([ref_ids + [eos] * (4 - len(ref_ids))], dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode(1, opts, forced=forced, return_logits=True)
    lg = logits[:, 0].cpu().numpy()[: len(ref_ids)]
    fin = np.isfinite(lg_ref)
    assert np.abs(lg[fin] - lg_ref[fin]).max() < 2 * LOGIT_TOL


def test_bf16_engine_runs_and_is_close(E, golden_dir):
    g, w, eng = _engine(E, "micro", dtype="bfloat16")
    G = np.load(os.path.join(golden_dir, "whisper_micro.npz"))
    audio = W.synthetic_audio(0, 160000)
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    out = eng.encode(1, return_output=True)[0].cpu().numpy()
    assert np.abs(out[G["row_idx"]] - G["enc_rows"]).max() < 6e-2  # bf16 operands: 3 fewer mantissa bits


def test_bad_arguments_raise(E):
    from speech_to_speech_b200._lib import S2SError
    g, w, eng = _engine(E, "micro")
    with pytest.raises(S2SError):
        eng.encode(2)  # more than max_batch
    with pytest.raises(S2SError):
        eng.load_state_dict({"model.encoder.nope": np.zeros(3, np.float32)})
    eng2 = E.WhisperEngine(g.to_dict())
    with pytest.raises(S2SError):
        eng2.encode(1)  # not finalized


# ------------------------------------------------------------------------------------------ the benchmarked configuration
# Whisper-small, 4-token prompt + 128 generated tokens (131 decoder steps: 5 self-attention key blocks), the real 88-entry
# suppress list of the bench, at 1 session (cluster kernel and 8-phase kernel) and 16 sessions per launch.
def _bench_opts(E, n=128):
    import bench
    return E.WhisperDecodeOptions(prefix=bench.PREFIX, eos_id=-1, max_new_tokens=n, suppress=bench.SUPPRESS,
                                  begin_suppress=bench.BEGIN_SUPPRESS)


def _check_session_against_oracle(w, g, enc_f32, opts, ids_free, ids_forced_run, lg_gpu, tol):
    """ids_free: the engine's free-running ids; lg_gpu [n, vocab]: its logits when teacher-forced with ids_free."""
    n = opts.max_new_tokens
    ref_ids, lg_ref = R.greedy_decode(w, g, enc_f32, list(opts.prefix), n, -1, list(opts.suppress), list(opts.begin_suppress),
                                      forced=[int(t) for t in ids_free], return_logits=True)
    fin = np.isfinite(lg_ref)
    assert (np.isfinite(lg_gpu) == fin).all()                     # same ids suppressed at every step
    err = float(np.abs(lg_gpu[fin] - lg_ref[fin]).max())
    assert err < tol, err
    srt = np.sort(lg_ref, axis=1)
    safe = (srt[:, -1] - srt[:, -2]) > 4 * tol
    ref_ids = np.asarray(ref_ids)
    # teacher-forced argmax agrees wherever the oracle's margin is above the tolerance band ...
    assert (np.asarray(ids_forced_run)[safe] == ref_ids[safe]).all()
    # ... and the free run IS the oracle's greedy sequence up to the first sub-margin step (fed tokens identical until then)
    k = int(np.argmin(safe)) if (~safe).any() else n
    assert (np.asarray(ids_free)[:k] == ref_ids[:k]).all()
    return err, int(safe.sum()), k


@pytest.mark.parametrize("cluster", ["1", "0"])
def test_small_128_tokens_single_session_vs_oracle(E, monkeypatch, cluster):
    monkeypatch.setenv("S2S_WHISPER_CLUSTER", cluster)
    g, w, eng = _engine(E, "small")
    audio = W.synthetic_audio(3, 160000)
    eng.logmel(torch.from_numpy(audio)[None].cuda(), [len(audio)])
    enc = eng.encode(1, return_output=True)[0].cpu().numpy()
    opts = _bench_opts(E)
    ids, lens = eng.decode(1, opts)
    ids_free = ids[0].cpu().numpy().copy()
    assert int(lens[0]) == 128
    ids_f, _, logits = eng.decode(1, opts, forced=ids.clone(), return_logits=True)
    err, n_safe, k = _check_session_against_oracle(w, g, enc, opts, ids_free, ids_f[0].cpu().numpy(), logits[:, 0].cpu().numpy(),
                                                   LOGIT_TOL)
    assert n_safe >= 64


def test_small_128_tokens_sixteen_sessions_vs_oracle(E):
    nb = 16
    g, w, eng = _engine(E, "small", max_batch=nb)
    auds = [W.synthetic_audio(200 + i, 160000 if i % 4 else 96000) for i in range(nb)]
    pcm = np.zeros((nb, 480000), np.float32)
    for i, a in enumerate(auds):
        pcm[i, : len(a)] = a
    eng.logmel(torch.from_numpy(pcm).cuda(), [len(a) for a in auds])
    enc = eng.encode(nb, return_output=True).cpu().numpy()
    opts = _bench_opts(E)
    ids, lens = eng.decode(nb, opts)
    ids_free = ids.cpu().numpy().copy()
    ids_f, _, logits = eng.decode(nb, opts, forced=ids.clone(), return_logits=True)
    lg = logits.cpu().numpy()
    for i in (0, 7, 15):   # the numpy oracle on three of the sixteen (lower half, upper half of the tensor-core tile, last)
        _check_session_against_oracle(w, g, enc[i], opts, ids_free[i], ids_f[i].cpu().numpy(), lg[:, i], LOGIT_TOL)
    # every session alone through the single-session path gives logits within the tolerance band of its batched run
    eng1 = E.WhisperEngine(g.to_dict(), dtype="float16", max_batch=1)
    eng1.load_state_dict(w)
    for i in (3, 12):
        eng1.logmel(torch.from_numpy(auds[i])[None].cuda(), [len(auds[i])])
        eng1.encode(1)
        _, _, l1 = eng1.decode(1, opts, forced=ids[i:i + 1].clone(), return_logits=True)
        a, b = l1[:, 0].cpu().numpy(), lg[:, i]
        fin = np.isfinite(a)
        assert np.abs(a[fin] - b[fin]).max() < LOGIT_TOL


@pytest.mark.parametrize("nb", [1, 16])
def test_small_131_steps_persistent_equals_phase_by_phase(E, monkeypatch, nb):
    """Timing-perturbed rerun of the benchmarked decode: the persistent launch (grid barriers) and one launch per phase
    (kernel boundaries instead of barriers) must agree BIT FOR BIT on ids and logits -- a missing acquire/release or a
    stale read shows up here.  Both single-session kernels and the 16-session kernel."""
    g = W.WHISPER_GEOMETRIES["small"]
    w = W.make_whisper_weights(g, 0)
    auds = [W.synthetic_audio(300 + i, 160000) for i in range(nb)]
    pcm = torch.from_numpy(np.stack(auds)).cuda()
    opts = _bench_opts(E)
    modes = [("0", "1"), ("1", "1")] + ([("0", "0"), ("1", "0")] if nb == 1 else [])
    outs = {}
    for dbg, cl in modes:
        monkeypatch.setenv("S2S_DEBUG_PHASES", dbg)
        monkeypatch.setenv("S2S_WHISPER_CLUSTER", cl)
        eng = E.WhisperEngine(g.to_dict(), dtype="float16", max_batch=nb)
        eng.load_state_dict(w)
        eng.logmel(pcm, [160000] * nb)
        eng.encode(nb)
        ids, lens = eng.decode(nb, opts)
        _, _, logits = eng.decode(nb, _bench_opts(E, 16), forced=ids[:, :16].contiguous(), return_logits=True)
        outs[(dbg, cl)] = (ids.cpu().numpy().copy(), logits.cpu().numpy().copy())
        eng.close()
    for cl in {m[1] for m in modes}:
        a, b = outs[("0", cl)], outs[("1", cl)]
        assert np.array_equal(a[0], b[0]), f"ids differ between persistent and per-phase launches (cluster={cl})"
        assert np.array_equal(a[1], b[1], equal_nan=True), f"logits differ (cluster={cl})"


def test_large_v3_geometry_slice(E):
    """Whisper-large-v3 layer shapes (d 1280, 20 heads, ffn 5120, 128 mels, vocab 51866) with 2 + 2 layers: encoder vs oracle
    and 6 teacher-forced decoder steps (the 8-phase kernel with the reduced batch this geometry allows)."""
    g0 = W.WHISPER_GEOMETRIES["large-v3"]
    g = W.WhisperGeometry(g0.d_model, g0.heads, 2, 2, g0.ffn, g0.n_mels, g0.vocab, 1500, 448)
    w = W.make_whisper_weights(g, 0)
    eng = E.WhisperEngine(g.to_dict(), dtype="float16", max_batch=2)
    eng.load_state_dict(w)
    auds = [W.synthetic_audio(5, 160000), W.synthetic_audio(6, 480000)]
    pcm = np.zeros((2, 480000), np.float32)
    for i, a in enumerate(auds):
        pcm[i, : len(a)] = a
    mel = eng.logmel(torch.from_numpy(pcm).cuda(), [len(a) for a in auds], return_mel=True).cpu().numpy()
    out = eng.encode(2, return_output=True).cpu().numpy()
    prefix, eos = [50258, 50259, 50360, 50364], 50257
    opts = E.WhisperDecodeOptions(prefix=prefix, eos_id=eos, max_new_tokens=6, suppress=[1, 2, 7], begin_suppress=[220, eos])
    refs = []
    for i, a in enumerate(auds):
        mel_ref = R.log_mel_spectrogram(a, g.n_mels)
        assert np.abs(mel[i] - mel_ref).max() < 1e-4
        enc_ref = R.encoder_forward(w, g, mel_ref)
        assert np.abs(out[i] - enc_ref).max() < 2 * ENC_TOL
        refs.append(R.greedy_decode(w, g, enc_ref, prefix, 6, -1, [1, 2, 7], [220, eos], return_logits=True))
    forced = torch.tensor(np.stack([np.asarray(r[0]) for r in refs]), dtype=torch.int32, device="cuda")
    ids, lens, logits = eng.decode(2, opts, forced=forced, return_logits=True)
    lg = logits.cpu().numpy()
    for i, (rid, rlg) in enumerate(refs):
        fin = np.isfinite(rlg)
        assert np.abs(lg[:, i][fin] - rlg[fin]).max() < 2 * LOGIT_TOL, i


def test_detect_language_matches_transformers_golden_and_shares_the_encoder_pass(E, golden_dir):
    """s2s_whisper_detect_language against the language tokens transformers' detect_language chose
    (tests/golden/whisper_langdetect_micro.npz), six utterances in one batch; then transcribe_auto: detection and decode on
    ONE encoder pass with a per-utterance prompt equal detect + transcribe done separately."""
    G = np.load(os.path.join(golden_dir, "whisper_langdetect_micro.npz"))
    g, w, eng = _engine(E, "micro", max_batch=6)
    auds = [W.synthetic_audio(int(s), int(n)) for s, n in zip(G["audio_seeds"], G["n_samples"])]
    pcm = np.zeros((6, 480000), np.float32)
    for i, a in enumerate(auds):
        pcm[i, : len(a)] = a
    eng.logmel(torch.from_numpy(pcm).cuda(), [len(a) for a in auds])
    eng.encode(6)
    sot, lang = int(G["sot"]), G["lang_ids"].tolist()
    got = eng.detect_language(6, sot, lang).cpu().tolist()
    srt = np.sort(G["lang_logits"], axis=1)
    safe = (srt[:, -1] - srt[:, -2]) > 4 * LOGIT_TOL
    assert safe.sum() >= 3
    assert [a for a, s in zip(got, safe) if s] == [int(b) for b, s in zip(G["detected"], safe) if s]
    tail, eos = [sot + 20, sot + 21], g.vocab - 1
    mk = lambda langs: E.WhisperDecodeOptions(prefix=[sot, langs[0]] + tail, eos_id=eos, max_new_tokens=6, suppress=[1, 2],
                                              begin_suppress=[220], prefix_rows=[[sot, t] + tail for t in langs])
    launches0 = E.launch_count(reset=True)
    ids, langs = eng.transcribe_auto(auds, sot, lang, mk)
    n_auto = E.launch_count()
    assert langs == got
    for i in (0, 3, 5):
        o = E.WhisperDecodeOptions(prefix=[sot, langs[i]] + tail, eos_id=eos, max_new_tokens=6, suppress=[1, 2], begin_suppress=[220])
        assert eng.transcribe([auds[i]], o)[0] == ids[i]
    eng.logmel(torch.from_numpy(pcm).cuda(), [len(a) for a in auds]); eng.encode(6)
    E.launch_count(reset=True)
    eng.encode(6)
    n_encode = E.launch_count()
    assert n_auto < 2 * n_encode      # one encoder pass, not two (the round-1 handler encoded twice in auto mode)
