"""GPU parity tests (H100) of the TTS codec decoder (csrc/codec_decode.cu) through the C ABI against the numpy oracle
(oracle/code2wav_ref.py) and the golden vectors generated from transformers' Qwen3OmniMoeCode2Wav.  fp32 arithmetic on
both sides: pre-transformer output within 2e-4, waveform (values in [-1, 1]) within 1e-3 (stated tolerance; measured far
below).  Parity with the real Qwen3-TTS codec stays unpinned (upstream absent)."""
import os

import numpy as np
import pytest
import torch

from oracle import code2wav_ref as C

pytestmark = pytest.mark.gpu
# precision 0 = fp32 FMA ("parity mode"): pre-transformer output 2e-4, waveform 1e-3.
# precision 1 = fp16 tensor-core contractions with fp32 accumulation (the default): 2e-2 / 1e-2 at the micro geometry (operands
# carry 11 significant bits through ~45 contractions; waveform values lie in [-1, 1]); at the real geometry the bound comes from
# the oracle's fp16-operand emulation (test_real_geometry_slice_vs_oracle).
HID_TOLS, WAV_TOLS = {0: 2e-4, 1: 2e-2}, {0: 1e-3, 1: 1e-2}


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "fp16tc"])
def model(E, request):
    g = C.GEOMETRIES["micro"]
    w = C.make_weights(g, 0)
    eng = E.CodecEngine(g.to_dict(), max_frames=40, precision=request.param)
    eng.load_state_dict(w)
    eng.hid_tol, eng.wav_tol = HID_TOLS[request.param], WAV_TOLS[request.param]
    return g, w, eng


def _codes_dev(codes_qt):
    return torch.from_numpy(np.ascontiguousarray(codes_qt.T.astype(np.int32))).cuda()   # [T, Q] frame-major


def test_full_decode_matches_transformers_golden(model, golden_dir):
    g, w, eng = model
    G = np.load(os.path.join(golden_dir, "code2wav_micro.npz"))
    wav, hid = eng.decode(_codes_dev(G["codes"]), 0, return_hidden=True)
    assert np.abs(hid.cpu().numpy() - G["hidden"]).max() < eng.hid_tol
    got = wav.cpu().numpy()
    assert got.shape == G["wav"].shape
    assert np.abs(got - G["wav"]).max() < eng.wav_tol


def test_chunked_streaming_decode_matches_golden(model, golden_dir):
    """Qwen3OmniMoeCode2Wav.chunked_decode: chunk 8 behind 6 frames of history, history samples dropped."""
    g, w, eng = model
    G = np.load(os.path.join(golden_dir, "code2wav_micro.npz"))
    codes = G["codes"]
    chunk, left = int(G["chunk_size"]), int(G["left_context"])
    T, outs, start = codes.shape[1], [], 0
    while start < T:
        end = min(start + chunk, T)
        ctx = left if start - left > 0 else start
        outs.append(eng.decode(_codes_dev(codes[:, start - ctx:end]), ctx).cpu().numpy())
        start = end
    got = np.concatenate(outs)
    assert got.shape == G["chunked"].shape
    assert np.abs(got - G["chunked"]).max() < eng.wav_tol


@pytest.mark.parametrize("T", [1, 2, 7, 33])
def test_lengths_and_values_vs_oracle(model, T):
    g, w, eng = model
    codes = np.random.default_rng(T).integers(0, g.codebook_size, (g.quantizers, T))
    ref = C.code2wav_forward(w, g, codes)
    got = eng.decode(_codes_dev(codes), 0).cpu().numpy()
    assert got.shape == ref.shape == (eng.samples(T),)
    assert np.abs(got - ref).max() < eng.wav_tol


@pytest.mark.parametrize("precision", [0, 1])
def test_real_geometry_slice_vs_oracle(E, precision):
    """The published 12 Hz geometry (hidden 1024, 16 heads, window 72, decoder 1536, x1920) with 2 transformer layers:
    tile shapes, channel counts and the sliding window of the real model; 3 frames so the numpy oracle stays fast."""
    g0 = C.GEOMETRIES["qwen3-12hz"]
    g = C.Code2WavGeometry(**{**g0.to_dict(), "layers": 2, "upsample_rates": tuple(g0.upsample_rates),
                              "upsampling_ratios": tuple(g0.upsampling_ratios), "max_positions": 256})
    w = C.make_weights(g, 3)
    eng = E.CodecEngine(g.to_dict(), max_frames=4, precision=precision)
    eng.load_state_dict(w)
    codes = np.random.default_rng(5).integers(0, g.codebook_size, (g.quantizers, 3))
    ref, hid_ref = C.code2wav_forward(w, g, codes, return_hidden=True)
    wav, hid = eng.decode(_codes_dev(codes), 0, return_hidden=True)
    assert eng.total_upsample == 1920
    he = float(np.abs(hid.cpu().numpy() - hid_ref).max())
    got = wav.cpu().numpy()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    we = float(np.abs(got - ref).max())
    if precision == 0:
        # K up to 10752 per output at this geometry: fp32 summation-order differences reach 1.2e-3 on the waveform (measured)
        assert he < 5e-4 and we < 2e-3, f"hidden err {he:.3e} (|ref| max {np.abs(hid_ref).max():.2f}), wav err {we:.3e}"
        return
    # fp16 operands: with seeded random weights the decoder's output saturates the [-1, 1] clamp on ~45 % of the samples, so
    # operand rounding alone moves the waveform by 0.17 (the oracle with both operands of every contraction rounded to fp16 and
    # fp32 sums, `operand_rounding`).  The kernel must (a) agree with that emulation more closely than the emulation agrees
    # with fp32 -- they differ in summation order and the rounding flips it causes (measured: hidden 1.4e-3 vs 2.7e-3, waveform
    # 0.12 vs 0.17, median 1.9e-3) -- and (b) stay within twice the emulation's own distance from the fp32 reference.  (The decoder with random weights is chaotic near the clamp: single
    # samples may differ from the emulation by as much as the emulation differs from fp32; the median must stay tiny.)
    with C.operand_rounding(np.float16):
        ref16, hid16 = C.code2wav_forward(w, g, codes, return_hidden=True)
    inherent_h, inherent_w = float(np.abs(hid16 - hid_ref).max()), float(np.abs(ref16 - ref).max())
    he16, we16 = float(np.abs(hid.cpu().numpy() - hid16).max()), float(np.abs(got - ref16).max())
    med16 = float(np.median(np.abs(got - ref16)))
    msg = (f"vs fp16 emulation: hidden {he16:.3e} wav max {we16:.3e} median {med16:.3e}; vs fp32: hidden {he:.3e} wav {we:.3e}; "
           f"emulation vs fp32: {inherent_h:.3e} {inherent_w:.3e}")
    print(msg)
    assert he16 < inherent_h and med16 < 3e-3 and we16 < inherent_w, msg
    assert he < 2 * inherent_h + 1e-3 and we < 2 * inherent_w + 1e-2, msg
