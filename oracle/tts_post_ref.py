"""TTS post-processing oracle (TEST INFRASTRUCTURE): the exact calls Qwen3TTSHandler._stream makes
(speech_to_speech/TTS/qwen3_tts_handler.py:612-613, 674-680, 695-749) -- scipy's
resample_poly is the reference implementation itself, so this oracle is pinned by construction; the
restatement `resample_direct` documents the arithmetic the CUDA kernel follows and is checked against scipy."""
from __future__ import annotations

import numpy as np

PIPELINE_SR = 16000


def taps_2_3() -> np.ndarray:
    """h of scipy.signal.resample_poly(x, 2, 3) for float32 input: 2 * firwin(61, 1/3, kaiser 5.0) in float32."""
    from scipy.signal import firwin
    h = firwin(61, 1.0 / 3.0, window=("kaiser", 5.0)).astype(np.float32)
    return (h * np.float32(2)).astype(np.float32)


def resample_to_16k(audio: np.ndarray, sr: int = 24000) -> np.ndarray:
    from scipy.signal import resample_poly
    g = np.gcd(PIPELINE_SR, sr)
    return resample_poly(audio, up=PIPELINE_SR // g, down=sr // g)


def to_int16(audio: np.ndarray) -> np.ndarray:
    return np.clip(audio * 32768, -32768, 32767).astype(np.int16)


def postproc(audio24k: np.ndarray) -> np.ndarray:
    return to_int16(resample_to_16k(np.asarray(audio24k, dtype=np.float32), 24000))


def resample_direct(x: np.ndarray) -> np.ndarray:
    """y[m] = sum_j x[j] * h[3*(m+11) - 2*j - 3], float32 accumulation in increasing j (what tts_post.cu does)."""
    h = taps_2_3()
    n = len(x)
    n_out = (2 * n + 2) // 3
    y = np.zeros(n_out, np.float32)
    for m in range(n_out):
        base = 3 * (m + 11) - 3
        acc = np.float32(0)
        for j in range(max(0, (base - 60 + 1) // 2), min(n - 1, base // 2) + 1):
            acc = np.float32(acc + np.float32(x[j] * h[base - 2 * j]))
        y[m] = acc
    return y


def stream_blocks(chunks, blocksize: int = 512):
    """Leading-silence trim (40 ms preroll), 512-sample re-blocking, zero-padded tail: _stream (:722-742)."""
    found, leftover, out = False, np.array([], np.int16), []
    for c in chunks:
        a = postproc(c)
        if not found:
            above = np.abs(a) > int(32768 * 0.01)
            if not above.any():
                continue
            a = a[max(0, int(np.argmax(above)) - int(PIPELINE_SR * 0.040)):]
            found = True
        a = np.concatenate([leftover, a])
        n = (len(a) // blocksize) * blocksize
        out += [a[i:i + blocksize] for i in range(0, n, blocksize)]
        leftover = a[n:]
    if len(leftover):
        out.append(np.pad(leftover, (0, blocksize - len(leftover))))
    return out
