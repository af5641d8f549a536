"""Record what the upstream huggingface/speech-to-speech handler helpers compute, so that the tests compare against it
without the upstream source tree.

    python tests/golden/make_reference_golden.py /path/to/speech-to-speech/src

writes tests/golden/reference_tts_helpers.npz:
  resample_<n>, int16_<n>    Qwen3TTSHandler._resample_to_pipeline_sr(x, 24000) and _to_int16 of it, x = the seeded input
                             of tests/test_oracle_tts.py (0.4 * default_rng(7).standard_normal(n), n in SIZES, drawn in order)
  resample_44k, int16_44k    the same at 44.1 kHz for 0.2 * default_rng(0).standard_normal(4410)
  budget_chunk, budget_cap, budget_len, budget_tokens
                             _estimate_max_new_tokens of the seeded random texts of tests/test_tts_handler.py
"""
import os
import sys

import numpy as np

SIZES = (1, 480, 1920, 15360, 48001)
BUDGET_CASES = ((8, 1536), (4, 700), (1, 5000))
ALPHABET = list("abcdefghij klmnop, qrst. uvw! xyz? 上海是一座城市，。") + [" "] * 6


def budget_texts():
    """(chunk, cap, text) in the order the test draws them."""
    rng = np.random.default_rng(0)
    for chunk, cap in BUDGET_CASES:
        for _ in range(200):
            yield chunk, cap, "".join(rng.choice(ALPHABET, int(rng.integers(0, 900))))


def main(src: str) -> None:
    sys.path.insert(0, src)
    from speech_to_speech.TTS.qwen3_tts_handler import Qwen3TTSHandler
    h = object.__new__(Qwen3TTSHandler)
    out = {}
    rng = np.random.default_rng(7)
    for n in SIZES:
        x = (0.4 * rng.standard_normal(n)).astype(np.float32)
        r = Qwen3TTSHandler._resample_to_pipeline_sr(h, x, 24000)
        out[f"resample_{n}"], out[f"int16_{n}"] = r, Qwen3TTSHandler._to_int16(h, r)
    x = (0.2 * np.random.default_rng(0).standard_normal(4410)).astype(np.float32)
    r = Qwen3TTSHandler._resample_to_pipeline_sr(h, x, 44100)
    out["resample_44k"], out["int16_44k"] = r, Qwen3TTSHandler._to_int16(h, r)
    rows = []
    for chunk, cap, text in budget_texts():
        h.streaming_chunk_size, h.max_new_tokens = chunk, cap
        rows.append((chunk, cap, len(text), h._estimate_max_new_tokens(text)))
    a = np.array(rows, np.int32)
    out.update(budget_chunk=a[:, 0], budget_cap=a[:, 1], budget_len=a[:, 2], budget_tokens=a[:, 3])
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_tts_helpers.npz"), **out)


if __name__ == "__main__":
    main(sys.argv[1])
