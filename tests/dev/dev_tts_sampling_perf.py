"""Cost of sampled Qwen3-TTS decoding: ms per frame at the 12 Hz geometry in bf16 (random weights), max_batch sessions on one
lane, greedy and the cousin preset alternating call by call, timed with CUDA events.  Prints the card and its power limit.
    python tests/dev/dev_tts_sampling_perf.py [frames_per_call] [calls]"""
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from speech_to_speech_b200 import engine as E                                           # noqa: E402
from speech_to_speech_b200.tts_model import CODEC_GEOMETRIES, COUSIN_SAMPLING, TTS_GEOMETRIES  # noqa: E402

frames = int(sys.argv[1]) if len(sys.argv) > 1 else 64
calls = int(sys.argv[2]) if len(sys.argv) > 2 else 6
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
eng = E.Qwen3TTSEngine(TTS_GEOMETRIES["qwen3-tts-12hz"], CODEC_GEOMETRIES["qwen3-tts-12hz"], dtype="bfloat16", max_sessions=16,
                       max_positions=frames + 64, max_text=32, codec_max_frames=41)
eng.init_random(11)
B = eng.max_batch()
slots = list(range(B))
rng = np.random.default_rng(0)
texts = [rng.integers(0, 1000, 8).tolist() for _ in slots]


def run(sampled: bool) -> float:
    for s in slots:
        eng.prefill(s, texts[s], 2301)
        if sampled:
            eng.set_sampling(s, talker=COUSIN_SAMPLING["talker"], predictor=COUSIN_SAMPLING["predictor"], seed=1000 + s)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    eng.decode_frames(slots, frames)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / frames


run(False), run(True)   # warm-up: module load, cooperative-launch set-up
times = {False: [], True: []}
for i in range(2 * calls):
    times[i % 2 == 1].append(run(i % 2 == 1))
g, s = np.array(times[False]), np.array(times[True])
print(f"card: {card}")
print(f"qwen3-tts-12hz bf16, B={B}, {frames} frames per call, {calls} calls each")
print(f"greedy        : {np.median(g):.3f} ms/frame (min {g.min():.3f}, max {g.max():.3f})")
print(f"cousin preset : {np.median(s):.3f} ms/frame (min {s.min():.3f}, max {s.max():.3f})  "
      f"+{np.median(s) - np.median(g):.3f} ms ({(np.median(s) / np.median(g) - 1) * 100:.1f} %)")
eng.close()
