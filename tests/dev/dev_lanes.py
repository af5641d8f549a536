"""Developer aid (not a test): does splitting the SMs between two concurrent persistent decode launches (two "lanes", each a
cooperative grid of half the SMs with its own sessions) raise the throughput of the latency-bound TTS frame loop?"""
import os, sys, threading, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from speech_to_speech_b200.tts_model import B200Qwen3TTS

B, NF = 16, 8
lanes = []
for i in range(2):
    tts = B200Qwen3TTS.from_random("qwen3-tts-12hz", seed=11, dtype="bfloat16", max_sessions=B, max_positions=512, max_text=128)
    for s in range(B):
        tts.engine.prefill(s, [3] * 20, 2301)
    tts.engine.decode_frames(list(range(B)), 26); torch.cuda.synchronize()
    lanes.append(tts.engine)
streams = [torch.cuda.Stream() for _ in lanes]

def timed(jobs, reps=3):
    """jobs: list of (lane index, callable); each runs in its own thread on its lane's stream; -> wall ms per rep"""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        bar = threading.Barrier(len(jobs) + 1)
        def run(i, fn):
            with torch.cuda.stream(streams[i]):
                bar.wait(); fn(); streams[i].synchronize()
        th = [threading.Thread(target=run, args=j) for j in jobs]
        [t.start() for t in th]
        bar.wait(); t0 = time.perf_counter()
        [t.join() for t in th]
        out.append((time.perf_counter() - t0) * 1e3)
    return min(out)

frames = lambda i: (lambda: lanes[i].decode_frames(list(range(B)), NF))
codec = lambda i: (lambda: lanes[i].decode_audio_batch(list(range(B)), 8, 25))
for ctas in (132, 66, 88, 44):
    os.environ["S2S_DECODE_CTAS"] = str(ctas)
    one = timed([(0, frames(0))])
    two = timed([(0, frames(0)), (1, frames(1))])
    print(f"ctas {ctas:3d}: one lane {one / NF:6.3f} ms/frame; two concurrent lanes {two / NF:6.3f} ms/frame "
          f"(-> {one / NF / 16 * 1e3:6.1f} vs {two / NF / 32 * 1e3:6.1f} us per session-frame)", flush=True)
os.environ["S2S_DECODE_CTAS"] = "74"
c1 = timed([(1, codec(1))])
mix = timed([(0, frames(0)), (1, codec(1))])
print(f"codec chunk alone {c1:.2f} ms; {NF} frames (74 CTAs) alone {timed([(0, frames(0))]):.2f} ms; both concurrently {mix:.2f} ms")
os.environ["S2S_DECODE_CTAS"] = "132"
print(f"full grid: frames {timed([(0, frames(0))]):.2f} ms, codec {timed([(1, codec(1))]):.2f} ms, sequential sum is the baseline")
