"""Developer aid (not a test): does splitting the SMs between two concurrent persistent decode launches (two "lanes", each a
cooperative grid of num_sms / lanes CTAs with its own sessions: s2s_set_sm_partition) raise the throughput of the
latency-bound TTS frame loop?  lanes = 1, 2, 3 give 132, 66 and 44 CTAs on an H100 SXM."""
import os, sys, threading, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from speech_to_speech_b200.tts_model import B200Qwen3TTS

B, NF = 16, 8


def timed(streams, jobs, reps=3):
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


for n in (1, 2, 3):
    models = []
    for i in range(2):   # lanes = 1: both engines on the full grid
        tts = B200Qwen3TTS.from_random("qwen3-tts-12hz", seed=11, dtype="bfloat16", max_sessions=B, max_positions=512, max_text=128,
                                       lane=i % n, lanes=n)
        for s in range(B):
            tts.engine.prefill(s, [3] * 20, 2301)
        tts.engine.decode_frames(list(range(B)), 26); torch.cuda.synchronize()
        models.append(tts)
    lanes = [m.engine for m in models]
    streams = [torch.cuda.Stream() for _ in lanes]
    frames = lambda i: (lambda: lanes[i].decode_frames(list(range(B)), NF))
    codec = lambda i: (lambda: lanes[i].decode_audio_batch(list(range(B)), 8, 25))
    ctas = torch.cuda.get_device_properties(0).multi_processor_count // n
    one = timed(streams, [(0, frames(0))])
    two = timed(streams, [(0, frames(0)), (1, frames(1))])
    print(f"lanes {n} ({ctas:3d} CTAs): one lane {one / NF:6.3f} ms/frame; two concurrent lanes {two / NF:6.3f} ms/frame "
          f"(-> {one / NF / 16 * 1e3:6.1f} vs {two / NF / 32 * 1e3:6.1f} us per session-frame)", flush=True)
    c1 = timed(streams, [(1, codec(1))])
    mix = timed(streams, [(0, frames(0)), (1, codec(1))])
    print(f"  codec chunk alone {c1:.2f} ms; {NF} frames alone {one:.2f} ms; both concurrently {mix:.2f} ms "
          f"(sequential sum {c1 + one:.2f} ms)", flush=True)
    for m in models:
        m.close()
