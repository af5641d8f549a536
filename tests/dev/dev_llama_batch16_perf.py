"""Developer aid (not a test): Llama-3-8B decode on both lanes at once (two SM partitions of an H100, the benchmark's layout),
16 sessions per lane as ONE launch vs as 8 + 8 launches, 127 steps after a 64-token prompt, alternating.  Prints ms per token
step and the achieved algorithmic HBM rate (weights once per launch and step + every session's KV reads, both lanes)."""
import os, statistics, subprocess, sys, threading
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from oracle import weights as W
from speech_to_speech_b200 import engine as E

B, STEPS, PROMPT, REPS = 16, 127, 64, 4
g = W.LLAMA_GEOMETRIES["llama-3-8b"]
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip(), flush=True)
except (OSError, subprocess.SubprocessError):
    pass


def launch_bytes(n_sessions):
    d, L, f, V = g.d_model, g.layers, g.ffn, g.vocab
    qd, kvd = g.heads * g.head_dim, g.kv_heads * g.head_dim
    w = L * ((qd + 2 * kvd) * d + d * qd + 3 * f * d) * 2 + V * d * 2
    kv = sum(L * 2 * (PROMPT + s + 1) * kvd * 2 for s in range(STEPS))
    return STEPS * w + n_sessions * kv


lanes = []
for i in range(2):
    eng = E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_sessions=B, max_positions=PROMPT + STEPS + 8, max_prefill=PROMPT * 8,
                        lane=i, lanes=2)
    eng.init_random(7)
    lanes.append(eng)
assert all(e.max_decode_batch() == B for e in lanes), [e.max_decode_batch() for e in lanes]
prompt = np.random.default_rng(0).integers(0, g.vocab, PROMPT).tolist()


def run_lane(i, per_launch, out):
    eng = lanes[i]
    with E.lane_context(0, i, 2):
        for s in range(B):
            eng.reset(s)
        first = torch.cat([eng.prefill_batch(list(range(b0, b0 + 8)), [prompt] * 8) for b0 in range(0, B, 8)])
        torch.cuda.current_stream().synchronize()
        bar.wait()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for b0 in range(0, B, per_launch):
            eng.decode(list(range(b0, b0 + per_launch)), first[b0:b0 + per_launch].contiguous(), STEPS)
        t1.record()
        t1.synchronize()
        out[i] = t0.elapsed_time(t1)


res = {16: [], 8: []}
for rep in range(REPS + 1):
    for per_launch in (16, 8):
        bar = threading.Barrier(2)
        out = {}
        th = [threading.Thread(target=run_lane, args=(i, per_launch, out)) for i in range(2)]
        [t.start() for t in th]
        [t.join() for t in th]
        if rep:                                           # rep 0 warms up both shapes
            res[per_launch].append(max(out.values()))
for per_launch in (16, 8):
    ms = statistics.median(res[per_launch])
    n_launch = B // per_launch
    gbs = 2 * n_launch * launch_bytes(per_launch) / (ms / 1e3) / 1e9
    print(f"{per_launch:2d} sessions per launch x {n_launch}: {ms:8.1f} ms per lane ({ms / STEPS:6.2f} ms per step, "
          f"spread {min(res[per_launch]):.1f}-{max(res[per_launch]):.1f}), both lanes {gbs:7.0f} GB/s algorithmic", flush=True)
for e in lanes:
    e.close()
