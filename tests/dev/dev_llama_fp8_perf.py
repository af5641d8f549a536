"""Developer aid (not a test): Llama-3-8B decode with bf16 and with FP8 E4M3 weights on the benchmark's two-lane layout (two SM
partitions of an H100), 1 / 8 / 16 sessions per launch, 127 steps after a 64-token prompt, device events.  One lane running
alone and both lanes at once.  The two formats do not fit the card together (two lanes x 32 GB of bf16 weights), so they
alternate in blocks: bf16, FP8, bf16, FP8, each block building its engines, warming every shape up and timing it twice.
Prints the device memory a lane's engine takes, ms per token step, the algorithmic bytes per step (weights once per launch
and step + every session's KV reads) and the rate they were streamed at."""
import os, statistics, subprocess, sys, threading
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from oracle import weights as W
from speech_to_speech_b200 import engine as E

MAX_B, STEPS, PROMPT, ROUNDS, REPS = 16, 127, 64, 2, 2
BATCHES = (1, 8, 16)
FORMATS = {"bf16": None, "fp8": "float8_e4m3"}
g = W.LLAMA_GEOMETRIES["llama-3-8b"]
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip(), flush=True)
except (OSError, subprocess.SubprocessError):
    pass
if not torch.cuda.is_available():
    sys.exit("dev_llama_fp8_perf: needs a GPU")


def step_bytes(fmt, n_sessions):
    """algorithmic bytes of one launch, averaged per token step: (weights + row scales, KV reads of the sessions)"""
    d, L, f, V = g.d_model, g.layers, g.ffn, g.vocab
    qd, kvd = g.heads * g.head_dim, g.kv_heads * g.head_dim
    elems = L * ((qd + 2 * kvd) * d + d * qd + 3 * f * d) + V * d
    rows = L * (qd + 2 * kvd + d + 2 * f + d) + V
    w = elems * 2 if fmt == "bf16" else elems + rows * 4
    kv = sum(L * 2 * (PROMPT + s + 1) * kvd * 2 for s in range(STEPS)) / STEPS
    return w, n_sessions * kv


prompt = np.random.default_rng(0).integers(0, g.vocab, PROMPT).tolist()


def run_lane(eng, i, n, bar, out):
    with E.lane_context(0, i, 2):
        for s in range(n):
            eng.reset(s)
        first = torch.cat([eng.prefill_batch(list(range(b0, min(b0 + 8, n))), [prompt] * (min(b0 + 8, n) - b0)) for b0 in range(0, n, 8)])
        torch.cuda.current_stream().synchronize()
        bar.wait()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        eng.decode(list(range(n)), first.contiguous(), STEPS)
        t1.record()
        t1.synchronize()
        out[i] = t0.elapsed_time(t1)


res, mem = {}, {}
for rnd in range(ROUNDS):
    for fmt, wd in FORMATS.items():
        lanes = []
        for i in range(2):
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            eng = E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_sessions=MAX_B, max_positions=PROMPT + STEPS + 8,
                                max_prefill=PROMPT * 8, lane=i, lanes=2, weight_dtype=wd)
            eng.init_random(7)
            torch.cuda.synchronize()
            mem.setdefault(fmt, []).append((free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30)
            lanes.append(eng)
        assert all(e.max_decode_batch() == MAX_B for e in lanes), [e.max_decode_batch() for e in lanes]
        for n in BATCHES:
            for n_lanes in (1, 2):
                for rep in range(REPS + 1):
                    bar, out = threading.Barrier(n_lanes), {}
                    th = [threading.Thread(target=run_lane, args=(lanes[i], i, n, bar, out)) for i in range(n_lanes)]
                    [t.start() for t in th]
                    [t.join() for t in th]
                    if rep:                                   # rep 0 warms the shape up
                        res.setdefault((fmt, n, n_lanes), []).append(max(out.values()) / STEPS)
        for e in lanes:
            e.close()
        del lanes, eng
        torch.cuda.empty_cache()

for fmt in FORMATS:
    print(f"{fmt}: device memory of one lane's engine {statistics.median(mem[fmt]):.2f} GiB "
          f"(range {min(mem[fmt]):.2f}-{max(mem[fmt]):.2f})", flush=True)
print("format sessions lanes | ms/step median (min-max) | GB/step per lane (weights + KV) | GB/s algorithmic, all lanes")
for n in BATCHES:
    for n_lanes in (1, 2):
        for fmt in FORMATS:
            v = res[(fmt, n, n_lanes)]
            ms = statistics.median(v)
            w, kv = step_bytes(fmt, n)
            print(f"{fmt:5s} {n:3d} {n_lanes} | {ms:7.3f} ({min(v):.3f}-{max(v):.3f}) | {w / 1e9:6.2f} + {kv / 1e9:5.3f} | "
                  f"{n_lanes * (w + kv) / (ms / 1e3) / 1e9:7.0f}", flush=True)
        b, f = statistics.median(res[("bf16", n, n_lanes)]), statistics.median(res[("fp8", n, n_lanes)])
        print(f"      {n:3d} {n_lanes} | bf16 / fp8 step time = {b / f:.2f}", flush=True)
