"""Per-step cost of the device token choice: Llama-3-8B decode (random bf16 weights) on one lane at the largest batch,
128 steps per launch, timed with CUDA events.  The settings alternate launch by launch (greedy, T=0.7/k=50/p=0.9,
k=0/p=0.9, penalty=1.1) so that clock drift spreads evenly.  Prints the card and its power limit with the numbers.

    python tests/dev/dev_sampling_perf.py [--rounds 4] [--steps 128]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

SETTINGS = {
    "greedy": dict(),
    "T0.7_k50_p0.9": dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9),
    "k0_p0.9": dict(do_sample=True, top_k=0, top_p=0.9),
    "penalty1.1": dict(repetition_penalty=1.1),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=128)
    a = ap.parse_args()
    from speech_to_speech_b200 import engine as E
    from speech_to_speech_b200.handlers.language_model_handler import LLAMA_GEOMETRIES
    eng = E.LlamaEngine(LLAMA_GEOMETRIES["llama-3-8b"], dtype="bfloat16", max_sessions=16, max_positions=1024, max_prefill=256)
    eng.init_random(0)
    B = eng.max_decode_batch()
    slots = list(range(B))
    prompt = list(range(100, 164))
    times = {k: [] for k in SETTINGS}

    def run(cfg, timed):
        for s in slots:
            eng.reset(s)
            eng.set_sampling(s, seed=s + 1, **cfg)
        first = torch.cat([eng.prefill(s, prompt)[0] for s in slots])
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        eng.decode(slots, first, a.steps)
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / a.steps

    for cfg in SETTINGS.values():   # warm-up of every setting
        run(cfg, False)
    for _ in range(a.rounds):
        for name, cfg in SETTINGS.items():
            times[name].append(run(cfg, True))
    g = min(times["greedy"])
    res = {"card": card(), "B": B, "steps": a.steps,
           "ms_per_step_min": {k: round(min(v), 4) for k, v in times.items()},
           "ms_per_step_all": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "extra_us_per_step_vs_greedy": {k: round((min(v) - g) * 1000, 1) for k, v in times.items()}}
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
