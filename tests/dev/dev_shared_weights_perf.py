"""Developer aid (not a test): what sharing one weight copy between two lanes (SM partitions of 66 CTAs on a 132-SM H100)
costs and saves.  Run from the repository root:  python tests/dev/dev_shared_weights_perf.py [--out results.json]

  memory   two lanes of the benchmark stack (Whisper-small, Llama-3-8B bf16 at 16 sessions x 4096 positions, Qwen3-TTS at 16
           sessions), own copies vs lane 1 sharing lane 0's weights: device_bytes / allocated_bytes (the library's count),
           and the device's used memory for information (other processes move it)
  speed    both lanes busy at once, lane 0 on the source engine and lane 1 on its own copy or on the shared one, the two arms
           alternated in blocks after warm-up: Llama-3-8B decode of 16 sessions (bf16 and FP8) in ms per step, a Qwen3-TTS
           frame of 16 sessions, a Whisper-small transcribe of 16 utterances; median (min-max) of the repetitions
  capacity two lanes of Qwen3-14B bf16 at 16 x 4096 per lane on one store: memory and one decode step per lane; the own-copy
           layout is given as weights + 2 x own state (not allocated)"""
import argparse
import gc
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from speech_to_speech_b200 import engine as E  # noqa: E402
from speech_to_speech_b200.handlers.language_model_handler import LLAMA_GEOMETRIES  # noqa: E402
from speech_to_speech_b200.handlers.whisper_stt_handler import GEOMETRIES as WHISPER_GEOMETRIES  # noqa: E402
from speech_to_speech_b200.tts_model import CODEC_GEOMETRIES, LEFT_CONTEXT_FRAMES, TTS_GEOMETRIES  # noqa: E402

GIB = float(1 << 30)
REPS = 5
RESULTS: dict = {}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def used_gib() -> float:
    free, total = torch.cuda.mem_get_info()
    return (total - free) / GIB


def both(jobs) -> float:
    """jobs: (lane, fn) pairs run at once, each on its own thread and lane stream -> wall ms until both have finished"""
    bar = threading.Barrier(len(jobs) + 1)

    def run(lane, fn):
        with E.lane_context(0, lane, 2):
            bar.wait()
            fn()
            torch.cuda.current_stream().synchronize()
    th = [threading.Thread(target=run, args=j) for j in jobs]
    [t.start() for t in th]
    bar.wait()
    t0 = time.perf_counter()
    [t.join() for t in th]
    return (time.perf_counter() - t0) * 1e3


def stat(v) -> dict:
    return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)), n=len(v))


def alternate(name, prepare, timed, arms, per=1.0):
    """prepare(arm) then timed(arm) -> ms, arms alternated in blocks of one after a warm-up of each; -> per-arm stats / per"""
    for a in arms:
        prepare(a)
        timed(a)
    out = {a: [] for a in arms}
    for _ in range(REPS):
        for a in arms:
            prepare(a)
            out[a].append(timed(a) / per)
    RESULTS[name] = {a: stat(v) for a, v in out.items()}
    print(name, {a: "%.3f (%.3f-%.3f)" % (s["median"], s["min"], s["max"]) for a, s in RESULTS[name].items()}, flush=True)


def llama(name, lane, fmt=None, sessions=16, positions=4096, seed=1, source=None):
    if source is not None:
        return source.share(lane, 2, max_sessions=sessions, max_positions=positions)
    eng = E.LlamaEngine(LLAMA_GEOMETRIES[name], max_sessions=sessions, max_positions=positions, max_prefill=512, lane=lane, lanes=2,
                        weight_dtype=fmt)
    eng.init_random(seed)
    return eng


def whisper(lane, source=None):
    if source is not None:
        return source.share(lane, 2, max_batch=16)
    eng = E.WhisperEngine(WHISPER_GEOMETRIES["small"], dtype="float16", max_batch=16, lane=lane, lanes=2)
    eng.init_random(2)
    return eng


def tts(lane, source=None):
    if source is not None:
        return source.share(lane, 2, max_sessions=16)
    eng = E.Qwen3TTSEngine(TTS_GEOMETRIES["qwen3-tts-12hz"], CODEC_GEOMETRIES["qwen3-tts-12hz"], max_sessions=16, max_positions=2048,
                           max_text=512, codec_max_frames=LEFT_CONTEXT_FRAMES + 16, lane=lane, lanes=2)
    eng.init_random(3)
    return eng


def release(*objs):
    for o in objs:
        o.close()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def memory():
    base, used0 = E.allocated_bytes(), used_gib()
    out = {}
    for arm in ("own", "shared"):
        lane0 = [whisper(0), llama("llama-3-8b", 0), tts(0)]
        lane1 = [whisper(1), llama("llama-3-8b", 1), tts(1)] if arm == "own" else \
            [whisper(1, lane0[0]), llama("llama-3-8b", 1, source=lane0[1]), tts(1, lane0[2])]
        torch.cuda.synchronize()
        db = [e.device_bytes() for e in lane0 + lane1]
        own_w = sum(w for w, _ in db[:3]) + (sum(w for w, _ in db[3:]) if arm == "own" else 0)
        out[arm] = dict(allocated_gib=(E.allocated_bytes() - base) / GIB,
                        device_bytes_gib=(own_w + sum(t - w for w, t in db)) / GIB,
                        weights_gib=own_w / GIB, mem_get_info_used_gib=used_gib() - used0,
                        per_engine_gib={k: [w / GIB, t / GIB] for k, (w, t) in zip(
                            ["whisper0", "llama0", "tts0", "whisper1", "llama1", "tts1"], db)})
        print("memory", arm, json.dumps(out[arm]), flush=True)
        release(*(lane1 + lane0))
    RESULTS["memory"] = out


def llama_speed(fmt):
    src = llama("llama-3-8b", 0, fmt, positions=1024)
    arms = {"own": llama("llama-3-8b", 1, fmt, positions=1024), "shared": llama("llama-3-8b", 1, positions=1024, source=src)}
    steps, prompts = 32, [[1 + s, 2, 3, 4, 5, 6, 7, 8] for s in range(16)]
    state = {}

    def prep(eng):
        for s in range(16):
            eng.reset(s)
        first = eng.prefill_batch(list(range(16)), prompts)
        torch.cuda.synchronize()
        return first

    def prepare(a):
        state["f0"], state["f1"] = prep(src), prep(arms[a])

    def timed(a):
        return both([(0, lambda: src.decode(list(range(16)), state["f0"], steps)),
                     (1, lambda: arms[a].decode(list(range(16)), state["f1"], steps))])
    alternate(f"llama3_8b_{fmt or 'bf16'}_decode_ms_per_step_both_lanes", prepare, timed, list(arms), per=steps)
    release(src, *arms.values())


def tts_speed():
    src = tts(0)
    arms = {"own": tts(1), "shared": tts(1, src)}
    nf = 8

    def prep(eng):
        for s in range(16):
            eng.prefill(s, [3 + s] * 20, 2301)
        torch.cuda.synchronize()

    def prepare(a):
        prep(src)
        prep(arms[a])

    def timed(a):
        return both([(0, lambda: src.decode_frames(list(range(16)), nf)), (1, lambda: arms[a].decode_frames(list(range(16)), nf))])
    alternate("tts_12hz_frame_ms_16_sessions_both_lanes", prepare, timed, list(arms), per=nf)
    release(src, *arms.values())


def whisper_speed():
    src = whisper(0)
    arms = {"own": whisper(1), "shared": whisper(1, src)}
    rng = np.random.default_rng(0)
    auds = [(0.1 * rng.standard_normal(16000 * 4)).astype(np.float32) for _ in range(16)]
    opts = E.WhisperDecodeOptions(prefix=[50258, 50259, 50359, 50363], eos_id=50257, max_new_tokens=48, suppress=[1, 2, 7],
                                  begin_suppress=[220, 50257])
    alternate("whisper_small_transcribe_ms_16_utterances_both_lanes", lambda a: None,
              lambda a: both([(0, lambda: src.transcribe(auds, opts)), (1, lambda: arms[a].transcribe(auds, opts))]), list(arms))
    release(src, *arms.values())


def capacity():
    base, used0 = E.allocated_bytes(), used_gib()
    src = llama("qwen3-14b", 0, positions=4096)
    sh = llama("qwen3-14b", 1, positions=4096, source=src)
    (w, t0), (_, t1) = src.device_bytes(), sh.device_bytes()
    first, nb = {}, min(16, src.max_decode_batch())   # sessions one decode launch carries at this geometry

    def prep(eng, k):
        for s in range(16):
            eng.reset(s)
        first[k] = eng.prefill_batch(list(range(16)), [[1 + s, 2, 3, 4] for s in range(16)])[:nb].contiguous()
        torch.cuda.synchronize()
    ms = []
    for _ in range(REPS + 1):
        prep(src, 0)
        prep(sh, 1)
        ms.append(both([(0, lambda: src.decode(list(range(nb)), first[0], 1)), (1, lambda: sh.decode(list(range(nb)), first[1], 1))]))
    RESULTS["qwen3_14b_bf16_two_lanes_16x4096"] = dict(
        weights_gib=w / GIB, own_state_gib=[(t0 - w) / GIB, (t1 - w) / GIB], shared_total_gib=(w + (t0 - w) + (t1 - w)) / GIB,
        own_copies_total_gib=(2 * w + (t0 - w) + (t1 - w)) / GIB, allocated_gib=(E.allocated_bytes() - base) / GIB,
        mem_get_info_used_gib=used_gib() - used0, max_decode_batch=[src.max_decode_batch(), sh.max_decode_batch()],
        one_step_both_lanes_ms=stat(ms[1:]))
    print("capacity", json.dumps(RESULTS["qwen3_14b_bf16_two_lanes_16x4096"]), flush=True)
    release(sh, src)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default="memory,llama,tts,whisper,capacity")
    a = ap.parse_args()
    RESULTS["card"] = card()
    print(RESULTS["card"], flush=True)
    only = a.only.split(",")
    if "memory" in only:
        memory()
    if "llama" in only:
        llama_speed(None)
        llama_speed("float8_e4m3")
    if "tts" in only:
        tts_speed()
    if "whisper" in only:
        whisper_speed()
    if "capacity" in only:
        capacity()
    RESULTS["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(RESULTS, f, indent=1)


if __name__ == "__main__":
    main()
