"""Developer aid (not a test): what storing the Llama projections once, in the tiled layout, costs and saves.

  gemm    the prefill GEMM with a row-major bf16 operand against the tiled bf16 and tiled FP8 operands, alternating, at the
          Llama-3-8B prefill shapes for M in {64, 1024}: median ms per call over ROUNDS rounds, with the min-max spread.
  engine  a full-geometry Llama-3-8B engine (random weights), bf16 and FP8: device memory by torch.cuda.mem_get_info around
          create + init_random + finalize, device_bytes() where the library has it, prefill of 1 x 64 and 16 x 64 rows.
          Runs against any build of the library (S2S_LIB_PATH), so the parent's build can be timed the same way.
  32b     a Qwen3-32B-geometry FP8 engine with random weights: footprint, prefill of 64 rows, 16 decode steps.

Prints the card's name and power limit first; writes the numbers as JSON to the path given by --out."""
import argparse, json, os, statistics, subprocess, sys, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from oracle import weights as W
from speech_to_speech_b200 import engine as E
from speech_to_speech_b200.handlers.language_model_handler import LLAMA_GEOMETRIES

ap = argparse.ArgumentParser()
ap.add_argument("--parts", default="gemm,engine,32b")
ap.add_argument("--out", default=None)
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("dev_one_copy_perf: needs a GPU")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                      text=True, timeout=30).stdout.strip()
print(card, flush=True)
out = {"card": card}
GIB = float(1 << 30)


def timed(fn, reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


if "gemm" in args.parts:
    SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (128256, 4096)]
    res = {}
    for M in (64, 1024):
        for N, K in SHAPES:
            a = (torch.randn((M, K), device="cuda") * 0.5).to(torch.bfloat16)
            w = (torch.randn((N, K), device="cuda") / K ** 0.5).to(torch.bfloat16)
            wt, wq = E.tile_weights(w), E.tile_weights(w, "float8_e4m3")
            arms = {"row_major_bf16": lambda: E.gemm(a, w, out_dtype=torch.float32),
                    "tiled_bf16": lambda: E.gemm_tiled(a, wt, N, out_dtype=torch.float32),
                    "tiled_fp8": lambda: E.gemm_tiled(a, wq, N, "float8_e4m3", out_dtype=torch.float32)}
            reps = max(5, int(2e11 / (2 * M * N * K) + 5))
            for f in arms.values():
                timed(f, 3)
            t = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, f in arms.items():
                    t[k].append(timed(f, reps))
            res[f"M{M}_N{N}_K{K}"] = {k: spread(v) for k, v in t.items()}
            print(f"M {M:5d} N {N:6d} K {K:5d}: " + "  ".join(f"{k} {statistics.median(v):.4f} ms [{min(v):.4f}-{max(v):.4f}]"
                                                           for k, v in t.items()), flush=True)
            del a, w, wt, wq
    out["gemm_ms"] = res

if "engine" in args.parts:
    g = LLAMA_GEOMETRIES["llama-3-8b"]
    res = {}
    for fmt in (None, "float8_e4m3", None, "float8_e4m3"):
        name = fmt or "bf16"
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        eng = E.LlamaEngine(g, max_sessions=16, max_positions=256, max_prefill=1024, weight_dtype=fmt)
        eng.init_random(0)
        torch.cuda.synchronize()
        r = res.setdefault(name, {"mem_gib": [], "prefill_1x64_ms": [], "prefill_16x64_ms": []})
        r["mem_gib"].append((free0 - torch.cuda.mem_get_info()[0]) / GIB)
        if hasattr(eng.lib, "s2s_llama_device_bytes"):
            wb, tb = eng.device_bytes()
            r["device_bytes_gib"] = [wb / GIB, tb / GIB]
        prompts = [np.random.default_rng(s).integers(0, g["vocab"], 64).tolist() for s in range(16)]

        def one():
            eng.reset(0)
            eng.prefill(0, prompts[0])

        def sixteen():
            for s in range(16):
                eng.reset(s)
            eng.prefill_batch(list(range(16)), prompts)

        for f in (one, sixteen):
            f()
        for _ in range(args.rounds):
            r["prefill_1x64_ms"].append(timed(one, 10))
            r["prefill_16x64_ms"].append(timed(sixteen, 5))
        eng.close()
        del eng
        torch.cuda.synchronize()
    for name, r in res.items():
        print(f"llama-3-8b {name}: device memory {['%.2f' % m for m in r['mem_gib']]} GiB, device_bytes {r.get('device_bytes_gib')}, "
              f"prefill 1x64 {spread(r['prefill_1x64_ms'])} ms, 16x64 {spread(r['prefill_16x64_ms'])} ms", flush=True)
    out["llama_3_8b"] = res

if "32b" in args.parts:
    g = LLAMA_GEOMETRIES["qwen3-32b"]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.time()
    eng = E.LlamaEngine(g, max_sessions=4, max_positions=512, max_prefill=256, weight_dtype="float8_e4m3")
    eng.init_random(0)
    torch.cuda.synchronize()
    r = {"load_s": time.time() - t0, "mem_gib": (free0 - torch.cuda.mem_get_info()[0]) / GIB,
         "device_bytes_gib": [b / GIB for b in eng.device_bytes()], "max_decode_batch": eng.max_decode_batch()}
    prompt = np.random.default_rng(1).integers(0, g["vocab"], 64).tolist()
    pre, dec = [], []
    for _ in range(3):
        eng.reset(0)
        t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t[0].record()
        nxt, _ = eng.prefill(0, prompt)
        t[1].record()
        t[1].synchronize()
        pre.append(t[0].elapsed_time(t[1]))
        t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t[0].record()
        ids, _ = eng.decode([0], nxt, 16)
        t[1].record()
        t[1].synchronize()
        dec.append(t[0].elapsed_time(t[1]) / 16)
    r["prefill_64_ms"], r["decode_ms_per_step"], r["ids"] = spread(pre), spread(dec), ids.cpu().tolist()
    eng.close()
    print(f"qwen3-32b FP8: {r}", flush=True)
    out["qwen3_32b_fp8"] = r

if args.out:
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
