"""Developer aid (not a test): %globaltimer phase timeline of the TTS talker and code-predictor launches (CTA 0), per phase
kind, at the bench's geometry and batch; plus wall time per frame and per codec chunk."""
import os, sys, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from speech_to_speech_b200 import _lib
from speech_to_speech_b200.tts_model import B200Qwen3TTS
B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
tts = B200Qwen3TTS.from_random("qwen3-tts-12hz", seed=11, dtype="bfloat16", max_sessions=B, max_positions=512, max_text=128)
eng = tts.engine
lib = _lib.load()
for s in range(B):
    eng.prefill(s, [3] * 20, 2301)
eng.decode_frames(list(range(B)), 8); torch.cuda.synchronize()
for which, name, L in ((0, "talker", eng.cfg.layers), (1, "predictor", eng.cfg.cp_layers)):
    cap = 4096
    tr = torch.zeros((2, cap, 6), dtype=torch.int64, device="cuda")
    lib.s2s_qwen3tts_set_trace(eng.handle, which, tr.data_ptr(), cap)
    eng.decode_frames(list(range(B)), 1); torch.cuda.synchronize()
    lib.s2s_qwen3tts_set_trace(eng.handle, which, None, 0)
    t = tr[0].cpu().numpy()[:, [0, 4, 5]]   # CTA 0: phase begin, body end, barrier exit
    t = t[t[:, 0] > 0]
    kinds = ["qkv", "attn", "o_proj", "gate_up", "down"]   # Qwen3 q/k norm runs inside the attention items
    body, wait = {}, {}
    n_ph = 5 * L + 2
    # only phases that run are recorded: the predictor's step 0 predicts nothing and has no logits phase
    seq = [ph for ph in range(n_ph) if not (which == 1 and ph == 5 * L)] + list(range(n_ph)) * (len(t) // n_ph + 1)
    for i, row in enumerate(t):
        ph = seq[i]
        k = kinds[ph % 5] if ph < 5 * L else ("logits" if ph == 5 * L else "select")
        body.setdefault(k, []).append((row[1] - row[0]) / 1e3)
        wait.setdefault(k, []).append((row[2] - row[1]) / 1e3)
    total = (t[-1, 2] - t[0, 0]) / 1e3
    print(f"{name}: {len(t)} phases, {total:.1f} us per launch (B={B})")
    for k in kinds + ["logits", "select"]:
        if k in body:
            print(f"  {k:8s} body {np.mean(body[k]):7.2f} us  barrier {np.mean(wait[k]):6.2f} us  x{len(body[k])}")
for n in (8, 8, 8):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); eng.decode_frames(list(range(B)), n); b.record(); torch.cuda.synchronize()
    print(f"decode_frames({n}) B={B}: {a.elapsed_time(b) / n:.3f} ms per frame")
for _ in range(3):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); eng.decode_audio_batch(list(range(B)), 8, 25); b.record(); torch.cuda.synchronize()
    print(f"decode_audio_batch(8 frames, ctx {eng.history_context(0, 8, 25)}) B={B}: {a.elapsed_time(b):.2f} ms")
