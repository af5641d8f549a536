"""Developer aid (not a test): phase timeline of the cluster decode kernel (1-2 sessions) from %globaltimer stamps."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from oracle import weights as W
from speech_to_speech_b200 import engine as E
import bench

name = sys.argv[1] if len(sys.argv) > 1 else "small"
NB = int(sys.argv[2]) if len(sys.argv) > 2 else 1
g = W.WHISPER_GEOMETRIES[name]
eng = E.WhisperEngine(g.to_dict(), max_batch=NB); eng.init_random(1)
opts = E.WhisperDecodeOptions(prefix=bench.PREFIX, eos_id=-1, max_new_tokens=16, suppress=bench.SUPPRESS, begin_suppress=bench.BEGIN_SUPPRESS)
pcm = torch.from_numpy(np.stack([W.synthetic_audio(i, 160000) for i in range(NB)])).cuda()
eng.logmel(pcm, [160000] * NB); eng.encode(NB)
for _ in range(2): eng.decode(NB, opts)
cap = 4000
tr = torch.zeros((2, cap, 6), dtype=torch.int64, device="cuda")
eng.set_trace(tr); eng.decode(NB, opts); torch.cuda.synchronize(); eng.set_trace(None)
t = tr.cpu().numpy().astype(np.int64)
L = g.dec_layers; nph = 4 * L + 2
names = ["self_blk", "cross_blk", "fc1", "fc2"]
idx = 3 * (nph - 1)
for cta in (0, 1):
    body = t[cta, :, 4] - t[cta, :, 0]; bar = t[cta, :, 5] - t[cta, :, 4]
    print(f"--- CTA {'0' if cta == 0 else 'last'}: mean over layers and 4 steps (ns)")
    for k in range(4):
        sel = [idx + s * nph + l * 4 + k for s in range(4) for l in range(L)]
        def rel(j):
            v = t[cta, sel, j]; return np.where(v > 0, v - t[cta, sel, 0], 0).mean()
        print(f"  {names[k]:10s} body {body[sel].mean():8.0f}  barrier {bar[sel].mean():8.0f}   [staged {rel(1):6.0f} | "
              f"q/k/v rows done {rel(2):6.0f} | cluster barrier 1 passed {rel(3):6.0f}]")
    sel = [idx + s * nph + 4 * L for s in range(4)]
    print(f"  {'logits':10s} body {body[sel].mean():8.0f}  barrier {bar[sel].mean():8.0f}")
    sel = [idx + s * nph + 4 * L + 1 for s in range(4)]
    print(f"  {'select':10s} body {body[sel].mean():8.0f}  barrier {bar[sel].mean():8.0f}")
    tot = t[cta, idx + 4 * nph - 1, 5] - t[cta, idx, 0]
    print(f"  4 steps: {tot / 4e3:.1f} us/step")
