"""Developer aid: Llama-3-8B prefill/decode timing on one H100 (random-init weights)."""
import os, sys, time, json
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT)
from oracle import weights as W
from speech_to_speech_b200 import engine as E
name = sys.argv[1] if len(sys.argv) > 1 else "llama-3-8b"
g = W.LLAMA_GEOMETRIES[name]
t0 = time.time()
eng = E.LlamaEngine(g.to_dict(), dtype="bfloat16", max_sessions=2, max_positions=1024, max_prefill=512); eng.init_random(1)
torch.cuda.synchronize(); print("init s", time.time() - t0)
prompt = np.random.default_rng(0).integers(0, g.vocab, 64).tolist()
def ev(): return torch.cuda.Event(enable_timing=True)
for it in range(3):
    eng.reset(0)
    a, b, c = ev(), ev(), ev()
    a.record(); nxt, _ = eng.prefill(0, prompt); b.record()
    ids, lens = eng.decode([0], nxt, 127); c.record(); torch.cuda.synchronize()
    pre, dec = a.elapsed_time(b), b.elapsed_time(c)
    wbytes = (g.layers * ((g.heads + 2 * g.kv_heads) * g.head_dim * g.d_model + g.d_model * g.heads * g.head_dim + 3 * g.ffn * g.d_model) + g.vocab * g.d_model) * 2
    print(f"iter {it}: prefill(64) {pre:.2f} ms; decode 127 tok {dec:.2f} ms = {dec/127*1e3:.1f} us/tok; weight stream {wbytes/1e9:.2f} GB/tok -> {wbytes/1e9/(dec/127/1e3):.0f} GB/s")
t = time.perf_counter(); out = eng.generate(prompt, 128); print("generate e2e ms", (time.perf_counter() - t) * 1e3, len(out))

# phase timeline (CTA 0), second token step
tr = torch.zeros((2000, 3), dtype=torch.int64, device="cuda")
eng.reset(0); nxt, _ = eng.prefill(0, prompt); eng.set_trace(tr); eng.decode([0], nxt, 4); torch.cuda.synchronize(); eng.set_trace(None)
t = tr.cpu().numpy(); nph = 5 * g.layers + 2
names = ["qkv+rope", "attn", "o_proj", "gate_up", "down"]
for k in range(5):
    sel = [nph + l * 5 + k for l in range(g.layers)]
    print(f"  {names[k]:9s} body {np.mean(t[sel,1]-t[sel,0])/1e3:8.2f} us  barrier {np.mean(t[sel,2]-t[sel,1])/1e3:6.2f} us")
print(f"  lm_head   body {(t[nph+5*g.layers,1]-t[nph+5*g.layers,0])/1e3:8.2f} us ; select {(t[nph+5*g.layers+1,1]-t[nph+5*g.layers+1,0])/1e3:6.2f} us; step {(t[2*nph-1,2]-t[nph,0])/1e3:.1f} us")
