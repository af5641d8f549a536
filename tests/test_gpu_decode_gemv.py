"""GPU tests (H100) of the decode kernels' skinny GEMM by itself (gemv_mma / gemv_mma_chunked, their staging routines and
epilogues in csrc/decode_common.cuh, through s2s_decode_gemv), against a float64 evaluation of the same projection

    v[b][n] = sum_k W[n][k] x[b][k] (+ bias[n]),   then the epilogue (STORE, RESID, GELU, QKV, QKV_ROPE, SWIGLU, LOGITS),

at the projections of Llama-3-8B, Qwen3-14B / 32B, Whisper small / large-v3 and the Qwen3-TTS talker and code predictor,
and off the fast paths (a partial ring unit, a one-tile tail, N = 8, odd N, grids of 132, 66, 37 and 8 CTAs).

Bound per output.  Products of 16-bit operands are exact in fp32.  Let S = sum_k |W[n][k] x[b][k]| over the operands the
kernel multiplies (the staged 16-bit operand; for FP8, W = dq(Q), which bf16 holds exactly).  Then
    accumulation:               |v - ref| <= acc = 2^-16 S
    fp32 outputs (STORE, QKV q, LOGITS):     acc + 8 * 2^-24 |ref|
    RESID (out = r + v):                     acc + 8 * 2^-24 (|ref| + |r|)
    16-bit outputs (K / V cache, GELU, SwiGLU): the propagated error + u_T |value| + sub_T,
u_T = 2^-11 for fp16 and 2^-8 for bf16 (the attention tests' unit roundoff), sub_T = 2^-25 for fp16 (below the smallest
normal), 0 for bf16.  The first term is the summation order of an fp32 accumulation, as in test_gpu_codec_contract.py; the
8 * 2^-24 term the epilogue's own fp32 roundings (bias, residual, scales).  The propagated error is acc times the
epilogue's slope: exact-erf GELU has slope <= 1.13 (plus 2^-22 |v| for erff near its cancellation); SwiGLU
silu(g) * u moves by <= 1.1 acc_g |u| + |silu(g)| acc_u, and __expf's error (at most 2 + 1.173 |g| ulps) moves silu(g)
by at most that relative amount; RoPE rotates the pair (v0, v1) with the kernel's own fp32 (cos, sin) table, so the
reference rotates the float64 pair with the same table: acc0 |cos| + acc1 |sin| + 3 * 2^-24 (|v0 cos| + |v1 sin|),
times q_scale for q.

Norms are checked on the staged 16-bit operand against float64 LayerNorm / RMSNorm rounded to T.  With n = K / 64 + 8
(the per-lane sequential partial sums and the warp / CTA reductions) and u = 2^-24:
    e_mean = n u mean|x|,   e_var = n u E[x^2] + 2 |mean| e_mean,   rstd relative error <= e_var / (2 var) + 3 u,
    |y - ref| <= |w| rstd (e_mean + |x - mean| (e_var / (2 var) + 3 u)) + 3 u |ref| + u |b|, then + u_T |ref| + sub_T.
The one-pass variance's cancellation shows as e_var / var ~ n u (1 + mean^2 / var): rows with |mean| / std up to 30 are
tested.

Exact designed inputs: integer weights and sparse {-1, 0, 1} activations keep every partial sum an integer below 2^8, so
STORE, RESID, QKV, the K / V caches (rotations by (cos, sin) in {(1, 0), (0, 1), (-1, 0), (0, -1)}, q_scale 1/8) and the
logits are exact and compared bit for bit; the argmax ties are placed in main-round and tail tiles, on both rows of a pair,
across lanes, warps and CTAs, and suppressed maxima with first_step 0 and 1.

Every run fills each output buffer and KV cache with NaN first (RESID: with the residual) and checks that everything
outside the epilogue's destination comes back bit for bit; the input rows past B and the weight padding rows of a partial
last tile hold NaN.  Every case runs twice with bit-identical results.  Invariances, bit for bit: a session's row does not
depend on B or on the other sessions; ring slots 1-4, prefetch and plan_id do not change the result; FP8 equals bf16 on
dq(Q), chunked included; a drain before a projection does not change it; the DEC_NORM_L2 operand equals the one staged in
groups of 4 rows.  The worst error / bound per epilogue and format is printed at the end of the module."""
import dataclasses
import math
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SUB16 = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
ACC, OUT, U32 = 2.0 ** -16, 8 * 2.0 ** -24, 2.0 ** -24
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp8": torch.bfloat16}
NAN16 = {torch.bfloat16: 0x7FC0, torch.float16: 0x7E00}
_WORST = {}


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, r in sorted(_WORST.items()):
        print(f"\ndecode gemv {k[0]} {k[1]}: worst error / bound = {r:.3f}")


def _note(what, fmt, err, bound):
    ratio = float((err / bound).max()) if err.numel() else 0.0
    _WORST[(what, fmt)] = max(_WORST.get((what, fmt), 0.0), ratio)
    assert ratio <= 1.0, f"{what} {fmt}: error / bound {ratio:.3f}"


# ---- host mirror of gemv_make_plan_ex / gemv_chunk_ok (decode_common.cuh), CTA 0 ---------------------------------------
def plan(N, K, grid):
    n_tiles = (N + 7) // 8
    slots = grid * 8
    main = n_tiles // slots
    tail = n_tiles - main * slots
    best, best_cost = 0, 1 << 62
    for lg in range(4):
        sl = K >> lg
        if sl % 32 == 0 and sl >= 32:
            pr = grid * (8 >> lg)
            cost = -(-tail // pr) * (352 + sl)
            if cost < best_cost:
                best, best_cost = lg, cost
    stride = grid * (8 >> best)
    return (n_tiles, main, best, K >> best, -(-tail // stride) if tail > 0 else 0)


def chunk_ok(N, K, kc, grid):
    if kc <= 0 or kc % 256 or K <= kc:
        return False
    p = plan(N, kc, grid)
    last = K % kc or kc
    return p[1] == 0 and p[0] <= grid * (8 >> p[2]) and last % (32 << p[2]) == 0


# ---- operands -----------------------------------------------------------------------------------------------------------
def _untile(tiled, N8, K, fmt):
    """tiled layout (include/s2s_b200.h s2s_tile_weights) -> float64 [N8, K] of the values the kernel multiplies."""
    T = N8 // 8
    if fmt == "fp8":
        codes = tiled[: N8 * K].view(T, K // 32, 8, 4, 8).permute(0, 2, 1, 3, 4).reshape(N8, K)
        scales = tiled[N8 * K: N8 * K + 4 * N8].view(torch.float32).double()
        return codes.view(torch.float8_e4m3fn).double() * scales[:, None]
    w = tiled.view(DT[fmt]).view(T, K // 32, 8, 4, 8).permute(0, 2, 1, 3, 4).reshape(N8, K)
    return w.double()


def weights(E, N, K, fmt, gen, std=None, ints=None):
    """Random (or integer, ints = [N, K] tensor) weights of a [N, K] projection, tiled; the padding rows of a partial last
    tile hold NaN codes.  -> (tiled bytes, float64 [N, K] of what the kernel multiplies)."""
    N8 = -(-N // 8) * 8
    if ints is not None:
        w = torch.zeros(N8, K, dtype=torch.float64, device="cuda")
        w[:N] = ints
        w = w.to(DT[fmt])
    else:
        w = (torch.randn(N8, K, device="cuda", generator=gen) * (std or K ** -0.5)).to(DT[fmt])
    tiled = E.tile_weights(w.contiguous(), "float8_e4m3" if fmt == "fp8" else None)
    if N8 > N:   # poison the padding rows g >= N % 8 of the last tile
        t = tiled[: N8 * K * (1 if fmt == "fp8" else 2)]
        if fmt == "fp8":
            t.view(N8 // 8, K // 32, 8, 4, 8)[-1, :, N % 8:] = 0x7F
        else:
            t.view(torch.int16).view(N8 // 8, K // 32, 8, 4, 8)[-1, :, N % 8:] = NAN16[DT[fmt]]
    return tiled, _untile(tiled, N8, K, fmt)[:N]


def nan_like(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def same_bits(a, b):
    if a.dtype in (torch.float32, torch.int32):
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    if a.element_size() == 2:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a, b)


def outside_nan(buf, mask):
    """every element outside `mask` is still NaN"""
    return bool(torch.isnan(buf.float()[~mask]).all())


def rope_table(P, hd, theta=500000.0):
    inv = theta ** (-torch.arange(0, hd, 2, dtype=torch.float64) / hd)
    ang = torch.arange(P, dtype=torch.float64)[:, None] * inv[None]
    return torch.stack([torch.cos(ang), torch.sin(ang)], -1).float().cuda().contiguous()   # [P, hd/2, 2]


# ---- one projection ------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Proj:
    name: str
    N: int
    K: int
    mode: str
    input: str = "copy"
    llama: bool = True
    kc: int = 0
    norm: int = 2              # 1 LayerNorm, 2 RMSNorm (input "norm")
    bias: bool = False
    hd: int = 128
    q_rows: int = 0
    k_rows: int = 0
    kraw: bool = False


L8 = dict(d=4096, H=32, KV=8, ffn=14336, vocab=128256)
PROJ = {
    "l8.qkv": Proj("l8.qkv", 6144, 4096, "qkv_rope", "norm", q_rows=4096, k_rows=1024),
    "l8.o": Proj("l8.o", 4096, 4096, "resid"),
    "l8.gate_up": Proj("l8.gate_up", 28672, 4096, "swiglu", "norm"),
    "l8.down": Proj("l8.down", 4096, 14336, "resid"),
    "l8.down_kc": Proj("l8.down_kc", 4096, 14336, "resid", "chunked", kc=4096),
    "l8.lm_head": Proj("l8.lm_head", 128256, 4096, "logits", "norm"),
    "q14.qkv": Proj("q14.qkv", 7168, 5120, "qkv_rope", "norm", q_rows=5120, k_rows=1024, kraw=True),
    "q14.down_kc": Proj("q14.down_kc", 5120, 17408, "resid", "chunked", kc=5120),
    "q32.down_kc": Proj("q32.down_kc", 5120, 25600, "resid", "chunked", kc=8192),
    "ws.qkv": Proj("ws.qkv", 2304, 768, "qkv", "norm", llama=False, norm=1, bias=True),
    "ws.fc1": Proj("ws.fc1", 3072, 768, "gelu", "norm", llama=False, norm=1, bias=True),
    "ws.fc2": Proj("ws.fc2", 768, 3072, "resid", llama=False, bias=True),
    "ws.logits": Proj("ws.logits", 51865, 768, "logits", "norm", llama=False, norm=1),
    "wl.qkv": Proj("wl.qkv", 3840, 1280, "qkv", "norm", llama=False, norm=1, bias=True),
    "wl.fc1": Proj("wl.fc1", 5120, 1280, "gelu", "norm", llama=False, norm=1, bias=True),
    "wl.fc2": Proj("wl.fc2", 1280, 5120, "resid", llama=False, bias=True),
    "wl.logits": Proj("wl.logits", 51866, 1280, "logits", "norm", llama=False, norm=1),
    "tts.talker_qkv": Proj("tts.talker_qkv", 2560, 1024, "qkv_rope", "norm", q_rows=2048, k_rows=256, kraw=True),
    "tts.talker_gate_up": Proj("tts.talker_gate_up", 4096, 1024, "swiglu", "norm"),
    "tts.talker_down": Proj("tts.talker_down", 1024, 2048, "resid"),
    "tts.talker_head": Proj("tts.talker_head", 3072, 1024, "logits", "norm"),
    "tts.cp_qkv": Proj("tts.cp_qkv", 4096, 1024, "qkv_rope", "norm", q_rows=2048, k_rows=1024, kraw=True),
    "tts.cp_gate_up": Proj("tts.cp_gate_up", 6144, 1024, "swiglu", "norm"),
    "tts.cp_down": Proj("tts.cp_down", 1024, 3072, "resid"),
    "tts.cp_head": Proj("tts.cp_head", 2048, 1024, "logits", "norm"),
    # off the fast paths
    "k96": Proj("k96", 1024, 96, "store"),                        # bf16: one ring unit of 96 k (partial)
    "k800": Proj("k800", 2048, 800, "store"),                      # FP8: 512 + 288
    "n8": Proj("n8", 8, 4096, "resid"),
    "tail1": Proj("tail1", 8 * (132 * 8 + 1), 4096, "store"),     # one tile past a full main round at 132 CTAs: ks = 8
    "tail1_37": Proj("tail1_37", 8 * (37 * 8 + 1), 2048, "store"),
    "odd": Proj("odd", 1023, 512, "logits", llama=False),
    # ks = 8 split tails of three rounds, so the double-buffered reduction alternates (tail only; after a main round)
    "ks8x3": Proj("ks8x3", 8 * 21, 8192, "store"),
    "ks8x3m": Proj("ks8x3m", 8 * (8 * 8 + 21), 8192, "resid"),
}

# (projection, format, B, grid)
CASES = [
    ("l8.qkv", "bf16", 1, 132), ("l8.qkv", "fp8", 16, 132), ("l8.qkv", "fp16", 4, 66),
    ("l8.o", "bf16", 8, 132), ("l8.o", "fp8", 1, 66),
    ("l8.gate_up", "bf16", 16, 132), ("l8.gate_up", "fp8", 2, 132),
    ("l8.down", "bf16", 4, 132), ("l8.down", "fp8", 1, 132),
    ("l8.down_kc", "bf16", 8, 132), ("l8.down_kc", "fp8", 16, 66),
    ("l8.lm_head", "bf16", 16, 132), ("l8.lm_head", "fp8", 3, 132),
    ("q14.qkv", "bf16", 2, 132), ("q14.qkv", "fp8", 8, 132),
    ("q14.down_kc", "bf16", 8, 96), ("q14.down_kc", "fp8", 16, 96),
    ("q32.down_kc", "bf16", 8, 96), ("q32.down_kc", "fp8", 8, 100),
    ("ws.qkv", "fp16", 1, 132), ("ws.fc1", "fp16", 5, 132), ("ws.fc2", "fp16", 16, 132), ("ws.logits", "fp16", 3, 132),
    ("ws.logits", "bf16", 1, 37),
    ("wl.qkv", "fp16", 2, 132), ("wl.fc1", "bf16", 16, 66), ("wl.fc2", "fp16", 1, 132), ("wl.logits", "fp16", 16, 132),
    ("tts.talker_qkv", "bf16", 1, 132), ("tts.talker_gate_up", "bf16", 4, 132), ("tts.talker_down", "bf16", 4, 132),
    ("tts.talker_head", "bf16", 8, 132), ("tts.cp_qkv", "bf16", 16, 132), ("tts.cp_gate_up", "bf16", 1, 132),
    ("tts.cp_down", "bf16", 16, 132), ("tts.cp_head", "bf16", 2, 132),
    ("k96", "bf16", 3, 132), ("k800", "fp8", 3, 132), ("n8", "bf16", 16, 8), ("n8", "fp8", 1, 132),
    ("tail1", "bf16", 2, 132), ("tail1", "fp8", 16, 132), ("tail1_37", "fp8", 1, 37), ("tail1_37", "bf16", 5, 37),
    ("odd", "fp16", 7, 8), ("l8.o", "bf16", 3, 8), ("l8.o", "fp8", 5, 37), ("l8.gate_up", "fp8", 9, 66),
    ("ks8x3", "bf16", 8, 8), ("ks8x3", "fp8", 3, 8), ("ks8x3m", "bf16", 9, 8), ("ks8x3m", "fp8", 2, 8),
]


def _regime(p):
    n_tiles, main, ks, _, _ = p
    return min(main, 2), ks


def test_parametrisation_covers_the_plan_regimes():
    """main_rounds in {0, 1, >= 2} and ks_log in {0, 1, 2, 3} each occur with 16-bit and with FP8 weights, and so does a split
    tail of two or more rounds (where the reduction buffer alternates) at ks_log 2 and 3.  The planner never gives ks_log 1 a
    second tail round: 2 rounds of K/2 cost 2 * 352 + K, more than the single unsplit round's 352 + K."""
    for fam in ("16", "fp8"):
        plans = [plan(PROJ[n].N, PROJ[n].kc or PROJ[n].K, g) for n, f, _, g in CASES if (f == "fp8") == (fam == "fp8")]
        seen = [_regime(p) for p in plans]
        assert {m for m, _ in seen} == {0, 1, 2}, (fam, seen)
        assert {k for _, k in seen} == {0, 1, 2, 3}, (fam, seen)
        assert {p[2] for p in plans if p[4] >= 2} >= {2, 3}, (fam, plans)
    for n, f, _, g in CASES:
        p = PROJ[n]
        if p.input == "chunked":
            assert chunk_ok(p.N, p.K, p.kc, g), (n, g)


def norm_rg(B, K):
    """rows of the fp32 statistics copy a norm input keeps resident, as the Llama planner would choose them: all B when they
    fit next to the operand, else read from L2 (K <= 4096) or 2 rows at a time"""
    if B * K * 4 + B * (K + 32) * 2 <= 150 * 1024:
        return 0
    return -1 if K <= 4096 else 2


class Run:
    """Operands, NaN-filled outputs and the float64 reference of one projection at B sessions."""

    def __init__(self, E, p: Proj, fmt, B, gen, exact=False, mean_std=(0.0, 3.0, 30.0)):
        self.p, self.fmt, self.B, self.dt = p, fmt, B, DT[fmt]
        dt, N, K = self.dt, p.N, p.K
        self.exact = exact
        if exact:
            wi = torch.randint(-3, 4, (N, K), device="cuda", generator=gen).double()
            self.tiled, self.W = weights(E, N, K, fmt, gen, ints=wi)
        else:
            self.tiled, self.W = weights(E, N, K, fmt, gen)
        self.bias = (torch.randn(N, device="cuda", generator=gen) * 0.5).float() if p.bias else None
        if exact and p.bias:
            self.bias = torch.randint(-4, 5, (N,), device="cuda", generator=gen).float()
        self.d = dict(w=self.tiled, N=N, K=K, mode=p.mode, input=p.input)
        if self.bias is not None:
            self.d["bias"] = self.bias
        if p.input in ("copy", "chunked"):
            if exact:
                xv = torch.randint(-1, 2, (B, K), device="cuda", generator=gen).double()
                xv *= (torch.rand(B, K, device="cuda", generator=gen) < 8.0 / K)
            else:
                xv = torch.randn(B, K, device="cuda", generator=gen, dtype=torch.float64)
            self.x16 = nan_like((16, K), dt)                 # rows past B poisoned
            self.x16[:B] = xv.to(dt)
            self.d.update(x16=self.x16, kc=p.kc)
        else:
            rows = []
            for b in range(B):
                ms = mean_std[b % len(mean_std)]
                rows.append(ms + torch.randn(K, device="cuda", generator=gen, dtype=torch.float64))
            self.xf = nan_like((16, K), torch.float32)
            self.xf[:B] = torch.stack(rows).float()
            self.nw = (1.0 + 0.25 * torch.randn(K, device="cuda", generator=gen)).float()
            self.nb = (0.1 * torch.randn(K, device="cuda", generator=gen)).float()
            self.staged = nan_like((B, K), dt)
            self.d.update(xf=self.xf, norm=p.norm, norm_w=self.nw, norm_b=self.nb, eps=1e-5, rg=norm_rg(B, K), staged=self.staged)
        self._outputs(gen)

    def _outputs(self, gen):
        p, B, dt, N = self.p, self.B, self.dt, self.p.N
        m = p.mode
        if m in ("store", "resid"):
            self.out = nan_like((B + 1, N + 6), torch.float32)
            if m == "resid":
                r = torch.randn(B + 1, N + 6, device="cuda", generator=gen)
                if self.exact:
                    r = torch.randint(-50, 50, (B + 1, N + 6), device="cuda", generator=gen).float()
                self.out.copy_(r)
            self.out0 = self.out.clone()
            self.d.update(out=self.out, ldo=N + 6)
        elif m in ("gelu", "swiglu"):
            ldh = (N // 2 if m == "swiglu" else N) + 8
            self.out_h = nan_like((B + 1, ldh), dt)
            self.d.update(out_h=self.out_h, ldh=ldh)
        elif m == "qkv":
            dd = N // 3
            self.out = nan_like((B + 1, dd + 2), torch.float32)
            self.kv = nan_like((2, B + 1, dd + 4), dt)
            self.d.update(out=self.out, ldo=dd + 2, kv0=self.kv, kv_which=(B + 1) * (dd + 4), kv_batch=dd + 4, d=dd)
        elif m == "qkv_rope":
            P = 64
            kvd = p.k_rows
            self.P = P
            self.out = nan_like((B + 1, p.q_rows + 2), torch.float32)
            self.kv = nan_like((B + 2, 2, P, kvd), dt)           # slots x (K, V) x positions
            self.slot = torch.tensor([B - b for b in range(B)] + [0] * (16 - B), dtype=torch.int32, device="cuda")
            self.pos = torch.randint(0, P, (16,), dtype=torch.int32, device="cuda", generator=gen)
            if self.exact:
                q = torch.randint(0, 4, (P, p.hd // 2), device="cuda", generator=gen)
                cs = torch.tensor([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]], device="cuda")
                self.rope = cs[q].contiguous()
                q_scale = 0.125
            else:
                self.rope = rope_table(P, p.hd)
                q_scale = p.hd ** -0.5
            self.q_scale = q_scale
            self.kraw = nan_like((B + 1, p.k_rows), torch.float32) if p.kraw else None
            self.d.update(out=self.out, ldo=p.q_rows + 2, kv0=self.kv, kv_which=P * kvd, kv_slot=2 * P * kvd, kv_ld=kvd,
                          pos=self.pos, slot=self.slot, rope=self.rope, hd=p.hd, q_rows=p.q_rows, k_rows=p.k_rows,
                          q_scale=q_scale)
            if self.kraw is not None:
                self.d["kraw"] = self.kraw
        else:   # logits
            self.logits = nan_like((B + 1, N + 5), torch.float32)
            self.argmax = torch.full((16,), -7, dtype=torch.int32, device="cuda")
            self.sup = torch.zeros(N, dtype=torch.uint8, device="cuda")
            self.sup[torch.randint(0, N, (N // 50,), device="cuda", generator=gen)] = 1
            self.sup[torch.randint(0, N, (N // 50,), device="cuda", generator=gen)] |= 2
            self.first_step = B % 2   # bit 2 applies at the first step only: both occur over the parametrisation
            self.d.update(logits_out=self.logits, logits_ld=N + 5, argmax_out=self.argmax, suppress=self.sup,
                          first_step=self.first_step)

    def refill(self):
        for n, t in self.snapshot().items():
            getattr(self, n).fill_(-7 if n == "argmax" else float("nan"))
        if self.p.mode == "resid":
            self.out.copy_(self.out0)

    def snapshot(self):
        names = ("out", "out_h", "kv", "kraw", "logits", "argmax", "staged")
        return {n: getattr(self, n).clone() for n in names if getattr(self, n, None) is not None}

    def run(self, E, grid, **kw):
        return E.decode_gemv([self.d], self.B, self.dt, weight_dtype="float8_e4m3" if self.fmt == "fp8" else None,
                             llama=self.p.llama, grid=grid, **kw)[0]

    # ---- reference -----------------------------------------------------------------------------------------------------
    def operand(self):
        if self.p.input in ("copy", "chunked"):
            return self.x16[: self.B].double()
        return self.staged.double()

    def check(self):
        p, B, dt, N, fmt = self.p, self.B, self.dt, self.p.N, self.fmt
        x = self.operand()
        assert torch.isfinite(x).all()
        v = x @ self.W.T
        S = x.abs() @ self.W.abs().T
        if self.bias is not None:
            v = v + self.bias.double()
            S = S + self.bias.double().abs()
        acc = ACC * S
        if self.exact:
            acc = torch.zeros_like(acc)
        u16, sub = U16[dt], SUB16[dt]
        m = p.mode
        if m in ("store", "resid"):
            r = self.out0[:B, :N].double() if m == "resid" else torch.zeros_like(v)
            ref = r + v
            got = self.out[:B, :N].double()
            bound = acc + OUT * (ref.abs() + r.abs())
            self._cmp(m, got, ref, bound)
            mask = torch.zeros_like(self.out, dtype=torch.bool)
            mask[:B, :N] = True
            assert same_bits(self.out[~mask], self.out0[~mask])
        elif m == "gelu":
            ref = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
            got = self.out_h[:B, :N].double()
            bound = 1.13 * acc + 2.0 ** -22 * v.abs() + u16 * ref.abs() + sub
            self._cmp(m, got, ref, bound)
            mask = torch.zeros_like(self.out_h, dtype=torch.bool)
            mask[:B, :N] = True
            assert outside_nan(self.out_h, mask)
        elif m == "swiglu":
            g, u = v[:, 0::2], v[:, 1::2]
            ag, au = acc[:, 0::2], acc[:, 1::2]
            silu = g / (1 + torch.exp(-g))
            ref = silu * u
            got = self.out_h[:B, : N // 2].double()
            bound = (1.1 * ag * u.abs() + silu.abs() * au + (silu * u).abs() * ((2 + 1.173 * g.abs()) * 2.0 ** -23 + 3 * U32)
                     + u16 * ref.abs() + sub)
            self._cmp(m, got, ref, bound)
            mask = torch.zeros_like(self.out_h, dtype=torch.bool)
            mask[:B, : N // 2] = True
            assert outside_nan(self.out_h, mask)
        elif m == "qkv":
            dd = N // 3
            self._cmp("qkv", self.out[:B, :dd].double(), v[:, :dd], acc[:, :dd] + OUT * v[:, :dd].abs())
            for w in (0, 1):
                vv, aa = v[:, (w + 1) * dd:(w + 2) * dd], acc[:, (w + 1) * dd:(w + 2) * dd]
                self._cmp("qkv", self.kv[w, :B, :dd].double(), vv, aa + u16 * vv.abs() + sub)
            mo = torch.zeros_like(self.out, dtype=torch.bool)
            mo[:B, :dd] = True
            mk = torch.zeros_like(self.kv, dtype=torch.bool)
            mk[:, :B, :dd] = True
            assert outside_nan(self.out, mo) and outside_nan(self.kv, mk)
        elif m == "qkv_rope":
            self._check_rope(v, acc)
        else:
            self._check_logits(v, acc)

    def _cmp(self, what, got, ref, bound):
        assert torch.isfinite(got).all(), what
        err = (got - ref).abs()
        if self.exact:
            assert torch.equal(got, ref), (what, float(err.max()))
            return
        _note(what, self.fmt, err, bound)

    def _check_rope(self, v, acc):
        p, B, dt = self.p, self.B, self.dt
        qr, kr, kv_end = p.q_rows, p.k_rows, p.q_rows + p.k_rows
        u16, sub = U16[dt], SUB16[dt]
        pos = self.pos[:B].long()
        slot = self.slot[:B].long()
        mk = torch.zeros_like(self.kv, dtype=torch.bool)
        if p.kraw:
            self._cmp("qkv_rope", self.out[:B, :qr].double(), v[:, :qr], acc[:, :qr] + OUT * v[:, :qr].abs())
            self._cmp("qkv_rope", self.kraw[:B].double(), v[:, qr:kv_end], acc[:, qr:kv_end] + OUT * v[:, qr:kv_end].abs())
        else:
            cs = self.rope.double()[pos]                      # [B, hd/2, 2]
            rows = torch.arange(kv_end, device="cuda")
            j = (rows % p.hd)[0::2] // 2
            c, s = cs[:, j, 0], cs[:, j, 1]
            v0, v1 = v[:, 0:kv_end:2], v[:, 1:kv_end:2]
            a0, a1 = acc[:, 0:kv_end:2], acc[:, 1:kv_end:2]
            t0, t1 = v0 * c - v1 * s, v1 * c + v0 * s
            bt = a0 * c.abs() + a1 * s.abs() + 3 * U32 * (v0 * c).abs() + 3 * U32 * (v1 * s).abs()
            bt1 = a1 * c.abs() + a0 * s.abs() + 3 * U32 * (v1 * c).abs() + 3 * U32 * (v0 * s).abs()
            ref = torch.stack([t0, t1], -1).reshape(B, kv_end)
            bnd = torch.stack([bt, bt1], -1).reshape(B, kv_end)
            qs = self.q_scale
            self._cmp("qkv_rope", self.out[:B, :qr].double(), ref[:, :qr] * qs, (bnd[:, :qr] + OUT * ref[:, :qr].abs()) * qs)
            kc = self.kv[slot, 0, pos].double()              # [B, kvd]
            kref = ref[:, qr:]
            self._cmp("qkv_rope", kc, kref, bnd[:, qr:] + u16 * kref.abs() + sub)
            mk[slot, 0, pos] = True
        vref, va = v[:, kv_end:], acc[:, kv_end:]
        self._cmp("qkv_rope", self.kv[slot, 1, pos].double(), vref, va + u16 * vref.abs() + sub)
        mk[slot, 1, pos] = True
        assert outside_nan(self.kv, mk)
        mo = torch.zeros_like(self.out, dtype=torch.bool)
        mo[:B, :qr] = True
        assert outside_nan(self.out, mo)
        if p.kraw:
            mr = torch.zeros_like(self.kraw, dtype=torch.bool)
            mr[:B] = True
            assert outside_nan(self.kraw, mr)

    def _check_logits(self, v, acc):
        B, N = self.B, self.p.N
        sup = self.sup.long()
        masked = (sup & 1).bool() | ((sup & 2).bool() & bool(self.first_step))
        ref = v.masked_fill(masked[None].expand_as(v), float("-inf"))
        got = self.logits[:B, :N].double()
        fin = ~masked
        assert torch.isneginf(got[:, masked]).all()
        self._cmp("logits", got[:, fin], ref[:, fin], acc[:, fin] + OUT * ref[:, fin].abs())
        mask = torch.zeros_like(self.logits, dtype=torch.bool)
        mask[:B, :N] = True
        assert outside_nan(self.logits, mask)
        ids = self.argmax[:B].long()
        assert (self.argmax[B:] == -7).all()
        best = ref.max(1).values
        picked = ref.gather(1, ids[:, None])[:, 0]
        slack = 2 * (acc + OUT * v.abs()).max(1).values
        assert (picked >= best - slack).all(), (ids, ref.argmax(1))
        if self.exact:
            first = torch.tensor([int(torch.nonzero(ref[b] == best[b])[0]) for b in range(B)], device="cuda")
            assert torch.equal(ids, first)


@pytest.mark.parametrize("name,fmt,B,grid", CASES, ids=[f"{n}-{f}-B{b}-g{g}" for n, f, b, g in CASES])
def test_projection_against_float64(E, name, fmt, B, grid):
    p = PROJ[name]
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(f"{name}{fmt}{B}{grid}".encode()))
    r = Run(E, p, fmt, B, gen)
    pl = r.run(E, grid)
    want = plan(p.N, p.kc or p.K, grid)
    assert tuple(pl) == want, (pl, want)
    if p.input == "norm":
        check_norm(r.xf[:B], r.nw, r.nb if p.norm == 1 else None, 1e-5, p.norm, r.staged, r.dt, fmt)
    r.check()
    first = r.snapshot()
    r.refill()   # the second run starts from NaN outputs (and the same residual): a write it skips shows
    r.run(E, grid)
    for n, t in r.snapshot().items():
        assert same_bits(t, first[n]), f"second run differs: {n}"


def check_norm(x, w, b, eps, mode, staged, dt, fmt):
    """the staged 16-bit operand against float64 LayerNorm (mode 1) / RMSNorm (2), rounded to dt; bound: module docstring"""
    x = x.double()
    K = x.shape[1]
    n = K / 64 + 8
    mean = x.mean(1, keepdim=True) if mode == 1 else torch.zeros_like(x[:, :1])
    var = ((x - mean) ** 2).mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    ref = (x - mean) * rstd * w.double()
    if b is not None:
        ref = ref + b.double()
    e_mean = n * U32 * x.abs().mean(1, keepdim=True) if mode == 1 else torch.zeros_like(mean)
    e_var = n * U32 * (x * x).mean(1, keepdim=True) + 2 * mean.abs() * e_mean
    rel = e_var / (2 * (var + eps)) + 3 * U32
    bound = w.double().abs() * rstd * (e_mean + (x - mean).abs() * rel) + 3 * U32 * ref.abs()
    if b is not None:
        bound = bound + U32 * b.double().abs()
    bound = (bound + U16[dt] * ref.abs()) * (1 + U16[dt]) + SUB16[dt]
    err = (staged.double() - ref).abs()
    what = "norm" if mode == 2 else "layernorm"
    _note(what, fmt, err, bound)
    # The statistics by themselves, against norm_from_smem's claim "var accurate to ~1e-6 (1 + mean^2 / var)", i.e. rstd to
    # half that (generously 1e-6 (1 + mean^2 / var) here).  The kernel's fp32 value y32 rounded to the staged value `got`, so
    # it lies within half a unit of `got` on the side of ref: |y32 - ref| >= |ref - got| - (half that unit) is a measured
    # lower bound on the pre-rounding error, which the claimed accuracy (plus the mean's worst case and the fp32 roundings)
    # must cover.
    got = staged.double()
    mis = (got != ref.to(dt).double()) & (got != 0) & (torch.sign(got) == torch.sign(ref))
    if mis.any():
        gb = staged.view(torch.int16)
        toward = torch.where(ref.abs() > got.abs(), gb + 1, gb - 1)       # the neighbour of `got` in the direction of ref
        half = (toward.view(dt).double() - got).abs() / 2
        lower = ((ref - got).abs() - half).clamp(min=0)
        claim = (w.double().abs() * rstd * (e_mean + (x - mean).abs() * (1e-6 * (1 + mean * mean / (var + eps)) + 4 * U32))
                 + 3 * U32 * ref.abs())
        if b is not None:
            claim = claim + U32 * b.double().abs()
        _note(what + " statistics", fmt, lower[mis], claim[mis])


# ---- norms by themselves -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [128, 768, 1280, 4096, 5120])
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_norm_staging(E, d, mode, fmt):
    """rows with |mean| / std in {0, 1, 3, 10, 30, -30}, 16 sessions (8 at d >= 4096), all rows resident (d <= 1280) and in
    groups of 4 or 2; at d <= 4096 the L2 variant stages the same bits as groups of 4 rows"""
    gen = torch.Generator(device="cuda").manual_seed(d * 7 + mode)
    p = Proj("norm", 8, d, "store", "norm", llama=True, norm=mode)
    B = 16 if d <= 1280 else 8
    r = Run(E, p, fmt, B, gen, mean_std=(0.0, 1.0, 3.0, 10.0, 30.0, -30.0))
    for rg in ((0, 4) if d <= 1280 else (4,) if d <= 4096 else (2,)):
        r.d["rg"] = rg
        r.staged.fill_(float("nan"))
        r.run(E, 132)
        check_norm(r.xf[:B], r.nw, r.nb if mode == 1 else None, 1e-5, mode, r.staged, r.dt, fmt)
        r.check()
    if d <= 4096:   # after rg = 4: the L2 variant's 2 warps per row are the association of a 4-row group
        s4, o4 = r.staged.clone(), r.out.clone()
        r.d["rg"] = -1
        r.staged.fill_(float("nan"))
        r.run(E, 132)
        assert same_bits(r.staged, s4) and same_bits(r.out, o4)


@pytest.mark.parametrize("K,n_parts,B", [(768, 12, 1), (768, 12, 2), (1280, 20, 1), (384, 6, 3)])
def test_norm_sum_staging(E, K, n_parts, B):
    """stage_rows_norm_sum: x_out = ((x + add_bias) + parts[0]) + ... bit for bit against sequential fp32 adds; the staged
    operand against float64 LayerNorm of x_out"""
    gen = torch.Generator(device="cuda").manual_seed(K + n_parts + B)
    p = Proj("ns", 8, K, "store", "norm", llama=False, norm=1)
    r = Run(E, p, "fp16", B, gen)
    x = (torch.randn(B, K, device="cuda", generator=gen) * 3).float()
    parts = torch.randn(n_parts, B, K, device="cuda", generator=gen).float()
    ab = torch.randn(K, device="cuda", generator=gen).float()
    x_out = nan_like((B, K), torch.float32)
    r.d.update(input="norm_sum", xf=x.contiguous(), parts=parts, n_parts=n_parts, add_bias=ab, x_out=x_out)
    r.run(E, 37)
    acc = x.cpu().numpy() + ab.cpu().numpy()[None]
    pn = parts.cpu().numpy()
    for i in range(n_parts):
        acc = (acc + pn[i]).astype(np.float32)
    assert np.array_equal(x_out.cpu().numpy().view(np.int32), acc.view(np.int32))
    check_norm(x_out, r.nw, r.nb, 1e-5, 1, r.staged, r.dt, "fp16")


# ---- invariances ---------------------------------------------------------------------------------------------------------
def test_session_rows_do_not_depend_on_batch(E):
    gen = torch.Generator(device="cuda").manual_seed(11)
    for fmt in ("bf16", "fp8"):
        p = PROJ["l8.o"]
        tiled, _ = weights(E, p.N, p.K, fmt, gen)
        xs = torch.randn(16, p.K, device="cuda", generator=gen).bfloat16()
        other = torch.randn(16, p.K, device="cuda", generator=gen).bfloat16()
        ref = None
        ref = {}
        mixed = torch.cat([xs[:1], other[1:9], xs[9:10], other[10:]])
        for B, x in ((1, xs), (3, xs), (8, xs), (10, xs), (16, xs), (16, mixed)):
            out = nan_like((B, p.N), torch.float32)
            E.decode_gemv([dict(w=tiled, N=p.N, K=p.K, mode="store", input="copy", x16=x.contiguous(), out=out, ldo=p.N)], B,
                          torch.bfloat16, weight_dtype="float8_e4m3" if fmt == "fp8" else None, grid=132)
            for b in (0, 9):   # a session of each half of the mma's m dimension (sessions 0-7 / 8-15)
                if b < B:
                    ref.setdefault(b, out[b].clone())
                    assert same_bits(out[b], ref[b]), (fmt, B, b)


def _three(E, gen, fmt):
    """three projections of one call at 66 CTAs: QKV_ROPE with one main round and a 2-way K-split tail, SWIGLU with six main
    rounds and an unsplit tail, a tail-only LOGITS head"""
    return [Run(E, PROJ[n], fmt, 2, gen) for n in ("l8.qkv", "l8.gate_up", "tts.talker_head")]


@pytest.mark.parametrize("fmt", ["bf16", "fp8"])
def test_ring_slots_prefetch_and_plans_do_not_change_results(E, fmt):
    gen = torch.Generator(device="cuda").manual_seed(5)
    runs = _three(E, gen, fmt)
    wd = "float8_e4m3" if fmt == "fp8" else None
    base = None
    for slots in (1, 2, 3, 4):
        for prefetch in (False, True):
            for use_plans in (False, True):
                for r in runs:
                    for t in (getattr(r, n, None) for n in ("out", "out_h", "kv", "kraw", "logits", "staged")):
                        if t is not None:
                            t.fill_(float("nan"))
                E.decode_gemv([r.d for r in runs], 2, torch.bfloat16, weight_dtype=wd, grid=66, slots=slots, prefetch=prefetch,
                              use_plans=use_plans)
                snap = [r.snapshot() for r in runs]
                if base is None:
                    base = snap
                    for r in runs:
                        r.check()
                for a, b in zip(snap, base):
                    for n in a:
                        assert same_bits(a[n], b[n]), (slots, prefetch, use_plans, n)
    # each projection alone gives the same bits as inside the call, and so does a drain before the last one
    for drain in (False, True):
        for i, r in enumerate(runs):
            for t in r.snapshot():
                getattr(r, t).fill_(-7 if t == "argmax" else float("nan"))
            if drain:
                E.decode_gemv([runs[0].d, r.d], 2, torch.bfloat16, weight_dtype=wd, grid=66, drain=True)
            else:
                E.decode_gemv([r.d], 2, torch.bfloat16, weight_dtype=wd, grid=66)
            s = r.snapshot()
            for n in s:
                assert same_bits(s[n], base[i][n]), (drain, i, n)


@pytest.mark.parametrize("name,B,grid", [("l8.o", 3, 132), ("l8.gate_up", 16, 132), ("l8.down_kc", 16, 132),
                                         ("q14.down_kc", 8, 96), ("tail1", 2, 132), ("k800", 1, 8), ("l8.lm_head", 2, 132)])
def test_fp8_equals_bf16_on_dequantised_weights(E, name, B, grid):
    p = PROJ[name]
    gen = torch.Generator(device="cuda").manual_seed(3)
    r = Run(E, p, "fp8", B, gen)
    N8 = -(-p.N // 8) * 8
    dq = _untile(r.tiled, N8, p.K, "fp8").bfloat16()
    dq[p.N:] = float("nan")
    tiled16 = E.tile_weights(dq.contiguous())
    r.run(E, grid)
    a = r.snapshot()
    for n in a:
        if n != "argmax":
            getattr(r, n).fill_(float("nan"))
    if p.mode == "resid":
        r.out.copy_(r.out0)
    r.d["w"] = tiled16
    E.decode_gemv([r.d], B, torch.bfloat16, grid=grid)
    b = r.snapshot()
    for n in a:
        assert same_bits(a[n], b[n]), n


# ---- exact designed inputs -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,fmt,B,grid", [("ws.qkv", "fp16", 3, 132), ("wl.fc2", "bf16", 16, 37), ("l8.qkv", "bf16", 16, 132),
                                             ("l8.qkv", "fp8", 2, 66), ("q14.qkv", "fp8", 5, 132), ("l8.down_kc", "fp8", 8, 66),
                                             ("n8", "bf16", 16, 8), ("odd", "fp16", 16, 8)])
def test_exact_integer_projection(E, name, fmt, B, grid):
    """integer weights, sparse {-1, 0, 1} activations: every output (fp32 and the 16-bit caches) is exact"""
    p = dataclasses.replace(PROJ[name], input="copy" if PROJ[name].input == "norm" else PROJ[name].input)
    gen = torch.Generator(device="cuda").manual_seed(17)
    r = Run(E, p, fmt, B, gen, exact=True)
    r.run(E, grid)
    r.check()


def _logits_call(E, L, sup, first_step, grid, fmt="bf16", B=None):
    """logits L [B, N] (integers) through x[b] = one-hot(b), W[n][b] = L[b][n]"""
    B = B or L.shape[0]
    N = L.shape[1]
    K = 64
    wi = torch.zeros(N, K, dtype=torch.float64, device="cuda")
    wi[:, :B] = L.T
    tiled, _ = weights(E, N, K, fmt, None, ints=wi)
    x = nan_like((16, K), torch.bfloat16)
    x[:B] = torch.eye(B, K, device="cuda").bfloat16()
    out = nan_like((B, N + 3), torch.float32)
    ids = torch.full((16,), -7, dtype=torch.int32, device="cuda")
    E.decode_gemv([dict(w=tiled, N=N, K=K, mode="logits", input="copy", x16=x, suppress=sup, first_step=first_step,
                        logits_out=out, logits_ld=N + 3, argmax_out=ids)], B, torch.bfloat16,
                  weight_dtype="float8_e4m3" if fmt == "fp8" else None, grid=grid)
    return ids[:B].tolist(), out


@pytest.mark.parametrize("fmt", ["bf16", "fp8"])
def test_argmax_ties_and_suppression(E, fmt):
    N, grid = 128256, 132
    tail_base_row = plan(N, 64, grid)[1] * grid * 8 * 8
    assert 0 < tail_base_row < N - 64
    T = 5000 // 8 * 8                                       # a main-round tile's first row
    ties = [
        (5000, tail_base_row + 17),                         # main-round tile vs tail tile
        (tail_base_row + 40, tail_base_row + 41),           # both rows of a tail pair
        (777, 776),                                         # both rows of a main pair
        (T + 6, T + 1),                                     # two lanes of one tile
        (T + 8 * grid, T),                                  # same CTA, two warps (tiles T / 8 and T / 8 + grid)
        (T + 8, T + 3),                                     # neighbouring tiles: two CTAs
        (N - 1, N - 2, 3),                                  # three-way, last pair and the first tile
    ]
    B = len(ties) + 4
    gen = torch.Generator(device="cuda").manual_seed(1)
    L = torch.randint(-40, 40, (B, N), device="cuda", generator=gen).double()
    sup = torch.zeros(N, dtype=torch.uint8, device="cuda")
    for b, ids in enumerate(ties):
        for i in ids:
            L[b, i] = 100
    # suppressed maxima: bit 1 always, bit 2 only at first_step
    b1, b2, b3 = len(ties), len(ties) + 1, len(ties) + 2
    L[b1, 9000], L[b1, 9001] = 120, 110
    sup[9000] = 1
    L[b2, 12345], L[b2, 70000] = 120, 110
    sup[12345] = 2
    L[b3, tail_base_row + 3] = 100
    b4 = len(ties) + 3                                      # bit 2 on an even id (the first row of a pair)
    L[b4, 20000], L[b4, 30001] = 120, 110
    sup[20000] = 2
    for first_step in (0, 1):
        got, out = _logits_call(E, L, sup, first_step, grid, fmt)
        want = [min(t) for t in ties] + [9001, 70000 if first_step else 12345, tail_base_row + 3, 30001 if first_step else 20000]
        assert got == want, (first_step, got, want)
        assert torch.isneginf(out[:, 9000]).all()
        assert torch.isneginf(out[:, 12345]).all() == bool(first_step)
        assert torch.isneginf(out[:, 20000]).all() == bool(first_step)
        assert torch.isnan(out[:, N:]).all()


def test_argmax_all_but_one_suppressed(E):
    """odd N (a partial last tile): every id but the last suppressed -> the last id wins although its logit is the lowest"""
    N = 51865
    gen = torch.Generator(device="cuda").manual_seed(2)
    L = torch.randint(-40, 40, (4, N), device="cuda", generator=gen).double()
    L[:, N - 1] = -100
    sup = torch.ones(N, dtype=torch.uint8, device="cuda")
    sup[N - 1] = 0
    for grid in (132, 37):
        got, out = _logits_call(E, L, sup, 0, grid)
        assert got == [N - 1] * 4
        assert (out[:, N - 1] == -100).all() and torch.isneginf(out[:, : N - 1]).all() and torch.isnan(out[:, N:]).all()


def test_argmax_all_nan_row_gives_a_valid_id(E):
    """a session whose logits are all NaN (a NaN input row) gets id 0 -- NaN counts as -inf, so nothing beats the lowest id
    -- and the other sessions keep their argmax"""
    N, K, B = 128256, 64, 3
    gen = torch.Generator(device="cuda").manual_seed(3)
    wi = torch.randint(-8, 9, (N, K), device="cuda", generator=gen).double()
    tiled, _ = weights(E, N, K, "bf16", None, ints=wi)
    x = nan_like((16, K), torch.bfloat16)
    x[:B] = torch.randint(-1, 2, (B, K), device="cuda", generator=gen).bfloat16()
    x[1] = float("nan")
    for grid in (132, 37):
        out = nan_like((B, N), torch.float32)
        ids = torch.full((16,), -7, dtype=torch.int32, device="cuda")
        E.decode_gemv([dict(w=tiled, N=N, K=K, mode="logits", input="copy", x16=x, logits_out=out, logits_ld=N, argmax_out=ids)],
                      B, torch.bfloat16, grid=grid)
        ref = x[:B].double() @ wi.T
        assert torch.isnan(out[1]).all()
        assert ids[:B].tolist() == [int(ref[0].argmax()), 0, int(ref[2].argmax())], ids[:B].tolist()


# ---- arguments the entry point rejects -----------------------------------------------------------------------------------
def test_rejects_bad_arguments(E):
    from speech_to_speech_b200._lib import S2SError
    gen = torch.Generator(device="cuda").manual_seed(0)
    tiled, _ = weights(E, 64, 256, "bf16", gen)
    x = torch.zeros(16, 256, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(16, 64, device="cuda")
    ok = dict(w=tiled, N=64, K=256, mode="store", input="copy", x16=x, out=out, ldo=64)
    E.decode_gemv([ok], 2, torch.bfloat16, grid=8)
    bias = torch.zeros(64, device="cuda")
    bad = [
        (dict(ok, K=240), 2, {}),                                   # K % 32
        (ok, 0, {}), (ok, 17, {}),                                  # B
        (ok, 2, dict(weight_dtype="float8_e4m3", llama=False)),     # FP8 outside the Llama family
        (dict(ok, mode="gelu"), 2, {}),                             # not in the Llama-family instantiation
        (dict(ok, mode="swiglu"), 2, dict(llama=False)),            # not in the Whisper instantiation
        (dict(ok, input="chunked", kc=128), 2, {}),                 # kc fails gemv_chunk_ok
        (dict(ok, N=63), 2, {}),                                    # odd N outside LOGITS
        (dict(ok, N=63, mode="logits", argmax_out=torch.zeros(16, dtype=torch.int32, device="cuda"), bias=bias), 2,
         dict(llama=False)),                                        # a bias with odd N
    ]
    bad += [
        (dict(ok, mode="gelu", out_h=x, ldh=63), 2, dict(llama=False)),          # GELU stores 16-bit pairs: ldh must be even
        (dict(ok, out=out.view(-1)[1:]), 2, {}),                                   # out not 8-byte aligned (float2 stores)
        (dict(ok, mode="qkv", N=96, K=256, d=32, kv0=x, kv_which=1001, kv_batch=64), 2, dict(llama=False)),   # odd cache stride
        (dict(ok, head_plan=2, N=256), 2, dict(llama=False)),                    # a head plan without virtual clusters
        (ok, 2, dict(cluster=3)),                                                # 8 CTAs are not a whole number of 3-CTA clusters
    ]
    for d, B, kw in bad:
        with pytest.raises(S2SError):
            E.decode_gemv([d], B, torch.float16 if kw.get("llama") is False and "weight_dtype" not in kw else torch.bfloat16,
                          grid=8, **kw)
    with pytest.raises(S2SError):
        E.decode_gemv([ok], 2, torch.float16, weight_dtype="float8_e4m3", grid=8)   # FP8 with fp16


# ---- the cluster kernel's per-head plans (gemv_head_plan) on virtual clusters ----------------------------------------------
@pytest.mark.parametrize("grid,heads", [(96, 12), (104, 12), (96, 11)])
@pytest.mark.parametrize("name,kind", [("ws.qkv", 1), ("ws.q", 2)])
def test_head_plans_write_exactly_their_heads_rows(E, name, kind, grid, heads):
    """Whisper small (12 heads of 64) on clusters of 8 CTAs, as the single-session kernel cuts its q / k / v (QKV, kind 1) and
    cross-attention q (kind 2) projections: integer operands, so every head's rows equal the whole-grid projection bit for bit;
    with 11 heads the rows of head 11 stay NaN, and with 13 clusters the one without a head writes nothing"""
    p = PROJ["ws.qkv"] if kind == 1 else Proj("ws.q", 768, 768, "store", llama=False, bias=True)
    p = dataclasses.replace(p, input="copy")
    gen = torch.Generator(device="cuda").manual_seed(kind * 100 + heads)
    r = Run(E, p, "fp16", 3, gen, exact=True)
    r.run(E, grid)
    r.check()
    whole = r.snapshot()
    r.refill()
    r.d["head_plan"] = kind
    pl = r.run(E, grid, cluster=8, heads=heads)
    assert pl[0] == (3 if kind == 1 else 1) * 8, pl   # CTA 0 = rank 0 of cluster 0: the tiles of one head
    got = r.snapshot()
    for n in whole:
        want = whole[n].clone()
        if heads < 12:   # columns [704, 768) of q (and of the k / v cache rows) belong to head 11
            want[..., 704:768] = float("nan")
        assert same_bits(got[n], want), n


def test_head_out_projection_partials_sum_to_the_projection(E):
    """kind 3 (the head's 64 columns of the out-projection, K = 64 of the 768-long weight rows, k_off = 64 h): each cluster's
    partial against float64, and their sum against the float64 projection of the concatenated head outputs"""
    H, d, B, grid = 12, 768, 4, 96
    gen = torch.Generator(device="cuda").manual_seed(9)
    tiled, W = weights(E, d, d, "fp16", gen)
    o = torch.randn(H, B, 64, device="cuda", generator=gen).half()
    out = nan_like((H + 1, B, d), torch.float32)
    pl = E.decode_gemv([dict(w=tiled, N=d, K=64, mode="store", input="copy", x16=o, out=out, ldo=d, head_plan=3,
                             x_cluster_stride=B * 64, out_cluster_stride=B * d)], B, torch.float16, llama=False, grid=grid,
                       cluster=8, heads=H)
    assert pl[0][0] == d // 8, pl
    assert torch.isnan(out[H]).all()
    total, total_bound = torch.zeros(B, d, dtype=torch.float64, device="cuda"), torch.zeros(B, d, dtype=torch.float64, device="cuda")
    for h in range(H):
        Wh, oh = W[:, 64 * h: 64 * h + 64], o[h].double()
        ref = oh @ Wh.T
        bound = ACC * (oh.abs() @ Wh.abs().T) + OUT * ref.abs()
        _note("head out slice", "fp16", (out[h].double() - ref).abs(), bound)
        total += out[h].double()
        total_bound += bound
    full = torch.cat(list(o.double()), dim=1) @ W.T
    _note("head out slice", "fp16", (total - full).abs(), total_bound)
