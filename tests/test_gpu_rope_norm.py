"""GPU tests (H100) of the kernels between the GEMMs and the attention, by themselves, against a float64 evaluation
(tests/rope_norm_ref.py, transformers' form) on the same operands and the same fp32 (cos, sin) table the kernels read:

  * the prefill / encoder row norm (norm_rows_kernel, csrc/elementwise.cu, through s2s_norm_rows): LayerNorm with bias at
    Whisper's d = 384 / 768 / 1280, RMSNorm at d = 1024 / 2560 / 4096 / 5120, and d = 4 / 36 / 132 off the 128-column step;
  * the prefill RoPE and K/V append (rope_prefill_kernel; Qwen3: qknorm_rope_prefill_kernel<T, HD>, csrc/llama.cu, through
    s2s_prefill_rope, the launcher prefill_layers calls) at Llama-3-8B, Qwen3-4B / 14B / 32B, the Qwen3-TTS talker and code
    predictor and qwen3-micro heads, n in {1, 2, 129, 512} new rows behind past in {0, 1, 511, 4096 - n};
  * the Qwen3 decode's q/k preparation and own-key append (ld_qk_prepare inside ld_attn, csrc/llama_decode.cu, through
    s2s_decode_attention in Qwen3 mode) followed by the attention that reads the new key;
  * the greedy choice after a prefill (argmax_row_kernel, through s2s_argmax_row).

Bounds, with u = 2^-24 and, for a 16-bit result, its unit roundoff u_T (2^-11 fp16, 2^-8 bf16) and sub_T (2^-25 fp16
below the smallest normal, 0 bf16) added as u_T |ref| + sub_T:

Row norm.  The kernel is two-pass: mean, then sum (x - mean)^2, then the write pass.  Each lane sums d / 128 float4 groups
(two tree levels each) sequentially and the warp adds five tree levels, so with n = ceil(d / 128) + 7 terms:
    e_mean = n u mean|x|,   e_var = (n + 3) u var + 2 e_mean mean|x - mean| + e_mean^2,
    rstd relative error r = e_var / (2 (var + eps)) + 4 u   (the division by d, + eps, rsqrtf),
    |y - ref| <= |w| rstd (1 + r) (e_mean + (r + u) |x - mean|) + 3 u |ref| + u |b|.
var is the float64 variance about the mean (RMSNorm: mean(x^2), mean = 0).  Because the second pass subtracts the mean
first, the cancellation term is e_mean^2 and 2 e_mean mean|x - mean|, not the one-pass n u mean^2: rows with |mean| / std
up to 30 stay within the same bound as centred rows.  A constant row has var = 0 and comes out as bias + O(e_mean / sqrt(eps)).

Llama RoPE.  A pair (v0, v1) of 16-bit inputs is rotated with the table's fp32 (c, s): y0 = v0 c - v1 s, y1 = v1 c + v0 s,
two products and a sum, so |y - ref| <= 3 u (|v0 c| + |v1 s|) before the 16-bit rounding.

Qwen3 q/k norm + RoPE.  A lane sums PER = hd / 32 squares with fmaf, the warp five tree levels: the sum of squares is
within (PER + 5) u relative, rstd within (PER + 5) u / 2 + 4 u, a = v rstd g two more roundings, the rotation three:
    |y - ref| <= ((PER + 5) / 2 + 9) u (|a0 c| + |a1 s|),   a the float64 normalised values;
the decode's q also carries the 1 / sqrt(hd) scale (one more rounding, exact for hd = 64) and stays fp32: + u |ref|.

Decode attention after the own-key append: the float64 softmax over the kernel's own qn (checked above) and the cache as
the kernel left it (the appended row checked above), with the decode bound of test_gpu_attention.py part B:
2 ds A + 2^-20 A + u_T |ref|.

Exact and structural checks, bit for bit: a table of (+-1, 0) / (0, +-1) entries with Llama rows of small integers makes
rotated q and K exact, which checks routing (position past + t, table column j for pair j, the q / k / v column
boundaries); V is copied; the caches are NaN-filled beforehand and everything outside rows [past, past + n) comes back
unchanged; the k and v columns of qkv are left as they were; n rows prefilled at once equal the same rows as two chunks and
as one segment of a batch at a non-zero row offset; in the decode every cache row but len - 1 of each session is untouched,
and row len - 1 is NaN beforehand so an attention that read it before the append would fail.  Every case runs twice with
bit-identical results.  Argmax: single maxima at 0, n - 1 and on both sides of the 32-lane and 1024-thread strides, ties
across lanes, warps and the final merge (the lowest id wins), +inf, all -inf, NaN entries and an all-NaN row, against
"NaN counts as -inf, the lowest id among the maxima".

The worst error / bound per kernel and dtype is printed at the end of the module."""
import math

import numpy as np
import pytest
import torch

import rope_norm_ref as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SUB16 = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
SMALL = 2.0 ** -20
DTYPES = [torch.float16, torch.bfloat16]
MAX_POS = 4096
_WORST = {}
_TABLES = {}

# heads, kv_heads, hd, qk_norm, rope_theta
GEOMS = {
    "llama3-8b": (32, 8, 128, False, 500000.0),
    "llama-hd64": (8, 2, 64, False, 10000.0),
    "qwen3-4b": (32, 8, 128, True, 1e6),
    "qwen3-14b": (40, 8, 128, True, 1e6),
    "qwen3-32b": (64, 8, 128, True, 1e6),
    "tts-talker": (16, 2, 128, True, 1e6),
    "tts-cp": (16, 8, 128, True, 1e6),
    "qwen3-micro": (4, 2, 64, True, 1e6),
}
QWEN3 = [g for g in GEOMS if GEOMS[g][3]]


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, r in sorted(_WORST.items()):
        print(f"\nrope / norm {k[0]} {k[1]}: worst error / bound = {r:.3f}")


def _note(what, dt, err, bound):
    ratio = float((err / bound).max()) if err.numel() else 0.0
    key = (what, str(dt).replace("torch.", ""))
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    assert ratio <= 1.0, f"{what} {dt}: error / bound {ratio:.3f}"


def _table(hd, theta):
    if (hd, theta) not in _TABLES:
        _TABLES[(hd, theta)] = R.rope_table(MAX_POS, hd, theta).cuda()
    return _TABLES[(hd, theta)]


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


# ============================================================================================================ row norms
NORM_CASES = []
for _d in (384, 768, 1280, 4, 36, 132):
    NORM_CASES += [("layer", _d, 1e-5, rows) for rows in ((1, 9, 512, 4500) if _d >= 384 else (1, 7, 8, 9, 512))]
for _d in (1024, 2560, 4096, 5120, 4, 36, 132):
    for _eps in (1e-5, 1e-6):
        NORM_CASES += [("rms", _d, _eps, rows) for rows in ((1, 8, 512) if _d >= 1024 else (1, 7, 9, 512))]
NORM_CASES += [("rms", 1024, 1e-6, 4500)]


def _norm_rows_input(kind, rows, d, gen):
    """row r % 4: 0 centred N(0, 1); 1 |mean| / std = 30 (sign alternating); 2 LayerNorm: a constant row, RMSNorm: mean(x^2)
    near eps (x ~ 1e-3); 3 LayerNorm: offset 1000 with std 30, RMSNorm: mean(x^2) near 1e6"""
    x = torch.randn(rows, d, device="cuda", generator=gen, dtype=torch.float64)
    r = torch.arange(rows, device="cuda")
    sign = torch.where(r % 8 < 4, 1.0, -1.0).double()[:, None]
    x = torch.where((r % 4 == 1)[:, None], x + 30 * sign, x)
    if kind == "layer":
        x = torch.where((r % 4 == 2)[:, None], torch.full_like(x, 1.0) * (1.0 + r[:, None] % 7 / 8.0), x)
        x = torch.where((r % 4 == 3)[:, None], 30 * x + 1000 * sign, x)
    else:
        x = torch.where((r % 4 == 2)[:, None], x * 1e-3, x)
        x = torch.where((r % 4 == 3)[:, None], x * 1e3, x)
    return x.float()


def _norm_bound(kind, x, w, b, eps, ref):
    d = x.shape[1]
    n = math.ceil(d / 128) + 7
    if kind == "layer":
        mean = x.mean(-1, keepdim=True)
        xc = x - mean
        e_mean = n * U * x.abs().mean(-1, keepdim=True)
    else:
        xc, e_mean = x, torch.zeros_like(x[:, :1])
    var = (xc * xc).mean(-1, keepdim=True)
    e_var = (n + 3) * U * var + 2 * e_mean * xc.abs().mean(-1, keepdim=True) + e_mean ** 2
    r = e_var / (2 * (var + eps)) + 4 * U
    rstd = torch.rsqrt(var + eps)
    bound = w.abs() * rstd * (1 + r) * (e_mean + (r + U) * xc.abs()) + 3 * U * ref.abs()
    return bound + U * b.abs() if b is not None else bound


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", NORM_CASES, ids=[f"{k}-d{d}-eps{e:g}-r{r}" for k, d, e, r in NORM_CASES])
def test_norm_rows_against_float64(E, case, dt):
    kind, d, eps, rows = case
    gen = torch.Generator(device="cuda").manual_seed(d * 7 + rows)
    x = _norm_rows_input(kind, rows, d, gen)
    w = (1 + 0.25 * torch.randn(d, device="cuda", generator=gen)).float()
    b = (0.5 * torch.randn(d, device="cuda", generator=gen)).float() if kind == "layer" else None
    xd, wd = x.double(), w.double()
    bd = b.double() if b is not None else None
    ref = R.layer_norm(xd, wd, bd, eps) if kind == "layer" else R.rms_norm(xd, wd, eps)
    bound = _norm_bound(kind, xd, wd, bd, eps, ref)
    outs = {}
    for which in ("h", "f", "hf"):
        oh = torch.full((rows + 1, d), float("nan"), dtype=dt, device="cuda") if "h" in which else None
        of = torch.full((rows + 1, d), float("nan"), dtype=torch.float32, device="cuda") if "f" in which else None
        for rep in range(2):
            if oh is not None:
                oh.fill_(float("nan"))
            if of is not None:
                of.fill_(float("nan"))
            E.norm_rows(x, w, b, eps, out_h=oh[:rows] if oh is not None else None, out_f=of[:rows] if of is not None else None,
                        dtype=dt)
            torch.cuda.synchronize()
            got = (oh.clone() if oh is not None else None, of.clone() if of is not None else None)
            if rep == 0:
                first = got
            else:
                for a, c in zip(first, got):
                    assert a is None or _same_bits(a, c), "two runs differ"
        oh, of = first
        if of is not None:
            assert torch.isnan(of[rows]).all()
            _note(f"norm_rows {kind} fp32", dt, (of[:rows].double() - ref).abs(), bound)
            outs["f"] = of[:rows]
        if oh is not None:
            assert torch.isnan(oh[rows]).all()
            _note(f"norm_rows {kind}", dt, (oh[:rows].double() - ref).abs(), bound * (1 + U16[dt]) + U16[dt] * ref.abs() + SUB16[dt])
            outs["h"] = oh[:rows]
        if which == "hf":   # both outputs of one launch are the fp32 value and its rounding
            assert torch.equal(outs["f"].to(dt).view(torch.int16), oh[:rows].view(torch.int16))
    if kind == "layer":     # constant rows: bias, up to e_mean / sqrt(eps)
        const = torch.arange(rows, device="cuda") % 4 == 2
        if const.any():
            assert torch.allclose(outs["f"][const].double(), bd.expand(int(const.sum()), d), rtol=0, atol=1e-3)


def test_norm_rows_rejects_bad_arguments(E):
    from speech_to_speech_b200._lib import S2SError
    x = torch.randn(8, 72, device="cuda")
    w = torch.ones(72, device="cuda")
    oh = torch.zeros(8, 72, dtype=torch.float16, device="cuda")
    of = torch.zeros(8, 72, device="cuda")
    buf = torch.zeros(1024, device="cuda")
    bad = [
        dict(x=x[:, :70].contiguous(), w=w[:70], out_h=oh[:, :70].contiguous()),          # d % 4
        dict(x=x, w=w),                                                                  # no output
        dict(x=buf[1:577].view(8, 72), w=w, out_f=of),                                   # x not 16-byte aligned
        dict(x=x, w=buf[2:74], out_f=of),                                                # w
        dict(x=x, w=w, bias=buf[3:75], out_f=of),                                        # bias
        dict(x=x, w=w, out_f=buf[1:577].view(8, 72)),                                    # out_f
        dict(x=x, w=w, out_h=torch.zeros(8 * 72 + 2, dtype=torch.float16, device="cuda")[2:].view(8, 72)),   # out_h 4 B off
    ]
    for kw in bad:
        with pytest.raises(S2SError):
            E.norm_rows(kw.pop("x"), kw.pop("w"), out_h=kw.pop("out_h", None), out_f=kw.pop("out_f", None), **kw)
    with pytest.raises(KeyError):
        E.norm_rows(x, w, out_f=of, dtype=torch.float32)
    from speech_to_speech_b200 import _lib
    lib = _lib.load()
    ctx = E.get_context(0)
    for dtc in (0, 3):
        assert lib.s2s_norm_rows(ctx, x.data_ptr(), w.data_ptr(), None, 1e-5, 8, 72, oh.data_ptr(), None, dtc, None) != 0
    torch.cuda.synchronize()


# ================================================================================================== prefill RoPE / Qwen3
PREFILL_NP = [(1, 0), (1, 511), (1, 4095), (2, 1), (2, 4094), (129, 0), (129, 1), (129, 3967), (512, 0), (512, 511), (512, 3584)]
PREFILL_CASES = [(g, dt, n, past) for g in GEOMS for dt in DTYPES for n, past in PREFILL_NP]


def _prefill_id(c):
    g, dt, n, past = c
    return f"{g}-{str(dt)[6:]}-n{n}-past{past}"


class Prefill:
    """Operands of one s2s_prefill_rope call: natural-layout q / k / v values (16-bit), the pair-adjacent qkv the kernel
    reads, NaN-filled caches [MAX_POS, kv_heads * hd] and the Qwen3 norm weights."""

    def __init__(self, geom, dt, n, past, seed, qkv_nat=None):
        self.H, self.KV, self.hd, self.qk, theta = GEOMS[geom]
        self.dt, self.n, self.past = dt, n, past
        H, KV, hd = self.H, self.KV, self.hd
        self.qd, self.kvd = H * hd, KV * hd
        self.tab = _table(hd, theta)
        gen = torch.Generator(device="cuda").manual_seed(seed)
        if qkv_nat is None:
            qkv_nat = torch.randn(n, self.qd + 2 * self.kvd, device="cuda", generator=gen)
            if self.qk:   # raw q / k of every third token near eps in mean square, and of some heads large
                t = torch.arange(n, device="cuda")
                qkv_nat = torch.where((t % 3 == 1)[:, None], qkv_nat * 1e-3, qkv_nat)
                qkv_nat[:, hd: 2 * hd] *= 40
        self.nat = qkv_nat.to(dt)                                     # the 16-bit values, natural head layout
        self.qkv = self.nat.clone()
        self.qkv[:, : self.qd + self.kvd] = R.to_pairs(self.nat[:, : self.qd + self.kvd], hd)
        self.qn = self.kn = None
        if self.qk:
            self.qn_nat = (1 + 0.3 * torch.randn(hd, device="cuda", generator=gen)).float()
            self.kn_nat = (1 + 0.3 * torch.randn(hd, device="cuda", generator=gen)).float()
            self.qn, self.kn = R.to_pairs(self.qn_nat, hd).contiguous(), R.to_pairs(self.kn_nat, hd).contiguous()
        self.eps = 1e-6
        self.kc = torch.full((MAX_POS, self.kvd), float("nan"), dtype=dt, device="cuda")
        self.vc = torch.full_like(self.kc, float("nan"))
        self.qkv0 = self.qkv.clone()

    def run(self, E, qkv=None, past=None, tab=None):
        E.prefill_rope(self.qkv if qkv is None else qkv, self.H, self.KV, self.past if past is None else past,
                       self.tab if tab is None else tab, self.kc, self.vc, q_norm=self.qn, k_norm=self.kn, eps=self.eps)

    def reference(self, tab=None):
        """-> (q, k) float64 in the pair layout, and the bound before the 16-bit rounding"""
        n, H, KV, hd = self.n, self.H, self.KV, self.hd
        pos = torch.arange(self.past, self.past + n, device="cuda")
        c, s = R.cos_sin(self.tab if tab is None else tab, pos)
        x = self.nat.double()
        q, k = x[:, : self.qd].view(n, H, hd), x[:, self.qd: self.qd + self.kvd].view(n, KV, hd)
        if self.qk:
            q, k = R.rms_norm(q, self.qn_nat.double(), self.eps), R.rms_norm(k, self.kn_nat.double(), self.eps)
            coef = ((hd // 32 + 5) / 2 + 9) * U
        else:
            coef = 3 * U
        out = []
        for a in (q, k):
            ref = R.rope(a, c, s)
            bound = coef * R.rope_abs(a, c, s)
            out += [R.to_pairs(ref.reshape(n, -1), hd), R.to_pairs(bound.reshape(n, -1), hd)]
        return out

    def check_structure(self):
        n, past = self.n, self.past
        # the k and v columns of qkv are left as they were; V is a bit copy
        assert _same_bits(self.qkv[:, self.qd:], self.qkv0[:, self.qd:]), "k / v columns of qkv changed"
        assert _same_bits(self.vc[past: past + n], self.qkv0[:, self.qd + self.kvd:]), "V cache rows are not the v columns"
        # nothing outside rows [past, past + n) of the caches
        for c in (self.kc, self.vc):
            outside = torch.cat([c[:past], c[past + n:]])
            assert torch.isnan(outside).all() and _same_bits(outside, torch.full_like(outside, float("nan"))), "cache row outside"

    def check_bound(self):
        q, qb, k, kb = self.reference()
        u, sub = U16[self.dt], SUB16[self.dt]
        kind = "qwen3 q/k norm + rope" if self.qk else "llama rope"
        _note(kind + " q", self.dt, (self.qkv[:, : self.qd].double() - q).abs(), qb * (1 + u) + u * q.abs() + sub)
        kgot = self.kc[self.past: self.past + self.n].double()
        _note(kind + " k", self.dt, (kgot - k).abs(), kb * (1 + u) + u * k.abs() + sub)


@pytest.mark.parametrize("case", PREFILL_CASES, ids=[_prefill_id(c) for c in PREFILL_CASES])
def test_prefill_rope_against_float64(E, case):
    geom, dt, n, past = case
    P = Prefill(geom, dt, n, past, seed=n * 31 + past)
    P.run(E)
    torch.cuda.synchronize()
    P.check_structure()
    P.check_bound()
    q1, k1, v1 = P.qkv.clone(), P.kc.clone(), P.vc.clone()
    P.qkv.copy_(P.qkv0)
    P.kc.fill_(float("nan"))
    P.vc.fill_(float("nan"))
    P.run(E)
    torch.cuda.synchronize()
    assert _same_bits(P.qkv, q1) and _same_bits(P.kc, k1) and _same_bits(P.vc, v1), "two runs differ"


def _unit_table(hd, gen):
    """(cos, sin) in {(1, 0), (0, 1), (-1, 0), (0, -1)}, random per (position, column)"""
    r = torch.randint(0, 4, (MAX_POS, hd // 2), device="cuda", generator=gen)
    c = torch.tensor([1.0, 0.0, -1.0, 0.0], device="cuda")[r]
    s = torch.tensor([0.0, 1.0, 0.0, -1.0], device="cuda")[r]
    return torch.stack([c, s], -1).contiguous()


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("geom,n,past", [("llama3-8b", 129, 3967), ("llama3-8b", 2, 1), ("llama-hd64", 512, 511), ("llama-hd64", 1, 4095)])
def test_prefill_rope_exact_routing(E, geom, n, past, dt):
    """small-integer rows and a table of (+-1, 0) / (0, +-1): every rotated value is exact, so q, K and V must equal the
    reference bit for bit -- a wrong position, table column or q / k / v boundary changes some value"""
    H, KV, hd = GEOMS[geom][:3]
    gen = torch.Generator(device="cuda").manual_seed(n + past)
    nat = torch.randint(-64, 65, (n, (H + 2 * KV) * hd), device="cuda", generator=gen).float()
    P = Prefill(geom, dt, n, past, 0, qkv_nat=nat)
    tab = _unit_table(hd, gen)
    P.run(E, tab=tab)
    torch.cuda.synchronize()
    q, _, k, _ = P.reference(tab)
    assert torch.equal(P.qkv[:, : P.qd].double(), q), "rotated q"
    assert torch.equal(P.kc[past: past + n].double(), k), "rotated K"
    P.check_structure()


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("geom", ["llama3-8b", "qwen3-32b", "tts-talker", "qwen3-micro"])
def test_prefill_chunks_and_batch_segments_agree(E, geom, dt):
    """n rows at `past` in one launch == the same rows as two chunks (the second at past + n1) == the rows as one segment
    of a batch, at a non-zero row offset of a larger qkv buffer, bit for bit"""
    n, past, n1, off = 300, 700, 129, 37
    A = Prefill(geom, dt, n, past, seed=5)
    A.run(E)
    B = Prefill(geom, dt, n, past, seed=5)
    B.run(E, qkv=B.qkv[:n1], past=past)
    B.run(E, qkv=B.qkv[n1:], past=past + n1)
    C = Prefill(geom, dt, n, past, seed=5)
    big = torch.full((off + n + 11, C.qkv.shape[1]), float("nan"), dtype=dt, device="cuda")
    big[off: off + n] = C.qkv
    big0 = big.clone()
    C.run(E, qkv=big[off: off + n])
    torch.cuda.synchronize()
    assert _same_bits(B.qkv, A.qkv) and _same_bits(B.kc, A.kc) and _same_bits(B.vc, A.vc)
    assert _same_bits(big[off: off + n], A.qkv) and _same_bits(C.kc, A.kc) and _same_bits(C.vc, A.vc)
    assert _same_bits(big[:off], big0[:off]) and _same_bits(big[off + n:], big0[off + n:]), "rows outside the segment"


def test_prefill_rope_rejects_bad_arguments(E):
    from speech_to_speech_b200 import _lib
    P = Prefill("qwen3-micro", torch.bfloat16, 4, 0, seed=1)
    lib, ctx = _lib.load(), E.get_context(0)
    flat = torch.zeros(MAX_POS * 128 + 8, dtype=torch.bfloat16, device="cuda")
    ok = dict(qkv=P.qkv.data_ptr(), n=4, heads=4, kv_heads=2, hd=64, past=0, rope=P.tab.data_ptr(), max_pos=MAX_POS,
              q_norm=P.qn.data_ptr(), k_norm=P.kn.data_ptr(), kc=P.kc.data_ptr(), vc=P.vc.data_ptr(), dtype=_lib.S2S_BF16)
    call = lambda a: lib.s2s_prefill_rope(ctx, a["qkv"], a["n"], a["heads"], a["kv_heads"], a["hd"], a["past"], a["rope"],
                                          a["max_pos"], a["q_norm"], a["k_norm"], 1e-6, a["kc"], a["vc"], a["dtype"], None)
    bad = [dict(ok, hd=96), dict(ok, hd=32), dict(ok, heads=3), dict(ok, past=MAX_POS - 3), dict(ok, past=-1), dict(ok, n=0),
           dict(ok, k_norm=None), dict(ok, q_norm=None), dict(ok, dtype=_lib.S2S_F32),
           dict(ok, qkv=P.qkv.data_ptr() + 2), dict(ok, kc=flat.data_ptr() + 2), dict(ok, rope=P.tab.data_ptr() + 8),
           dict(ok, q_norm=P.qn.data_ptr() + 4), dict(ok, kc=None)]
    for a in bad:
        assert call(a) != 0, a
    torch.cuda.synchronize()
    assert _same_bits(P.qkv, P.qkv0) and torch.isnan(P.kc).all() and torch.isnan(P.vc).all(), "a rejected call wrote"
    assert call(ok) == 0
    torch.cuda.synchronize()
    assert not torch.isnan(P.kc[:4]).any()


# ============================================================================================ Qwen3 decode own-key path
DEC_WARPS = 8


def attn_plan(BH, n_blocks, s_max, grid):
    """decode_common.cuh attn_plan, restated: splits | 0x80 for warp-level items."""
    best, best_cost = 1, 0x7FFFFFFF
    lim = min(n_blocks, s_max)
    for S in range(1, min(lim, 16) + 1):
        bps = -(-n_blocks // S)
        cost = -(-BH * S // grid) * ((bps + DEC_WARPS - 1) // DEC_WARPS + 2)
        if cost < best_cost:
            best, best_cost = S, cost
    for S in range(1, min(lim, 32) + 1):
        bpi = -(-n_blocks // S)
        cost = -(-BH * S // (grid * DEC_WARPS)) * (bpi + 2)
        if cost < best_cost:
            best, best_cost = S | 0x80, cost
    return best


LENS16 = [4096, 1, 31, 32, 33, 256, 257, 513, 2047, 3841, 4095, 1025, 64, 65, 2, 3000]
DEC_LENS = [(132, [1]), (132, [33]), (37, [32, 4096, 1]), (66, [4096, 33, 1025]), (132, LENS16), (37, LENS16)]
DEC_CASES = [(g, dt, grid, lens) for g in QWEN3 for dt in DTYPES for grid, lens in DEC_LENS]


def _dec_id(c):
    g, dt, grid, lens = c
    return f"{g}-{str(dt)[6:]}-g{grid}-b{len(lens)}-" + "-".join(map(str, lens[:3]))


def _assoc_b(lens):
    return 8 if len(lens) == 16 else 0


class OwnKey:
    def __init__(self, geom, dt, grid, lens, seed):
        self.H, self.KV, self.hd, _, theta = GEOMS[geom]
        self.dt, self.grid, self.lens, self.B = dt, grid, list(lens), len(lens)
        H, KV, hd, B = self.H, self.KV, self.hd, self.B
        self.tab = _table(hd, theta)
        self.slots = [B - 1 - b for b in range(B)]
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.kv = torch.full((B + 1, 2, MAX_POS, KV * hd), float("nan"), dtype=dt, device="cuda")
        for b, L in enumerate(self.lens):   # keys [0, len - 1) and values [0, len) cached; K row len - 1 stays NaN
            self.kv[self.slots[b], 0, : L - 1] = torch.randn(L - 1, KV * hd, device="cuda", generator=gen).to(dt)
            self.kv[self.slots[b], 1, :L] = torch.randn(L, KV * hd, device="cuda", generator=gen).to(dt)
        self.q = torch.randn(B, H, hd, device="cuda", generator=gen)
        self.kraw = torch.randn(B, KV, hd, device="cuda", generator=gen)
        self.q[1::3] *= 1e-3                                  # mean square near eps
        self.kraw[1::3] *= 1e-3
        self.q[2::3] *= 30
        self.qn_nat = (1 + 0.3 * torch.randn(hd, device="cuda", generator=gen)).float()
        self.kn_nat = (1 + 0.3 * torch.randn(hd, device="cuda", generator=gen)).float()
        self.eps = 1e-6
        self.kv0 = self.kv.clone()

    def run(self, E):
        qn = torch.full((self.B, self.H, self.hd), float("nan"), device="cuda")
        out, plan = E.decode_attention(self.q, self.kv, self.slots, self.lens, self.H, self.KV, grid=self.grid,
                                       assoc_b=_assoc_b(self.lens), kraw=self.kraw, q_norm=R.to_pairs(self.qn_nat, self.hd).contiguous(),
                                       k_norm=R.to_pairs(self.kn_nat, self.hd).contiguous(), rope=self.tab, eps=self.eps, qn_out=qn)
        return out, qn, plan

    def check(self, out, qn):
        H, KV, hd, dt = self.H, self.KV, self.hd, self.dt
        coef = ((hd // 32 + 5) / 2 + 9) * U
        g = H // KV
        for b, L in enumerate(self.lens):
            pos = torch.tensor([L - 1], device="cuda")
            c, s = R.cos_sin(self.tab, pos)
            qa = R.rms_norm(R.from_pairs(self.q[b].double().reshape(1, -1), hd).view(1, H, hd), self.qn_nat.double(), self.eps)
            ka = R.rms_norm(R.from_pairs(self.kraw[b].double().reshape(1, -1), hd).view(1, KV, hd), self.kn_nat.double(), self.eps)
            sc = hd ** -0.5
            qref = R.to_pairs((R.rope(qa, c, s) * sc).reshape(1, -1), hd)
            qb = R.to_pairs((coef * R.rope_abs(qa, c, s) * sc).reshape(1, -1), hd) + U * qref.abs()
            _note("decode qn (fp32)", dt, (qn[b].reshape(1, -1).double() - qref).abs(), qb)
            kref = R.to_pairs(R.rope(ka, c, s).reshape(1, -1), hd)
            kb = R.to_pairs((coef * R.rope_abs(ka, c, s)).reshape(1, -1), hd)
            krow = self.kv[self.slots[b], 0, L - 1].double()[None]
            _note("decode own key", dt, (krow - kref).abs(), kb * (1 + U16[dt]) + U16[dt] * kref.abs() + SUB16[dt])
            # attention over the cache as the kernel left it, with the kernel's qn
            kk = self.kv[self.slots[b], 0, :L].double().view(L, KV, hd).repeat_interleave(g, 1)
            vv = self.kv[self.slots[b], 1, :L].double().view(L, KV, hd).repeat_interleave(g, 1)
            qq = qn[b].double()
            sco = torch.einsum("hc,jhc->hj", qq, kk)
            sab = torch.einsum("hc,jhc->hj", qq.abs(), kk.abs())
            w = torch.softmax(sco, -1)
            ref = torch.einsum("hj,jhc->hc", w, vv)
            A = torch.einsum("hj,jhc->hc", w, vv.abs())
            ds = hd * U * sab.amax(-1, keepdim=True)
            _note("decode attention after the append", dt, (out[b].double() - ref).abs(), (2 * ds + SMALL) * A + U16[dt] * ref.abs())
        # every cache row but K row len - 1 of each session is untouched
        mask = torch.ones(self.kv.shape[:3], dtype=torch.bool, device="cuda")
        for b, L in enumerate(self.lens):
            mask[self.slots[b], 0, L - 1] = False
        assert _same_bits(self.kv[mask], self.kv0[mask]), "a cache row other than the own key changed"


@pytest.mark.parametrize("case", DEC_CASES, ids=[_dec_id(c) for c in DEC_CASES])
def test_decode_own_key_against_float64(E, case):
    geom, dt, grid, lens = case
    D = OwnKey(geom, dt, grid, lens, seed=sum(lens) + grid)
    out, qn, plan = D.run(E)
    assert plan == attn_plan((_assoc_b(lens) or len(lens)) * D.H, -(-max(lens) // 32), MAX_POS // 64, grid)
    assert torch.isfinite(out.float()).all(), "the attention read K row len - 1 before the append"
    D.check(out, qn)
    kv1 = D.kv.clone()
    D.kv.copy_(D.kv0)                                          # K rows len - 1 back to NaN
    out2, qn2, _ = D.run(E)
    assert _same_bits(out, out2) and torch.equal(qn.view(torch.int32), qn2.view(torch.int32)) and _same_bits(D.kv, kv1), "two runs differ"


def test_decode_own_key_plan_coverage():
    """the cases reach CTA-level and warp-level items, with one and with several key splits"""
    plans = {attn_plan((_assoc_b(ls) or len(ls)) * GEOMS[g][0], -(-max(ls) // 32), MAX_POS // 64, grid)
             for g in QWEN3 for grid, ls in DEC_LENS}
    cta = {p for p in plans if not p & 0x80}
    warp = {p & 0x7F for p in plans if p & 0x80}
    assert 1 in cta and any(s > 1 for s in cta), plans
    assert any(s > 1 for s in warp), plans


def test_decode_qk_norm_rejects_bad_arguments(E):
    from speech_to_speech_b200._lib import S2SError
    D = OwnKey("qwen3-micro", torch.bfloat16, 37, [5, 9], seed=3)
    nw = torch.ones(64, device="cuda")
    with pytest.raises(S2SError):   # rope missing
        E.decode_attention(D.q, D.kv, D.slots, D.lens, 4, 2, kraw=D.kraw, q_norm=nw, k_norm=nw)
    with pytest.raises(S2SError):   # k_norm missing
        E.decode_attention(D.q, D.kv, D.slots, D.lens, 4, 2, kraw=D.kraw, q_norm=nw, rope=D.tab)
    buf = torch.zeros(4 * 64 + 4, device="cuda")
    with pytest.raises(S2SError):   # kraw not 16-byte aligned
        E.decode_attention(D.q, D.kv, D.slots, D.lens, 4, 2, kraw=buf[1:1 + 2 * 2 * 64].view(2, 2, 64), q_norm=nw, k_norm=nw, rope=D.tab)
    torch.cuda.synchronize()
    assert _same_bits(D.kv, D.kv0), "a rejected call wrote"


# ================================================================================================================ argmax
def _argmax_ref(row):
    """NaN counts as -inf; the lowest id among the maxima"""
    r = np.where(np.isnan(row), -np.inf, row)
    return int(np.argmax(r))


def _argmax_rows(n, gen):
    base = lambda: torch.randint(-1000, 1000, (n,), generator=gen).float() / 8
    rows, names = [], []

    def add(name, row):
        rows.append(row)
        names.append(name)

    for i in sorted({0, 1, 31, 32, 33, 1023, 1024, 1025, 2047, n - 1025, n - 33, n - 1} & set(range(n))):
        r = base()
        r[i] = 200
        add(f"max@{i}", r)
    for ids in ([1029, 5], [7, 40], [33, 1], [n - 1, 999], [2047, 64, 3000 % n], [n - 1, n - 2], [1024, 0], [n - 1, 31]):
        r = base()
        r[torch.tensor(ids)] = 200
        add(f"tie{ids}", r)
    r = base()
    r[torch.tensor([n - 5, 600])] = float("inf")
    add("+inf tie", r)
    add("all -inf", torch.full((n,), float("-inf")))
    r = base()
    r[torch.tensor([0, 1, 1024, n - 1])] = float("nan")
    r[777] = 300
    add("nan entries", r)
    r = torch.full((n,), float("nan"))
    r[n // 2] = -5.0
    add("nan but one", r)
    add("all nan", torch.full((n,), float("nan")))
    r = torch.full((n,), float("nan"))
    r[torch.arange(3, n, 2)] = float("-inf")
    add("nan and -inf", r)
    return rows, names


@pytest.mark.parametrize("n", [2048, 128256, 151936])
def test_argmax_row(E, n):
    gen = torch.Generator().manual_seed(n)
    rows, names = _argmax_rows(n, gen)
    out = torch.full((len(rows) + 1,), -7, dtype=torch.int32, device="cuda")
    dev_rows = torch.stack(rows).cuda()
    for i in range(len(rows)):
        E.argmax_row(dev_rows[i], out=out[i: i + 1])
    got = out.tolist()
    out2 = torch.full_like(out, -7)
    for i in range(len(rows)):
        E.argmax_row(dev_rows[i], out=out2[i: i + 1])
    assert out2.tolist() == got, "two runs differ"
    assert got[-1] == -7
    for i, name in enumerate(names):
        assert 0 <= got[i] < n, (name, got[i])
        assert got[i] == _argmax_ref(rows[i].numpy()), (name, got[i], _argmax_ref(rows[i].numpy()))
