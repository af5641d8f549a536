"""GPU tests (H100) of the prefill / encoder GEMM by itself (csrc/gemm_tc.cu through s2s_gemm_ex), against a float64
evaluation of the same operation

    v[b][m][n] = sum_k A[b][m][k] W[n][k] (+ bias[n]),   then the epilogue (GELU, SwiGLU, residual, positional table, stores),

in every form the engines call it: Whisper conv1 / conv2 (overlapping windows, a grid over the batch, padded output rows,
the positional table), the encoder's qkv / o / fc1 / fc2 and the head-major cross-attention K/V projection (small and
large-v3), the Llama-3-8B / Qwen3-14B / Qwen3-32B prefill projections and lm_head over tiled bf16, tiled fp16 and FP8
weights -- each in both N-tile instantiations (BN 64 and 128) -- and off the production shapes (M around the 128-row tile,
K tails, ring wrap-around, N = 64, strided A and W).

Bound per output, the model of tests/test_gpu_decode_gemv.py.  Products of 16-bit operands are exact in fp32.  Let
S = |A| |W|^T (+ |bias|) over the operands the kernel multiplies (the 16-bit A and W; W recovered by untiling the bytes;
FP8: dq(Q) = Q * 2^e_n, which bf16 holds exactly).  Then
    accumulation:                              |v - ref| <= acc = 2^-16 S
    fp32 outputs (with residual / table r):    acc + 8 * 2^-24 (|ref| + |r|)
    16-bit outputs:                            (1 + u_T) (the propagated error) + u_T |value| + sub_T,
u_T = 2^-11 for fp16 and 2^-8 for bf16, sub_T = 2^-25 for fp16, 0 for bf16 (rounding the fp32 value y to T moves it by at
most u_T |y| + sub_T, and |y| <= |value| + the propagated error).  The propagated error is acc times the
epilogue's slope: exact-erf GELU <= 1.13 acc + 2^-22 |v| (erff near its cancellation); SwiGLU silu(g) * u moves by
<= 1.1 acc_g |u| + |silu(g)| acc_u, and __expf's error (at most 2 + 1.173 |g| ulps) moves silu(g) by that relative amount.
2^-16 = 256 u covers the fp32 accumulation of K / 16 wgmma steps in the measured cases up to K = 25600 (the worst
ratio per case is printed at the end of the module); it is not widened to fit.

Exact designed inputs: integer weights and sparse {-1, 0, 1} activations keep every partial sum a small integer, so the
fp32 and 16-bit stores are exact and compared bit for bit -- the conv window and batch of every row, out_row_offset /
out_batch_rows, the positional-table row, the head-major address, and the (gate, up) pairing of SwiGLU (act 0 on the
interleaved columns, and act 2 with gates in {0, 20, 24, 28}, where silu(g) is g or 0 in fp32).

Every output buffer covers whole 128-row tiles with ldo > N and is filled with NaN (or with the residual) first; everything
outside the epilogue's destination must come back bit for bit (rows 0 and 3001 of every batch of conv1's output included).
A holds NaN in the rows after its last row and in the columns between K and a larger row stride; W in the columns
between K and a larger ldw.  Invariances, bit for bit: BN 64 = BN 128; bn = 0 equals the instantiation the rule names (and
is a second run of it); tiled 16-bit = row-major and FP8 = bf16 row-major over dq(Q), for every epilogue; in-place
residual = out-of-place; a batch's rows do not depend on the batch size."""
import dataclasses
import math
import zlib

import pytest
import torch

import gemm_ref as G

pytestmark = pytest.mark.gpu

U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SUB16 = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
ACC, OUT, U32 = 2.0 ** -16, 8 * 2.0 ** -24, 2.0 ** -24
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
ROWS, COLS = 2048, 4096          # reference block: a few hundred MB of float64 at K = 25600
_WORST = {}


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, r in sorted(_WORST.items()):
        print(f"\ngemm {k[0]} {k[1]} {k[2]} BN {k[3]}: worst error / bound = {r:.3f}")


def _note(key, err, bound):
    ratio = float((err / bound).max()) if err.numel() else 0.0
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    assert ratio <= 1.0, f"{key}: error / bound {ratio:.3f}"


def nan_(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def same_bits(a, b):
    if a.element_size() == 4:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- one call ------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Spec:
    site: str
    dt: str                  # "fp16" | "bf16" (FP8 weights: bf16)
    M: int
    N: int
    K: int
    layout: str = "row_major"   # "row_major" | "tiled" | "float8_e4m3"
    batch: int = 1
    a_row_stride: int = 0       # 0 = K
    frame: int = 0              # > 0: A is [batch][a_rows][frame] with zero rows 0 and a_rows - 1 (Whisper's padded convs)
    a_rows: int = 0
    ldw: int = 0                # row-major W: 0 = K
    bias: bool = False
    act: int = 0
    out: str = "h"              # "h" 16-bit, "f" fp32, "resid" fp32 in place, "pos" fp32 + table (resid_mode 2), "hm" head-major
    out_batch_rows: int = 0
    out_row_offset: int = 0
    hmr: int = 0

    @property
    def fmt(self):
        return "fp8" if self.layout == "float8_e4m3" else self.dt

    def rule_bn(self):
        tiles128 = (self.N // 128) * -(-self.M // 128) * self.batch
        return 128 if self.N % 128 == 0 and tiles128 >= num_sms() else 64


class Prob:
    """Operands, initial output buffers and the float64 reference of one Spec."""

    def __init__(self, E, s: Spec, exact=False, gen=None):
        self.s, self.dt, self.exact = s, DT[s.dt], exact
        gen = gen or torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(s).encode()) + exact)
        self.gen = gen
        M, N, K, B, dt = s.M, s.N, s.K, s.batch, self.dt
        self.rs = s.a_row_stride or K
        self.bs = s.a_rows * s.frame if s.frame else M * self.rs
        # A: the batches, then 128 rows of NaN
        A = nan_((B * self.bs + 128 * self.rs,), dt)
        body = A[: B * self.bs]
        if s.frame:
            vals = self._act((B, s.a_rows, s.frame))
            vals[:, 0] = 0
            vals[:, -1] = 0
            body.copy_(vals.reshape(-1).to(dt))
        else:
            body.view(B * M, self.rs)[:, :K] = self._act((B * M, K)).to(dt)
        self.A = A
        # W, and W_eff [N, K]: the 16-bit values the kernel multiplies; drawn in row chunks (lm_head: 778 M weights)
        w = torch.empty(N, K, dtype=dt, device="cuda")
        for r0 in range(0, N, 8192):
            r1 = min(N, r0 + 8192)
            if exact:
                w[r0:r1] = torch.randint(-3, 4, (r1 - r0, K), device="cuda", generator=gen).to(dt)
            else:
                c = torch.randn(r1 - r0, K, device="cuda", generator=gen) / math.sqrt(K)
                if s.layout != "row_major":   # rows of different magnitudes: different FP8 row scales within a tile
                    c *= torch.exp(torch.empty(r1 - r0, 1, device="cuda").uniform_(-1.5, 1.5, generator=gen))
                w[r0:r1] = c.to(dt)
        self._set_weights(E, w)
        self.bias = None
        if s.bias:
            self.bias = (torch.randint(-4, 5, (N,), device="cuda", generator=gen).float() if exact
                         else (torch.randn(N, device="cuda", generator=gen) * 0.5).float())
        self._outputs()

    def _act(self, shape):
        if self.exact:
            x = torch.randint(-1, 2, shape, device="cuda", generator=self.gen).double()
            return x * (torch.rand(shape, device="cuda", generator=self.gen) < min(1.0, 8.0 / self.s.K))
        return torch.randn(shape, device="cuda", generator=self.gen, dtype=torch.float64)

    def _set_weights(self, E, w):
        s, N, K, dt = self.s, self.s.N, self.s.K, self.dt
        if s.layout == "row_major":
            self.ldw = s.ldw or K
            W = nan_((N, self.ldw), dt)
            W[:, :K] = w.to(dt)
            self.W, self.W_eff = W, W[:, :K].contiguous()
            return
        self.ldw = 0
        self.W = E.tile_weights(w.to(dt).contiguous(), s.layout if s.layout == "float8_e4m3" else None)
        del w
        self.W_eff = torch.empty(N, K, dtype=dt, device="cuda")
        esz = 1 if s.fmt == "fp8" else 2
        for r0 in range(0, N, 8192):   # untile the bytes in whole 8-row tiles
            r1 = min(N, r0 + 8192)
            part = self.W[r0 * K * esz: r1 * K * esz]
            if s.fmt == "fp8":
                part = torch.cat([part, self.W[N * K + 4 * r0: N * K + 4 * r1]])
            self.W_eff[r0:r1] = G.untile(part, r1 - r0, K, s.fmt)
        assert torch.isfinite(self.W_eff).all()

    def out_rows(self):
        s = self.s
        return (s.batch - 1) * s.out_batch_rows + s.out_row_offset + -(-s.M // 128) * 128 + 1

    def _outputs(self):
        s, O, N = self.s, self.out_rows(), self.s.N
        self.init, self.table = {}, None
        cols = N // 2 if s.act == 2 else N
        if s.out == "h":
            self.init["out_h"] = nan_((O, cols + 8), self.dt)
        elif s.out == "hm":
            assert s.batch == 1 and s.M % s.hmr == 0
            self.init["out_h"] = nan_((((O - 1) // s.hmr + 1) * s.hmr * N + 64,), self.dt)
        elif s.out in ("f", "pos"):
            self.init["out_f"] = nan_((O, N + 8), torch.float32)
        else:   # resid
            r = (torch.randint(-50, 50, (O, N + 8), device="cuda", generator=self.gen).float() if self.exact
                 else torch.randn(O, N + 8, device="cuda", generator=self.gen))
            self.init["out_f"] = r
        if s.out == "pos":   # the table has as many rows as the output (rows >= M NaN): a wrong row index reads NaN
            self.table = nan_((O, N), torch.float32)
            self.table[: s.M] = (torch.randint(-9, 10, (s.M, N), device="cuda", generator=self.gen).float() if self.exact
                                 else torch.randn(s.M, N, device="cuda", generator=self.gen))

    # ---- runs ----------------------------------------------------------------------------------------------------------
    def run(self, E, bn, *, w=None, layout=None, out_of_place=False, batch=None, a=None):
        s = self.s
        outs = {k: v.clone() for k, v in self.init.items()}
        kw = dict(a_row_stride=self.rs, a_batch_stride=self.bs, w_layout=layout or s.layout, ldw=self.ldw if w is None else s.K,
                  batch=batch or s.batch, bias=self.bias, act=s.act, out_batch_rows=s.out_batch_rows,
                  out_row_offset=s.out_row_offset, head_major_rows=s.hmr, bn=bn)
        if "out_h" in outs:
            kw.update(out_h=outs["out_h"], ldo_h=(s.N // 2 if s.act == 2 else s.N) + 8 if s.out == "h" else 0)
        if "out_f" in outs:
            kw.update(out_f=outs["out_f"], ldo_f=s.N + 8)
        if s.out == "resid":
            resid = self.init["out_f"].clone() if out_of_place else outs["out_f"]
            if out_of_place:
                outs["out_f"].fill_(float("nan"))
            kw.update(resid=resid, ld_resid=s.N + 8, resid_mode=1)
        if s.out == "pos":
            kw.update(resid=self.table, ld_resid=s.N, resid_mode=2)
        E.gemm_ex(self.A if a is None else a, self.W if w is None else w, s.M, s.N, s.K, dtype=self.dt, **kw)
        torch.cuda.synchronize()
        return outs

    def bns(self):
        return (64, 128) if self.s.N % 128 == 0 else (64,)

    def written_mask(self, name):
        """True where the epilogue writes `name`"""
        s, buf = self.s, self.init[name]
        if s.out == "hm":
            m = torch.zeros(buf.numel(), dtype=torch.bool, device="cuda")
            m[: s.M * s.N] = True                   # batch 1, M a multiple of R: a permutation of the first M N elements
            return m
        m = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
        cols = s.N // 2 if s.act == 2 else s.N
        for b in range(s.batch):
            r0 = b * s.out_batch_rows + s.out_row_offset
            m[r0: r0 + s.M, :cols] = True
        return m

    def check_outside(self, outs):
        for name, buf in outs.items():
            keep = ~self.written_mask(name)
            assert same_bits(buf[keep], self.init[name][keep]), f"{self.s.site}: {name} written outside its destination"

    # ---- reference -----------------------------------------------------------------------------------------------------
    def check(self, runs):
        """runs: {bn: outputs}.  Every output of every run within the bound (bit for bit with exact inputs), the runs
        bit-identical to each other, nothing outside the destination touched."""
        s, dt, N, K = self.s, self.dt, self.s.N, self.s.K
        u16, sub = U16[dt], SUB16[dt]
        Aw = G.window_rows(self.A, self.rs, self.bs, s.M, K, s.batch)
        assert torch.isfinite(Aw).all()
        first = next(iter(runs.values()))
        for outs in runs.values():
            self.check_outside(outs)
            for n in outs:
                assert same_bits(outs[n], first[n]), f"{s.site}: BN {list(runs)} differ in {n}"
        for b in range(s.batch):
            for m0 in range(0, s.M, ROWS):
                m1 = min(s.M, m0 + ROWS)
                a = Aw[b, m0:m1].double()
                orow = b * s.out_batch_rows + s.out_row_offset + torch.arange(m0, m1, device="cuda")
                for n0 in range(0, N, COLS):
                    n1 = min(N, n0 + COLS)
                    w = self.W_eff[n0:n1].double()
                    v = a @ w.T
                    S = a.abs() @ w.abs().T
                    if self.bias is not None:
                        bb = self.bias[n0:n1].double()
                        v, S = v + bb, S + bb.abs()
                    acc = torch.zeros_like(S) if self.exact else ACC * S
                    del S
                    for bn, outs in runs.items():
                        self._compare(bn, outs, v, acc, orow, m0, m1, n0, n1, u16, sub)

    def _compare(self, bn, outs, v, acc, orow, m0, m1, n0, n1, u16, sub):
        s = self.s
        key = (s.site, s.fmt, "exact" if self.exact else s.layout, bn)
        if s.act == 2:
            g, u, ag, au = v[:, 0::2], v[:, 1::2], acc[:, 0::2], acc[:, 1::2]
            sl = G.silu(g)
            ref = sl * u
            prop = 1.1 * ag * u.abs() + sl.abs() * au + ref.abs() * ((2 + 1.173 * g.abs()) * 2.0 ** -23 + 3 * U32)
            bound = prop * (1 + u16) + u16 * ref.abs() + sub
            got = outs["out_h"][orow, n0 // 2: n1 // 2]
            return self._cmp(key, got, ref, bound)
        if s.act == 1:
            val, prop = G.gelu(v), 1.13 * acc + 2.0 ** -22 * v.abs()
        else:
            val, prop = v, acc
        if s.out in ("f", "resid", "pos"):
            if s.out == "resid":
                r = self.init["out_f"][orow, n0:n1].double()
            elif s.out == "pos":
                r = self.table[m0:m1, n0:n1].double()
            else:
                r = torch.zeros_like(v)
            ref = val + r
            got = outs["out_f"][orow, n0:n1]
            return self._cmp(key, got, ref, prop + OUT * (ref.abs() + r.abs()), exact_ok=s.act == 0)
        if s.out == "hm":
            idx = G.head_major_index(orow[:, None], torch.arange(n0, n1, device="cuda")[None], s.N, s.hmr)
            got = outs["out_h"][idx]
        else:
            got = outs["out_h"][orow, n0:n1]
        self._cmp(key, got, val, prop * (1 + u16) + u16 * val.abs() + sub, exact_ok=s.act == 0)

    def _cmp(self, key, got, ref, bound, exact_ok=True):
        got = got.double()
        assert torch.isfinite(got).all(), key
        if self.exact and exact_ok:
            assert torch.equal(got, ref), (key, float((got - ref).abs().max()))
            return
        _note(key, (got - ref).abs(), bound)

    # ---- the whole treatment of one spec -------------------------------------------------------------------------------
    def full(self, E):
        s = self.s
        runs = {bn: self.run(E, bn) for bn in self.bns()}
        self.check(runs)
        rule = s.rule_bn()
        base = runs[rule]
        del runs
        again = self.run(E, 0)                       # the rule's instantiation, run a second time
        for n in again:
            assert same_bits(again[n], base[n]), f"{s.site}: bn = 0 differs from bn = {rule} in {n}"
        if s.layout != "row_major":                  # tiled 16-bit = row-major; FP8 = bf16 row-major over dq(Q)
            rm = self.run(E, rule, w=self.W_eff, layout="row_major")
            for n in rm:
                assert same_bits(rm[n], base[n]), f"{s.site}: {s.layout} differs from row-major in {n}"
        if s.out == "resid":
            oop = self.run(E, rule, out_of_place=True)
            dst = self.written_mask("out_f")
            assert same_bits(oop["out_f"][dst], base["out_f"][dst]), f"{s.site}: in-place residual differs from out-of-place"


# ---- call sites at production geometry -------------------------------------------------------------------------------------
WHISPER = {"small": dict(d=768, f=3072, mels=80, Ld=12), "large-v3": dict(d=1280, f=5120, mels=128, Ld=32)}
T, TP = 1500, 3002   # encoder positions; mel frames + 2 padding rows


def whisper_spec(site, geo, B, dt):
    g = WHISPER[geo]
    d, f, C = g["d"], g["f"], g["mels"]
    name = f"whisper-{geo}.{site}"
    if site == "conv1":
        return Spec(name, dt, 3000, d, 3 * C, batch=B, a_row_stride=C, frame=C, a_rows=TP, bias=True, act=1, out="h",
                    out_batch_rows=TP, out_row_offset=1)
    if site == "conv2":
        return Spec(name, dt, T, d, 3 * d, batch=B, a_row_stride=2 * d, frame=d, a_rows=TP, bias=True, act=1, out="pos",
                    out_batch_rows=T)
    shapes = {"qkv": (3 * d, d, 0, "h"), "fc1": (f, d, 1, "h"), "o": (d, d, 0, "resid"), "fc2": (d, f, 0, "resid"),
              "ckv": (g["Ld"] * 2 * d, d, 0, "hm")}
    N, K, act, out = shapes[site]
    return Spec(name, dt, B * T, N, K, bias=True, act=act, out=out, hmr=T if out == "hm" else 0)


WHISPER_CASES = []
for _i, (_geo, _site) in enumerate([(g, s) for g in WHISPER for s in ("conv1", "conv2", "qkv", "fc1", "o", "fc2", "ckv")]):
    for _j, _dt in enumerate(("fp16", "bf16")):
        _B = (1, 3, 16)[(_i + _j) % 3]
        if _site == "ckv":
            _B = min(_B, 3 if _geo == "small" else 1)   # the head-major K/V of 16 large-v3 utterances is 4 GB per copy
        WHISPER_CASES.append((_geo, _site, _B, _dt))


@pytest.mark.parametrize("geo,site,B,dt", WHISPER_CASES, ids=[f"{g}-{s}-B{b}-{d}" for g, s, b, d in WHISPER_CASES])
def test_whisper_site(E, geo, site, B, dt):
    Prob(E, whisper_spec(site, geo, B, dt)).full(E)


LLAMA = {
    "llama-3-8b": dict(d=4096, qkv=6144, qd=4096, f=14336, vocab=128256),
    "qwen3-14b": dict(d=5120, qkv=7168, qd=5120, f=17408, vocab=151936),
    "qwen3-32b": dict(d=5120, qkv=10240, qd=8192, f=25600, vocab=151936),
}
LAYOUTS = [("tiled", "bf16"), ("tiled", "fp16"), ("float8_e4m3", "bf16")]


def llama_spec(site, geo, R, layout, dt):
    g = LLAMA[geo]
    shapes = {"qkv": (g["qkv"], g["d"], 0, "h"), "o": (g["d"], g["qd"], 0, "resid"), "gate_up": (2 * g["f"], g["d"], 2, "h"),
              "down": (g["d"], g["f"], 0, "resid"), "lm_head": (g["vocab"], g["d"], 0, "f")}
    N, K, act, out = shapes[site]
    return Spec(f"{geo}.{site}", dt, R, N, K, layout=layout, act=act, out=out)


LLAMA_CASES = []
for _i, (_geo, _site) in enumerate([(g, s) for g in LLAMA for s in ("qkv", "o", "gate_up", "down")]):
    for _j, (_lay, _dt) in enumerate(LAYOUTS):
        LLAMA_CASES.append((_geo, _site, (129, 512, 37)[(_i + _j) % 3], _lay, _dt))
# lm_head: the last row of a prefill (M = 1), the batched prefill's last rows (M = B <= 16), every row (M = n)
LLAMA_CASES += [("llama-3-8b", "lm_head", 1, "float8_e4m3", "bf16"), ("llama-3-8b", "lm_head", 16, "tiled", "bf16"),
                ("llama-3-8b", "lm_head", 130, "tiled", "fp16"), ("qwen3-14b", "lm_head", 1, "tiled", "bf16"),
                ("qwen3-14b", "lm_head", 7, "float8_e4m3", "bf16"), ("qwen3-32b", "lm_head", 64, "float8_e4m3", "bf16")]


@pytest.mark.parametrize("geo,site,R,layout,dt", LLAMA_CASES, ids=[f"{g}-{s}-R{r}-{l}-{d}" for g, s, r, l, d in LLAMA_CASES])
def test_llama_site(E, geo, site, R, layout, dt):
    Prob(E, llama_spec(site, geo, R, layout, dt)).full(E)


# ---- edges ---------------------------------------------------------------------------------------------------------------
EDGES = [
    # M around the 128-row tile, with each epilogue (K = 200: K % 64 = 8)
    Spec("edge.M1", "fp16", 1, 128, 200, bias=True, out="h"),
    Spec("edge.M63", "bf16", 63, 128, 200, out="resid"),
    Spec("edge.M64", "fp16", 64, 256, 200, bias=True, act=1, out="h"),
    Spec("edge.M127", "bf16", 127, 128, 200, bias=True, act=1, out="f"),
    Spec("edge.M128", "fp16", 128, 128, 200, act=2, out="h"),
    Spec("edge.M129", "bf16", 129, 192, 200, bias=True, out="f"),
    Spec("edge.M1500", "fp16", 1500, 128, 200, bias=True, out="hm", hmr=500),
    # K tails: row-major K % 64 in {8, 24, 56}, K in {8, 32}; GELU into fp32 at short K (small acc)
    Spec("edge.K88", "fp16", 130, 128, 88, bias=True, act=1, out="f"),
    Spec("edge.K184", "bf16", 130, 128, 184, bias=True, act=1, out="f"),
    Spec("edge.K520", "fp16", 300, 256, 520, out="resid"),
    Spec("edge.K8", "fp16", 200, 128, 8, bias=True, act=1, out="f"),
    Spec("edge.K32", "bf16", 200, 128, 32, bias=True, act=1, out="f"),
    Spec("edge.K32h", "fp16", 70, 64, 32, act=1, out="h"),
    # tiled / FP8: K % 64 = 32
    Spec("edge.tiledK96", "bf16", 129, 128, 96, layout="tiled", bias=True, act=1, out="f"),
    Spec("edge.tiledK4128", "fp16", 65, 256, 4128, layout="tiled", out="resid"),
    Spec("edge.fp8K96", "bf16", 129, 128, 96, layout="float8_e4m3", bias=True, act=1, out="f"),
    Spec("edge.fp8K1056", "bf16", 200, 256, 1056, layout="float8_e4m3", act=2, out="h"),
    # N = 64: one N tile (BN 64 only)
    Spec("edge.N64", "bf16", 129, 64, 256, bias=True, out="f"),
    Spec("edge.N64fp8", "bf16", 129, 64, 256, layout="float8_e4m3", out="resid"),
    # strides: A rows longer than K (NaN between), W rows longer than K (NaN between)
    Spec("edge.lda", "fp16", 257, 128, 200, a_row_stride=264, bias=True, out="f"),
    Spec("edge.ldw", "bf16", 257, 128, 200, ldw=264, act=1, out="h"),
]
# plain [M, K] x [N, K] products, bias + GELU into 16-bit and bias into fp32 (the shapes of the encoder's first GEMM test)
for _M, _N, _K in ((128, 64, 64), (1500, 768, 768), (200, 64, 240), (3000, 2304, 768), (333, 512, 3072), (1, 128, 8),
                   (129, 192, 72)):
    for _dt in ("fp16", "bf16"):
        EDGES.append(Spec(f"plain.{_M}x{_N}x{_K}", _dt, _M, _N, _K, bias=True, act=1, out="h"))
        EDGES.append(Spec(f"plain.{_M}x{_N}x{_K}", _dt, _M, _N, _K, bias=True, out="f"))
# ring wrap: num_kb = ceil(K / 64) in {STAGES - 1, STAGES, STAGES + 1} for 8 stages (BN 64), 6 (BN 128, 16-bit) and
# 5 (BN 128, FP8); every spec runs in both instantiations
for _lay, _dt in (("row_major", "fp16"), ("tiled", "bf16"), ("float8_e4m3", "bf16")):
    for _kb in ((7, 8, 9, 5, 6) if _lay != "float8_e4m3" else (7, 8, 9, 4, 5, 6)):
        EDGES.append(Spec(f"edge.ring{_kb}", _dt, 129, 256, 64 * _kb - (32 if _kb % 2 and _lay != "row_major" else 0),
                          layout=_lay, bias=True, out="f"))


@pytest.mark.parametrize("spec", EDGES, ids=[f"{s.site}-{s.layout}-{s.dt}-K{s.K}-{s.out}{s.act}" for s in EDGES])
def test_edge(E, spec):
    Prob(E, spec).full(E)


# ---- exact designed inputs ---------------------------------------------------------------------------------------------
EXACT = [
    whisper_spec("conv1", "small", 3, "fp16"), whisper_spec("conv1", "large-v3", 2, "bf16"),
    whisper_spec("conv2", "small", 3, "bf16"), whisper_spec("conv2", "large-v3", 2, "fp16"),
    whisper_spec("ckv", "small", 2, "fp16"), whisper_spec("o", "small", 3, "bf16"),
    llama_spec("qkv", "llama-3-8b", 129, "tiled", "bf16"), llama_spec("down", "qwen3-14b", 37, "float8_e4m3", "bf16"),
    llama_spec("gate_up", "llama-3-8b", 130, "tiled", "fp16"), llama_spec("gate_up", "qwen3-14b", 64, "float8_e4m3", "bf16"),
]


@pytest.mark.parametrize("spec", EXACT, ids=[f"{s.site}-{s.layout}-{s.dt}" for s in EXACT])
def test_exact_routing(E, spec):
    """integer weights and sparse {-1, 0, 1} activations: every store exact.  GELU and SwiGLU become act 0 on the same
    columns, so the window and batch of every row, the output row, the table row, the head-major address and the
    interleaved (gate, up) columns are compared bit for bit."""
    spec = dataclasses.replace(spec, act=0)
    p = Prob(E, spec, exact=True)
    runs = {bn: p.run(E, bn) for bn in p.bns()}
    p.check(runs)


@pytest.mark.parametrize("layout,dt", [("tiled", "bf16"), ("tiled", "fp16"), ("float8_e4m3", "bf16"), ("row_major", "fp16")])
def test_exact_swiglu_pairing(E, layout, dt):
    """one-hot activation rows, gate rows in {0, 20, 24, 28} and up rows in [-8, 8]: silu(gate) is exactly gate (or 0) in
    fp32, so out[m][j] = gate_j * up_j bit for bit -- a swapped or shifted (gate, up) pair gives silu(up) * gate"""
    s = Spec("swiglu-exact", dt, 200, 512, 256, layout=layout, act=2, out="h")
    p = Prob(E, s, exact=True)
    gen = torch.Generator(device="cuda").manual_seed(8)
    w = torch.empty(s.N, s.K, dtype=torch.float64, device="cuda")
    choice = torch.tensor([0.0, 20.0, 24.0, 28.0], dtype=torch.float64, device="cuda")
    w[0::2] = choice[torch.randint(0, 4, (s.N // 2, s.K), device="cuda", generator=gen)]
    w[1::2] = torch.randint(-8, 9, (s.N // 2, s.K), device="cuda", generator=gen).double()
    p._set_weights(E, w.to(p.dt))
    assert torch.equal(p.W_eff.double(), w)
    A = torch.zeros(s.M, s.K, dtype=torch.float64, device="cuda")
    A[torch.arange(s.M), torch.arange(s.M) % s.K] = 1
    p.A.view(-1)[: s.M * s.K] = A.reshape(-1).to(p.dt)
    runs = {bn: p.run(E, bn) for bn in p.bns()}
    want = (w[0::2] * w[1::2]).T[torch.arange(s.M) % s.K]          # [M, N/2]
    for bn, outs in runs.items():
        got = outs["out_h"][: s.M, : s.N // 2].double()
        assert torch.equal(got, want), (bn, float((got - want).abs().max()))
        p.check_outside(outs)


# ---- invariances ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("site", ["conv1", "conv2"])
def test_batch_rows_do_not_depend_on_batch(E, site):
    """batch 5 of a B = 16 call equals the same sequence run alone (B = 1), bit for bit"""
    s = whisper_spec(site, "small", 16, "fp16")
    p = Prob(E, s)
    full = p.run(E, 0)
    one = Prob(E, dataclasses.replace(s, batch=1))
    one.A[: p.bs] = p.A[5 * p.bs: 6 * p.bs]
    one.W, one.bias = p.W, p.bias
    if p.table is not None:
        one.table[: s.M] = p.table[: s.M]
    alone = one.run(E, 0)
    name = "out_h" if site == "conv1" else "out_f"
    r5 = 5 * s.out_batch_rows
    assert same_bits(full[name][r5: r5 + s.out_batch_rows + s.out_row_offset],
                     alone[name][: s.out_batch_rows + s.out_row_offset])


# ---- rejections ----------------------------------------------------------------------------------------------------------
def test_rejects_bad_arguments_and_launches_nothing(E):
    from speech_to_speech_b200._lib import S2SError
    M, N, K = 64, 128, 256
    a = torch.zeros(M + 8, K, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(N, K, dtype=torch.bfloat16, device="cuda")
    wt = E.tile_weights(w)
    wq = E.tile_weights(w, "float8_e4m3")
    out_h = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    out_f = torch.zeros(M, N, device="cuda")
    ok = dict(out_f=out_f, ldo_f=N)
    E.gemm_ex(a, w, M, N, K, **ok)
    torch.cuda.synchronize()
    bad = [
        (a, w, M, 96, K, ok),                                             # N % 64
        (a, w, M, N, 100, ok),                                            # K % 8
        (a, wt, M, N, 80, dict(ok, w_layout="tiled")),                    # K % 32 with tiled weights
        (a, wq, M, N, K, dict(ok, w_layout="float8_e4m3", dtype=torch.float16)),   # FP8 without bf16
        (a.view(-1)[1:], w, M, N, K, ok),                                 # A not 16-byte aligned
        (a, w.view(-1)[4:], M, N, K, ok),                                 # W not 16-byte aligned
        (a, w, M, N, K, dict(ok, a_row_stride=K + 4)),                    # row stride not a multiple of 8
        (a, w, M, N, K, dict(ok, ldw=K + 4)),
        (a, w, M, N, K, dict(ok, w_layout=3)),                            # unknown layout
        (a, w, 0, N, K, ok),                                              # empty
        (a, w, M, N, K, {}),                                              # no output
        (a, w, M, N, K, dict(out_h=out_h, ldo_h=N, resid=out_f, ld_resid=N, resid_mode=1)),   # residual without out_f
        (a, w, M, N, K, dict(ok, resid=out_f, ld_resid=N, resid_mode=0)),                       # resid_mode outside {1, 2}
        (a, w, M, N, K, dict(ok, resid=out_f, ld_resid=N, resid_mode=3)),
        (a, w, M, N, K, dict(ok, act="swiglu")),                                               # SwiGLU into fp32
        (a, w, M, N, K, dict(ok, out_h=out_h, ldo_h=N, act="swiglu")),                         # SwiGLU with both outputs
        (a, w, M, N, K, dict(out_h=out_h, ldo_h=N, act="swiglu", head_major_rows=64)),         # SwiGLU head-major
        (a, w, M, N, K, dict(ok, head_major_rows=64)),                                         # head-major without out_h
        (a, w, M, N, K, dict(ok, act=3)),                                                      # unknown act
        (a, w, M, N, K, dict(ok, bn=96)),                                                      # bn outside {0, 64, 128}
        (a, w, M, 192, K, dict(ok, bn=128)),                                                   # bn 128 with N % 128
    ]
    before = E.launch_count()
    for i, (aa, ww, m, n, k, kw) in enumerate(bad):
        with pytest.raises(S2SError):
            E.gemm_ex(aa, ww, m, n, k, **kw)
    assert E.launch_count() == before, "a rejected call launched a kernel"
