"""GPU tests (H100) of the codec decoder's contraction kernels one at a time (csrc/codec_decode.cu through
s2s_codec_contract): path 0 = conv1d_f32_kernel (fp32 FMA), path 1 = conv1d_tc_kernel (tensor cores, fp32 activations
converted to fp16 while staged), path 2 = conv1d_tc16_kernel (tensor cores fed fp16 activations through cp.async), against
a float64 evaluation of the same contraction

    Y[t, n] = epi(bias[n % bias_mod] + sum_j sum_c X[t + x_row0 + j * dil, c] * W[j][c][n]),   rows of X outside [0, T_in) = 0,
    epi = activation (exact GELU / SiLU), then * scale[n], then + resid[t, n].

Bound per output.  S = sum_j sum_c |X W| over the operands the kernel multiplies (fp16-rounded on paths 1 and 2), times
|scale[n]| where there is a scale:
    every path, against the reference on the same operands:       |y - ref| <= 2^-16 S + 8 * 2^-24 (|ref| + |resid|)
    paths 1 and 2, against the reference on the fp32 operands:    |y - ref| <= 2^-9 S  + 8 * 2^-24 (|ref| + |resid|)
The first term is the summation order of an fp32 accumulation (with random signs it stays near 2^-24 S); the second, on
paths 1 and 2, what rounding both operands to fp16 costs (at most ~2^-10 S, times the activation's slope, <= 1.13); the
last one the epilogue's own roundings.

Shapes: every contraction the decoder issues at the published geometry (hidden 1024, inter 3072, decoder_dim 1536, rates
(8, 5, 4, 3), ratios (2, 2)), built as the decoder builds its ConvArgs, and the Qwen3-TTS text projection (path 0 only), at
row counts on both sides of the 64-row (fp32) and 128-row (tensor-core) tiles, with one or three sequences per launch;
plus shapes off the fast paths (odd C_in, C_in and N off the 16/32/64 tiles, row strides that are not a multiple of 4).
Every run also checks: y is filled with NaN beforehand and everything outside rows [t0, T_out) x columns [0, N) of each
sequence -- rows below t0, columns [N, ldy), the rows between sequences -- comes back bit for bit; the rows between the
sequences of x are NaN (a read past T_in shows); two runs are bit-identical; paths 1 and 2 are bit-identical when
x16 = fp16(x); the transposed convolutions also match torch's conv_transpose1d (float64) with the cousin's trim."""
import dataclasses
import functools
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

H, I, D, RATES = 1024, 3072, 1536, (8, 5, 4, 3)
SUM_REL, FP16_REL, OUT_REL = 2.0 ** -16, 2.0 ** -9, 8 * 2.0 ** -24
S2S_ERR_INVALID = -1


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@dataclasses.dataclass(frozen=True)
class Spec:
    name: str
    k: int
    C_in: int
    N: int
    w_scale: float            # weights uniform in [-w_scale, w_scale), the scale codec_init_random gives the tensor (cslot)
    dil: int = 1
    x_row0: int = 0
    bias_mod: int = 0         # 0: no bias
    act: int = 0              # 0 none, 1 exact GELU, 2 SiLU
    scale: bool = False
    resid: bool = False       # residual added in place (resid = y), as the decoder adds every residual
    tconv: int = 0            # stride of the transposed convolution this contraction computes (0: none)
    paths: tuple = (0, 1, 2)

    @property
    def T_in_extra(self):     # the 2-tap transposed convolution reads rows t and t + 1: T_out = T_in - 1
        return 1 if self.tconv and self.k == 2 else 0


def _linear(name, K, N, rs, **kw):
    return Spec(name, 1, K, N, rs, **kw)


def _conv7(name, C_in, C_out, dil, rs, **kw):   # causal_conv_args(..., k = 7, dil, ...)
    return Spec(name, 7, C_in, C_out, rs, dil=dil, x_row0=-6 * dil, bias_mod=C_out, **kw)


SPECS = [
    _linear("tf_qkv", H, 3 * H, H ** -0.5),
    _linear("tf_o", H, H, H ** -0.5, scale=True, resid=True),
    _linear("tf_gate_up", H, 2 * I, H ** -0.5),
    _linear("tf_down", I, H, I ** -0.5, scale=True, resid=True),
    Spec("up_tconv_k2s2", 1, H, 2 * H, H ** -0.5, bias_mod=H, tconv=2),
    _linear("convnext_pw1", H, 4 * H, H ** -0.5, bias_mod=4 * H, act=1),
    _linear("convnext_pw2", 4 * H, H, 0.5 * H ** -0.5, bias_mod=H, scale=True, resid=True),
    _conv7("decoder0", H, D, 1, (7 * H) ** -0.5),
]
for _i, _r in enumerate(RATES):
    _cin, _cout = D >> _i, D >> (_i + 1)
    SPECS.append(Spec(f"block{_i}_tconv_s{_r}", 2, _cin, _r * _cout, (2 * _cin) ** -0.5, bias_mod=_cout, tconv=_r))
    SPECS += [_conv7(f"block{_i}_conv7_d{_d}", _cout, _cout, _d, (7 * _cout) ** -0.5) for _d in (1, 3, 9)]
    SPECS.append(_linear(f"block{_i}_1x1", _cout, _cout, _cout ** -0.5, bias_mod=_cout, resid=True))
SPECS += [
    _conv7("final_conv", D >> 4, 1, 1, 0.5 * (7 * (D >> 4)) ** -0.5),
    _linear("text_fc1", 2048, 2048, 2048 ** -0.5, bias_mod=2048, act=2, paths=(0,)),   # qwen3tts.cu linear_f32
    _linear("text_fc2", 2048, 1024, 0.7 * 2048 ** -0.5, bias_mod=1024, paths=(0,)),
]
# off the fast paths: odd C_in (pair padding of the packed weights; no fp16-operand path), C_in and N off the 16 / 32 / 64
# tiles, bias_mod below N, taps reaching past T_in (x_row0 > 0), a single input channel, a single output
EDGE_SPECS = [
    Spec("odd_cin75_n100", 3, 75, 100, (3 * 75) ** -0.5, dil=2, x_row0=-4, bias_mod=100, act=1, paths=(0, 1)),
    Spec("cin40_n36", 7, 40, 36, (7 * 40) ** -0.5, dil=3, x_row0=-18, bias_mod=12, act=2, scale=True, resid=True),
    Spec("cin24_n68_ahead", 2, 24, 68, (2 * 24) ** -0.5, dil=2, x_row0=1, bias_mod=68),
    Spec("cin1_n33", 1, 1, 33, 1.0, bias_mod=33, paths=(0, 1)),
    Spec("cin7_n1", 5, 7, 1, 35 ** -0.5, dil=4, x_row0=-16, bias_mod=1, paths=(0, 1)),
]
# (output rows per sequence, sequences): around the 64-row fp32 and 128-row tensor-core tiles; 99 = 33 frames x 3 sessions
# as the transformer sees them, 33 x 3 as the batched convolutions see them
ROWS = [(1, 1), (63, 1), (64, 3), (65, 1), (99, 1), (128, 1), (129, 3), (33, 3)]
CASES = [(s, r, b) for s in SPECS + EDGE_SPECS for r, b in ROWS]


def _f32_tile(sms, rows, N, B):
    """The n tile conv1d_f32_launch picks: 32 while fewer (64-row x 64-column) tiles than SMs, else 64."""
    return 32 if math.ceil(rows / 64) * math.ceil(N / 64) * B < sms else 64


def _tconv_taps(wct, s):
    """ConvTranspose1d weight [C, O, k] (k = s or 2 s) -> the documented taps x [C][s * O] layout (codec_bind_tensor, C_TCONV)."""
    C, O, k = wct.shape
    flat = lambda w: w.transpose(0, 2, 1).reshape(C, s * O)   # W'[c][r * O + o] = W[c][o][r]
    if k == s:
        return np.ascontiguousarray(flat(wct)[None])
    return np.ascontiguousarray(np.stack([flat(wct[:, :, s:]), flat(wct[:, :, :s])]))   # tap 0 reads X[t], tap 1 X[t + 1]


@functools.lru_cache(maxsize=None)
def _weights(spec):
    """(W [k][C_in][N] f32, ConvTranspose1d weight or None) on the device, seeded by the contraction's name."""
    rng = np.random.Generator(np.random.PCG64(zlib.crc32(spec.name.encode())))
    uni = lambda shape: (spec.w_scale * (2 * rng.random(shape, dtype=np.float32) - 1)).astype(np.float32)
    if spec.tconv:
        wct = uni((spec.C_in, spec.N // spec.tconv, spec.k * spec.tconv))
        return torch.from_numpy(_tconv_taps(wct, spec.tconv)).cuda(), torch.from_numpy(wct).cuda()
    return torch.from_numpy(uni((spec.k, spec.C_in, spec.N))).cuda(), None


def _reference(spec, x, w, T_out, bias, scale, resid):
    """float64 contraction of x [B, T_in, C_in] with w [k, C_in, N] -> (Y [B, T_out, N], S = sum |x w| (* |scale|))."""
    B, T_in, C_in = x.shape
    idx = torch.arange(T_out, device=x.device)[:, None] + spec.x_row0 + spec.dil * torch.arange(spec.k, device=x.device)
    ok = (idx >= 0) & (idx < T_in)
    g = (x[:, idx.clamp(0, T_in - 1)] * ok[None, :, :, None]).reshape(B, T_out, spec.k * C_in)
    w2 = w.reshape(spec.k * C_in, spec.N)
    v, S = g @ w2, g.abs() @ w2.abs()
    if bias is not None:
        v = v + bias.double()[torch.arange(spec.N, device=x.device) % spec.bias_mod]
    if spec.act == 1:
        v = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
    elif spec.act == 2:
        v = v * torch.sigmoid(v)
    if scale is not None:
        v, S = v * scale.double(), S * scale.double().abs()
    if resid is not None:
        v = v + resid
    return v, S


def _tconv_op(x, wct, bias, s):
    """conv_transpose1d in float64, trimmed by k - s at both ends (Qwen3OmniMoeCausalTransConvNet), as [B, rows, s * O]."""
    out = F.conv_transpose1d(x.transpose(1, 2), wct, bias.double(), stride=s)
    pad = wct.shape[2] - s
    if pad:
        out = out[:, :, pad:out.shape[2] - pad]
    return out.transpose(1, 2).reshape(x.shape[0], -1, s * wct.shape[1])


def _check(got, ref, S, resid_abs, rel, what):
    """Assert |got - ref| <= rel S + OUT_REL (|ref| + |resid|) everywhere; -> the largest err / bound."""
    if got.numel() == 0:
        return 0.0
    bound = rel * S + OUT_REL * (ref.abs() + resid_abs)
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} outputs outside the bound; first at (b, t - t0, n) = {i}: "
                             f"got {float(got[i]):.9g}, reference {float(ref[i]):.9g}, bound {float(bound[i]):.3g}")
    return float((err / bound.clamp_min(1e-300)).max())


def _bits(t):
    return t.view(torch.int32)


def _run(E, spec, rows, B, *, t0=0, ldx=None, gap=2, col_pad=3):
    """Run `spec` on each of its paths (T_out = rows per sequence, B sequences) and check everything the module docstring lists.
    -> {path: (err / bound against the same operands, err / bound against the fp32 operands or None)}."""
    T_out, T_in = rows, rows + spec.T_in_extra
    C_in, N = spec.C_in, spec.N
    ldx = ldx or C_in
    rng = np.random.Generator(np.random.PCG64([zlib.crc32(spec.name.encode()), rows, B, t0, ldx]))
    w, wct = _weights(spec)
    xh = np.full((B, T_in + gap, ldx), np.nan, np.float32)              # NaN: padding columns and the rows between sequences
    xh[:, :T_in, :C_in] = rng.standard_normal((B, T_in, C_in), dtype=np.float32)
    x = torch.from_numpy(xh).cuda()
    x16 = x.half()
    bias = torch.from_numpy(rng.uniform(-0.02, 0.02, spec.bias_mod).astype(np.float32)).cuda() if spec.bias_mod else None
    scale = torch.from_numpy(rng.uniform(0.2, 0.6, N).astype(np.float32)).cuda() if spec.scale else None
    y0 = torch.full((B, T_out + gap, N + col_pad), float("nan"), device="cuda")
    if spec.resid:
        y0[:, :T_out, :N] = torch.from_numpy(rng.standard_normal((B, T_out, N), dtype=np.float32)).cuda()
    keep = torch.ones(y0.shape, dtype=torch.bool, device="cuda")
    keep[:, t0:T_out, :N] = False
    paths = [p for p in spec.paths if p != 2 or (C_in % 8 == 0 and N % 4 == 0 and ldx % 8 == 0)]
    outs = {}
    for p in paths:
        runs = []
        for _ in range(2):
            y = y0.clone()
            E.codec_contract(None if p == 2 else x, w, y, path=p, x16=x16 if p == 2 else None, T_in=T_in, T_out=T_out,
                             x_row0=spec.x_row0, dil=spec.dil, bias=bias, bias_mod=spec.bias_mod or None, act=spec.act,
                             scale=scale, resid=y if spec.resid else None, t0=t0)
            runs.append(y)
        what = f"{spec.name} rows {rows} x {B} t0 {t0} ldx {ldx} path {p}"
        assert torch.equal(_bits(runs[0]), _bits(runs[1])), f"{what}: two runs differ"
        assert torch.equal(_bits(runs[0])[keep], _bits(y0)[keep]), f"{what}: wrote outside rows [t0, T_out) x columns [0, N)"
        outs[p] = runs[0]
    if 1 in outs and 2 in outs:
        assert torch.equal(_bits(outs[1]), _bits(outs[2])), f"{spec.name} rows {rows} x {B}: paths 1 and 2 differ"

    xv = x[:, :T_in, :C_in].double()
    xr = x[:, :T_in, :C_in].half().double()
    resid = y0[:, :T_out, :N].double() if spec.resid else None
    ref32, S32 = _reference(spec, xv, w.double(), T_out, bias, scale, resid)
    ref16, S16 = _reference(spec, xr, w.half().double(), T_out, bias, scale, resid) if set(outs) - {0} else (None, None)
    ra = resid[:, t0:].abs() if resid is not None else 0.0
    ratios = {}
    for p, y in outs.items():
        got = y[:, t0:T_out, :N].double()
        what = f"{spec.name} rows {rows} x {B} t0 {t0} ldx {ldx} path {p}"
        if p == 0:
            ratios[p] = (_check(got, ref32[:, t0:], S32[:, t0:], ra, SUM_REL, what), None)
        else:
            ratios[p] = (_check(got, ref16[:, t0:], S16[:, t0:], ra, SUM_REL, what + " vs fp16 operands"),
                         _check(got, ref32[:, t0:], S16[:, t0:], ra, FP16_REL, what + " vs fp32 operands"))
        if wct is not None:   # the operation itself: torch's transposed convolution on the same operands
            xo, wo = (xv, wct.double()) if p == 0 else (xr, wct.half().double())
            op = _tconv_op(xo, wo, bias, spec.tconv)
            assert op.shape == (B, T_out, N)
            _check(got, op[:, t0:], (S32 if p == 0 else S16)[:, t0:], 0.0, SUM_REL, what + " vs conv_transpose1d")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"RATIO {spec.name} rows={rows} B={B} t0={t0} ldx={ldx} f32_tile={_f32_tile(sms, max(T_out - t0, 0), N, B)} "
          + " ".join(f"path{p}={a:.4f}" + (f"/{b:.4f}" if b is not None else "") for p, (a, b) in ratios.items()))
    return ratios


@pytest.mark.parametrize("spec,rows,B", CASES, ids=[f"{s.name}-{r}x{b}" for s, r, b in CASES])
def test_contraction_matches_float64(E, spec, rows, B):
    _run(E, spec, rows, B)


_BY_NAME = {s.name: s for s in SPECS + EDGE_SPECS}


@pytest.mark.parametrize("t0", [0, 5, 69, 70, 75])
@pytest.mark.parametrize("name", ["decoder0", "block1_conv7_d9", "block2_tconv_s4", "tf_o", "cin40_n36"])
def test_trimmed_rows(E, name, t0):
    """Causal trimming: only rows [t0, T_out) are computed (t0 = T_out - 1: one row; t0 >= T_out: nothing at all)."""
    _run(E, _BY_NAME[name], 70, 3, t0=t0)


@pytest.mark.parametrize("pad", [5, 8], ids=["ldx_pad5_scalar_staging", "ldx_pad8"])
@pytest.mark.parametrize("name", ["block2_conv7_d3", "decoder0", "convnext_pw2", "cin40_n36", "odd_cin75_n100"])
def test_padded_rows_of_x(E, name, pad):
    """ldx > C_in with NaN in the padding columns.  ldx = C_in + 5 is not a multiple of 4: conv1d_tc_kernel stages element
    by element and the fp16-operand path does not apply; C_in + 8 keeps every path."""
    _run(E, _BY_NAME[name], 65, 2, t0=3, ldx=_BY_NAME[name].C_in + pad)


def test_both_f32_tiles_are_covered():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {_f32_tile(sms, r, s.N, b) for s, r, b in CASES if 0 in s.paths}
    assert tiles == {32, 64}, tiles


def test_invalid_arguments_are_refused(E):
    import ctypes as C

    from speech_to_speech_b200 import _lib
    lib, ctx = _lib.load(), E.get_context(0)
    x = torch.zeros(64, 32, device="cuda")
    x16 = torch.zeros(64, 32, dtype=torch.float16, device="cuda")
    w = torch.zeros(1, 16, 8, device="cuda")
    y = torch.zeros(64, 8, device="cuda")
    b = torch.zeros(8, device="cuda")

    def call(path, **kw):
        a = dict(x=x.data_ptr(), ldx=16, T_in=8, x_row0=0, x16=x16.data_ptr(), w=w.data_ptr(), k=1, dil=1, C_in=16, N=8,
                 bias=None, bias_mod=8, act=0, scale=None, resid=None, ldr=0, y=y.data_ptr(), ldy=8, T_out=8, t0=0, batch=1,
                 x_bs=0, y_bs=0, r_bs=0)
        a.update(kw)
        return lib.s2s_codec_contract(ctx, C.byref(_lib.ConvArgs(**a)), path, None)

    assert call(0) == 0 and call(1) == 0 and call(2) == 0
    refused = [(0, dict(N=0)), (0, dict(C_in=0)), (0, dict(k=0)), (0, dict(dil=0)), (0, dict(bias=b.data_ptr(), bias_mod=0)),
               (0, dict(x=None)), (0, dict(w=None)), (0, dict(y=None)), (2, dict(x16=None)), (0, dict(act=3)), (3, {}),
               (-1, {}), (0, dict(ldx=8)), (0, dict(ldy=4)), (0, dict(resid=y.data_ptr(), ldr=4)), (0, dict(batch=0)),
               (0, dict(T_out=-1)), (0, dict(t0=-1)), (2, dict(C_in=12)), (2, dict(N=6, ldy=8)), (2, dict(ldx=20)),
               (2, dict(batch=2, x_bs=4)), (2, dict(x16=x16.data_ptr() + 2))]
    for path, kw in refused:
        assert call(path, **kw) == S2S_ERR_INVALID, (path, kw)
