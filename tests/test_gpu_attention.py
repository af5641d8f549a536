"""GPU tests (H100) of the two attention kernels by themselves, against a float64 evaluation of the same operation on the
same 16-bit operands, at the shapes and cache lengths the models reach (caches of 4096 positions).

Part A -- prefill attention (csrc/attention_tc.cu through s2s_attention): O = softmax(Q K^T * scale [+ causal mask]) V, a
CTA per 128 query rows and head, 64-key tiles.  Chunked prefill calls it with Tq = n new rows behind `past` cached keys
(Tk = past + n), so query i sees keys j <= i + Tk - Tq; the K and V caches are separate [max_pos, kv_heads * hd] buffers.

Part B -- decode attention (ld_attn in csrc/llama_decode.cu, items planned by attn_plan in csrc/decode_common.cuh, through
s2s_decode_attention): one query per (session, head) over the session's `len` cached keys, cut into S key splits of
32-key blocks; CTA-level items (8 warps per split, a shared-memory merge) or warp-level items, the last split to finish
merges the split records.

Bound per output.  Let w_j be the float64 softmax weights of the output's query, A = sum_j w_j |v_j| (per component), and
    ds = hd * 2^-24 * max_j sum_c |q_c k_jc| * scale      (visible keys j; scale = 1 in part B: q carries it)
a bound on the error of an fp32 score (an fp32 dot product of hd terms, the scaling and the exponent argument; the
latter two are below |s| * 2^-23, which hd >= 64 covers).  A perturbation e_j of the scores, |e_j| <= ds, moves the
output by sum_j w_j (e_j - sum_i w_i e_i) v_j, at most 2 ds A.  Then
    part A:  |o - ref| <= u_P A + 2 ds A + 2^-20 A + u_o |ref| + sub * max_j w_j * sum_j |v_j|
    part B:  |o - ref| <=         2 ds A + 2^-20 A + u_o |ref|
u_P is the unit roundoff of the 16-bit P operand of the P V product: 2^-11 for fp16 (11 significant bits) and 2^-8 for
bf16 (8 significant bits).  Measured bf16 errors exceed a bound built on 2^-9 by up to 1.6x on causal rows with few keys.
The rounding of P is not normalised away: the kernel's row sum l adds the unrounded fp32 p, while P V multiplies the
rounded p, so each weight carries its own relative error of up to u_P.
sub = 2^-25 on fp16 bounds the absolute error of a p below the smallest normal fp16 (2^-14); it is 0 on bf16, which has
fp32's exponent range.  u_o is the output's unit roundoff (the same values as u_P).  2^-20 A covers exp2f / __expf (a few
ulps), the fp32 accumulation of P V and of l, and the normalisation.  Part B keeps P in fp32, hence no u_P term.  The
worst ratio error / bound per dtype is printed at the end of the module.

Exact designed inputs (bit equality, no tolerance):
  counting -- q = 0, so every visible score is exactly 0 and every p exactly 1; V_j = one-hot(f(j)) with f(j) = (j + 7 g)
    mod hd (g = kv head) or one component per key tile / block (j // 64 in part A, j // 32 in part B).  The output is
    round16(fl32(count_c * fl32(1 / n_visible))) -- the library builds without fast math, so 1.f / l is IEEE.  A key
    that is masked wrongly, a tile, block or split that is dropped, counted twice or cut short shows as a wrong count.
  peaks -- K rows are random unit vectors and q = alpha * k_t (alpha * scale = 60): query i scores > 25 higher on key t
    than on any other key.  t = the first masked key i + off + 1, the last visible key i + off, key 0 (part A); key 0,
    key len - 1, block edges 32k - 1 / 32k and split edges (part B).  The bound above then separates the right answer
    from one with the peak key dropped or leaked by O(1).

Every part A run also checks: the output buffer (row stride ldo > heads * hd, one row more than B * Tq) is NaN-filled
beforehand and everything outside [B * Tq rows] x [heads * hd columns] comes back bit for bit; cache rows at and past Tk
hold NaN.  Every part B case runs twice with bit-identical outputs, and the entry point fails when a split counter is
left non-zero; cache rows at and past a session's len hold NaN."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_POS = 4096
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SUB = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}
SMALL = 2.0 ** -20
ALPHA = 60.0                      # peak score advantage scale (alpha * scale)
DTYPES = [torch.float16, torch.bfloat16]
_WORST = {}                       # (part, dtype) -> worst error / bound


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (part, dt), r in sorted(_WORST.items(), key=str):
        print(f"\nattention part {part} {dt}: worst error / bound = {r:.3f}")


def _note(part, dt, ratio):
    key = (part, str(dt).replace("torch.", ""))
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)


def _unit_rows(n, hd, gen):
    x = torch.randn(n, hd, device="cuda", generator=gen, dtype=torch.float64)
    return x / x.norm(dim=1, keepdim=True)


def _exact_counts(counts, n, dt):
    """round16(fl32(count * fl32(1 / n))) as the kernels' epilogues compute it (IEEE fp32 on the CPU)."""
    inv = torch.ones_like(n, dtype=torch.float32) / n.to(torch.float32)
    return (counts.to(torch.float32) * inv).to(dt)


# =============================================================================================== part A: prefill attention
def _prefill(E, dt, q, k, v, o, B, Tq, Tk, H, KVH, hd, ldq, ldk, ldv, ldo, scale, causal):
    from speech_to_speech_b200 import _lib
    code = {torch.float16: _lib.S2S_F16, torch.bfloat16: _lib.S2S_BF16}[dt]
    lib = _lib.load()
    _lib.check(lib.s2s_attention(E.get_context(0), C.c_void_p(q.data_ptr()), C.c_void_p(k.data_ptr()),
                                 C.c_void_p(v.data_ptr()), C.c_void_p(o.data_ptr()), B, Tq, Tk, H, KVH, hd, ldq, ldk, ldv,
                                 ldo, float(scale), 1 if causal else 0, code,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)), "s2s_attention")


class Prefill:
    """Operands of one s2s_attention call in the layout a caller uses.  B == 1 ("cache"): q rows inside a fused qkv row
    buffer [Tq, (H + 2 KVH) hd] as llama.cu passes them, K and V in one slot of the model's cache [2][MAX_POS][KVH hd]
    (rows >= Tk NaN, the V rows follow the K rows).  B > 1: q [B Tq, H hd + 8], K and V interleaved in one [B Tk, 2 KVH hd]
    buffer.  The output is [B Tq + 1, H hd + 24], NaN-filled."""

    def __init__(self, dt, B, Tq, Tk, H, KVH, hd):
        self.dt, self.B, self.Tq, self.Tk, self.H, self.KVH, self.hd = dt, B, Tq, Tk, H, KVH, hd
        kvd = KVH * hd
        nan = float("nan")
        if B == 1:
            assert Tk <= MAX_POS
            self.ldq, self.ldk, self.ldv = H * hd + 2 * kvd, kvd, kvd
            self.qbuf = torch.full((Tq, self.ldq), nan, dtype=dt, device="cuda")
            self.kv = torch.full((2, MAX_POS, kvd), nan, dtype=dt, device="cuda")
            self.q = self.qbuf[:, : H * hd]
            self.k, self.v = self.kv[0, :Tk], self.kv[1, :Tk]
            self.kptr, self.vptr = self.kv[0], self.kv[1]
        else:
            self.ldq, self.ldk, self.ldv = H * hd + 8, 2 * kvd, 2 * kvd
            self.qbuf = torch.full((B * Tq, self.ldq), nan, dtype=dt, device="cuda")
            self.kv = torch.full((B * Tk, 2 * kvd), nan, dtype=dt, device="cuda")
            self.q = self.qbuf[:, : H * hd]
            self.k, self.v = self.kv[:, :kvd], self.kv[:, kvd:]
            self.kptr, self.vptr = self.k, self.v
        self.ldo = H * hd + 24
        self.o = torch.full((B * Tq + 1, self.ldo), nan, dtype=dt, device="cuda")

    def views(self):
        """float64 [B, Tq, H, hd] q and [B, Tk, KVH, hd] k, v of what was stored."""
        B, Tq, Tk, H, KVH, hd = self.B, self.Tq, self.Tk, self.H, self.KVH, self.hd
        return (self.q.double().reshape(B, Tq, H, hd), self.k.double().reshape(B, Tk, KVH, hd),
                self.v.double().reshape(B, Tk, KVH, hd))

    def run(self, E, scale, causal):
        nan_bits = self.o.view(torch.int16)[-1, 0].item()
        _prefill(E, self.dt, self.q, self.kptr, self.vptr, self.o, self.B, self.Tq, self.Tk, self.H, self.KVH, self.hd,
                 self.ldq, self.ldk, self.ldv, self.ldo, scale, causal)
        rows, cols = self.B * self.Tq, self.H * self.hd
        bits = self.o.view(torch.int16)
        outside = torch.ones_like(bits, dtype=torch.bool)
        outside[:rows, :cols] = False
        assert bool((bits[outside] == nan_bits).all()), "s2s_attention wrote outside [B*Tq rows] x [heads*hd columns]"
        out = self.o[:rows, :cols]
        assert bool(torch.isfinite(out).all()), "non-finite output (a NaN cache row past Tk was read)"
        return out.reshape(self.B, self.Tq, self.H, self.hd)


def _visible(Tq, Tk, off):
    i = torch.arange(Tq, device="cuda")[:, None]
    j = torch.arange(Tk, device="cuda")[None, :]
    return (j <= i + off) if off is not None else torch.ones(Tq, Tk, dtype=torch.bool, device="cuda")


def _prefill_check_bound(P, out, scale, off, dt):
    """out [B, Tq, H, hd] against the float64 softmax of the stored operands; returns the worst error / bound."""
    return _bound_ratio(*P.views(), out, scale, off, dt)


def _bound_ratio(q, k, v, out, scale, off, dt):
    """q [B, Tq, H, hd], k / v [B, Tk, KVH, hd] float64; out [B, Tq, H, hd]; off None = non-causal."""
    B, Tq, H, hd = q.shape
    g = H // k.shape[2]
    q = q.permute(0, 2, 1, 3)
    k = k.repeat_interleave(g, 2).permute(0, 2, 1, 3)
    v = v.repeat_interleave(g, 2).permute(0, 2, 1, 3)
    vis = _visible(Tq, k.shape[2], off)
    worst = 0.0
    for h0 in range(0, H, 8):        # heads in groups: the [Tq, Tk] float64 score blocks of 32 heads at 4096 keys add up
        hs = slice(h0, h0 + 8)
        s = (q[:, hs] @ k[:, hs].transpose(-1, -2) * scale).masked_fill(~vis, -math.inf)
        sab = (q[:, hs].abs() @ k[:, hs].abs().transpose(-1, -2) * scale).masked_fill(~vis, 0.0)
        w = torch.softmax(s, -1)
        ref = w @ v[:, hs]
        A = w @ v[:, hs].abs()
        ds = hd * 2.0 ** -24 * sab.amax(-1, keepdim=True)
        tail = SUB[dt] * w.amax(-1, keepdim=True) * (vis.double() @ v[:, hs].abs())
        bound = (U16[dt] + 2 * ds + SMALL) * A + U16[dt] * ref.abs() + tail
        err = (out.permute(0, 2, 1, 3)[:, hs].double() - ref).abs()
        worst = max(worst, (err / bound).max().item())
        del s, sab, w
    return worst


GEOMS = [(4, 4), (8, 4), (32, 8), (2, 1), (4, 2)]   # heads / kv_heads: 1:1, 2:1, 4:1 (Llama-3-8B, Qwen3-4B), micro, qwen3-micro
TQS = [1, 7, 127, 128, 129, 512]
PASTS = [0, 1, 63, 64, 65, 511, 3072, None]       # None: the rest of the 4096-position cache (4096 - Tq)
CAUSAL = [(tq, MAX_POS - tq if p is None else p) for tq in TQS for p in PASTS]


def _geom(i):
    H, KVH = GEOMS[i % len(GEOMS)]
    return H, KVH, (64, 128)[(i // len(GEOMS)) % 2]


def _fill_random(P, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    P.q.copy_(torch.randn(P.q.shape, device="cuda", generator=gen))
    P.k.copy_(torch.randn(P.k.shape, device="cuda", generator=gen))
    P.v.copy_(torch.randn(P.v.shape, device="cuda", generator=gen))


def _prefill_random(E, dt, B, Tq, Tk, H, KVH, hd, causal, seed):
    P = Prefill(dt, B, Tq, Tk, H, KVH, hd)
    _fill_random(P, seed)
    scale = hd ** -0.5
    out = P.run(E, scale, causal)
    r = _prefill_check_bound(P, out, scale, Tk - Tq if causal else None, dt)
    _note("A (prefill)", dt, r)
    assert r <= 1.0, f"error / bound {r:.3f}"


# (Tq, past) over the grid, one geometry per case in turn (every geometry and hd meets every dtype)
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("ci", range(len(CAUSAL)), ids=[f"tq{t}-past{p}" for t, p in CAUSAL])
def test_prefill_causal_random(E, dt, ci):
    Tq, past = CAUSAL[ci]
    H, KVH, hd = _geom(ci + (dt == torch.bfloat16))
    _prefill_random(E, dt, 1, Tq, past + Tq, H, KVH, hd, True, 1000 + ci)


# every geometry and head size at a full-cache chunk and at a chunk straddling tile edges
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("geom", GEOMS, ids=[f"{h}x{k}" for h, k in GEOMS])
@pytest.mark.parametrize("tq,past", [(512, 3584), (129, 65)])
def test_prefill_causal_geometries(E, dt, hd, geom, tq, past):
    _prefill_random(E, dt, 1, tq, past + tq, geom[0], geom[1], hd, True, tq * 31 + past)


# the chunks the LLM handler issues for a 3600-token prompt at max_prefill = 512, appended to one cache slot
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("geom", [(32, 8, 128), (4, 2, 64)], ids=["llama8b", "qwen3-micro"])
def test_prefill_chunked_prompt_3600(E, dt, geom):
    H, KVH, hd = geom
    n, chunk, past = 3600, 512, 0
    gen = torch.Generator(device="cuda").manual_seed(3600)
    kfull = torch.randn(n, KVH * hd, device="cuda", generator=gen).to(dt)
    vfull = torch.randn(n, KVH * hd, device="cuda", generator=gen).to(dt)
    while past < n:
        tq = min(chunk, n - past)
        P = Prefill(dt, 1, tq, past + tq, H, KVH, hd)
        P.q.copy_(torch.randn(P.q.shape, device="cuda", generator=gen))
        P.k.copy_(kfull[: past + tq])
        P.v.copy_(vfull[: past + tq])
        out = P.run(E, hd ** -0.5, True)
        r = _prefill_check_bound(P, out, hd ** -0.5, past, dt)
        _note("A (prefill)", dt, r)
        assert r <= 1.0, (past, tq, r)
        past += tq


# non-causal: Tq != Tk, and B > 1 with Tk % 64 != 0 (a sequence's last key tile runs into the next sequence's rows)
NONCAUSAL = [(1, 1500, 1500, 6, 6, 64), (2, 200, 200, 2, 2, 64), (1, 65, 65, 1, 1, 64), (3, 100, 1500, 6, 6, 64),
             (2, 129, 65, 8, 2, 128), (4, 1, 77, 4, 2, 64), (2, 300, 100, 32, 8, 128), (3, 64, 191, 2, 1, 128)]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", NONCAUSAL, ids=[f"b{c[0]}-tq{c[1]}-tk{c[2]}-h{c[3]}x{c[4]}-hd{c[5]}" for c in NONCAUSAL])
def test_prefill_noncausal_random(E, dt, case):
    B, Tq, Tk, H, KVH, hd = case
    _prefill_random(E, dt, B, Tq, Tk, H, KVH, hd, False, Tq * 7 + Tk)


# engine.attention on a fused [B, T, (H + 2 KVH) hd] qkv buffer: the Whisper encoder / decoder self-attention shapes
WHISPER = [(1, 1500, 6, 6, 64, False), (2, 200, 2, 2, 64, False), (1, 300, 8, 2, 128, True), (1, 64, 4, 4, 64, True),
           (3, 1, 2, 1, 128, True), (1, 65, 1, 1, 64, False)]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("cfg", WHISPER, ids=[f"b{c[0]}-t{c[1]}-h{c[2]}x{c[3]}-hd{c[4]}-{'causal' if c[5] else 'full'}"
                                              for c in WHISPER])
def test_prefill_engine_fused_qkv(E, dt, cfg):
    B, T, H, KVH, hd, causal = cfg
    gen = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B, T, (H + 2 * KVH) * hd, device="cuda", generator=gen).to(dt)
    q, k, v = qkv[:, :, : H * hd], qkv[:, :, H * hd: (H + KVH) * hd], qkv[:, :, (H + KVH) * hd:]
    scale = hd ** -0.5
    o = E.attention(q, k, v, H, KVH, scale, causal)
    r = _bound_ratio(q.double().reshape(B, T, H, hd), k.double().reshape(B, T, KVH, hd), v.double().reshape(B, T, KVH, hd),
                     o.reshape(B, T, H, hd), scale, 0 if causal else None, dt)
    _note("A (prefill)", dt, r)
    assert r <= 1.0, f"error / bound {r:.3f}"


def _count_tables(Tk, KVH, hd, mode):
    """one-hot component index f(j, g) [KVH, Tk]: (j + 7 g) mod hd, or (j // 64 + g) mod hd (one component per key tile)."""
    j = torch.arange(Tk)[None, :]
    g = torch.arange(KVH)[:, None]
    return ((j + 7 * g) if mode == "mod" else (j // 64 + g)) % hd


def _prefill_counting(E, dt, B, Tq, Tk, H, KVH, hd, causal):
    P = Prefill(dt, B, Tq, Tk, H, KVH, hd)
    P.q.zero_()
    P.k.copy_(torch.randn(P.k.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(Tk)))
    off = Tk - Tq if causal else None
    vis = _visible(Tq, Tk, off).cpu()
    n = vis.sum(1)                                             # [Tq]
    g_of_h = torch.arange(H) // (H // KVH)
    for mode in ("mod", "tile"):
        f = _count_tables(Tk, KVH, hd, mode)                    # [KVH, Tk]
        onehot = torch.nn.functional.one_hot(f, hd).to(torch.float64)       # [KVH, Tk, hd]
        P.v.copy_(onehot.permute(1, 0, 2).reshape(Tk, KVH * hd).repeat(B, 1).to(dt).cuda())
        counts = torch.einsum("qk,gkc->qgc", vis.double(), onehot)          # [Tq, KVH, hd]
        want = _exact_counts(counts[:, g_of_h], n[:, None, None], dt)       # [Tq, H, hd]
        out = P.run(E, hd ** -0.5, causal).cpu()
        for b in range(B):
            bad = (out[b].view(torch.int16) != want.view(torch.int16)).nonzero()
            assert bad.numel() == 0, (f"{mode}: {len(bad)} outputs differ from the exact count, first (row, head, comp) "
                                      f"{bad[0].tolist()}: {out[b][tuple(bad[0])].item()} vs {want[tuple(bad[0])].item()}")


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("ci", range(len(CAUSAL)), ids=[f"tq{t}-past{p}" for t, p in CAUSAL])
def test_prefill_causal_counting_exact(E, dt, ci):
    Tq, past = CAUSAL[ci]
    H, KVH, hd = _geom(ci + 2 * (dt == torch.bfloat16))
    _prefill_counting(E, dt, 1, Tq, past + Tq, H, KVH, hd, True)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("case", NONCAUSAL, ids=[f"b{c[0]}-tq{c[1]}-tk{c[2]}-h{c[3]}x{c[4]}-hd{c[5]}" for c in NONCAUSAL])
def test_prefill_noncausal_counting_exact(E, dt, case):
    B, Tq, Tk, H, KVH, hd = case
    _prefill_counting(E, dt, B, Tq, Tk, H, KVH, hd, False)


@pytest.mark.parametrize("where", ["first_masked", "last_visible", "key0"])
@pytest.mark.parametrize("ci", range(len(CAUSAL)), ids=[f"tq{t}-past{p}" for t, p in CAUSAL])
def test_prefill_causal_peaks(E, ci, where):
    Tq, past = CAUSAL[ci]
    Tk, off = past + Tq, past
    dt = DTYPES[ci % 2]
    H, KVH, hd = _geom(ci + 1)
    P = Prefill(dt, 1, Tq, Tk, H, KVH, hd)
    gen = torch.Generator(device="cuda").manual_seed(ci * 3 + len(where))
    codes = torch.stack([_unit_rows(Tk, hd, gen) for _ in range(KVH)], 1)      # [Tk, KVH, hd]
    P.k.copy_(codes.reshape(Tk, KVH * hd).to(dt))
    P.v.copy_(torch.randn(P.v.shape, device="cuda", generator=gen).to(dt))
    i = torch.arange(Tq, device="cuda")
    if where == "first_masked":
        t = torch.clamp(i + off + 1, max=Tk - 1)      # the last query row has no masked key: its peak is its last key
    elif where == "last_visible":
        t = i + off
    else:
        t = torch.zeros_like(i)
    k16 = P.k.double().reshape(Tk, KVH, hd)
    scale = hd ** -0.5
    g_of_h = torch.arange(H, device="cuda") // (H // KVH)
    q = ALPHA / scale * k16[t][:, g_of_h]                                    # [Tq, H, hd]
    P.q.copy_(q.reshape(Tq, H * hd).to(dt))
    out = P.run(E, scale, True)
    r = _prefill_check_bound(P, out, scale, off, dt)
    _note("A (prefill)", dt, r)
    assert r <= 1.0, f"error / bound {r:.3f}"
    if where != "first_masked":   # the design: the visible peak carries the softmax
        qs, ks, _ = P.views()
        s = torch.einsum("qhd,qhd->qh", qs[0], ks[0][t][:, g_of_h]) * scale
        assert bool((s > 0.9 * ALPHA).all())


# ================================================================================================ part B: decode attention
DEC_WARPS = 8
GEOMS_DEC = {"llama8b": (32, 8, 128), "micro": (2, 1, 128), "qwen3-micro": (4, 2, 64)}


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


def _assoc_b(lens):
    return 8 if len(lens) == 16 else 0       # 16 sessions: the 13-16-session tier of the Llama-3-8B decode launch


def _plan_of(geom, lens, grid, assoc_b):
    H = GEOMS_DEC[geom][0]
    return attn_plan((assoc_b or len(lens)) * H, -(-max(lens) // 32), -(-MAX_POS // 64), grid)


def _has_empty_split(plan, lens):
    S = plan & 0x7F
    bps = -(-(-(-max(lens) // 32)) // S)
    return any((S - 1) * bps >= -(-n // 32) for n in lens)


def _plan_name(plan):
    return ("W" if plan & 0x80 else "C") + str(plan & 0x7F)


LENS_B1 = sorted({1, 31, 32, 33, 256, 257, 513, 2047, 3841, 4095, 4096} | {256 * s + 1 for s in range(16)})
LENSETS = [
    [4096, 1, 257], [33, 2047, 513], [257, 300, 3841],
    [1, 4096, 32, 33, 256, 257, 2047, 4095], [97, 5, 64, 96, 31, 1, 200, 150],
    [4096, 1, 31, 32, 33, 256, 257, 513, 2047, 3841, 4095, 1025, 64, 65, 2, 3000], [33] * 15 + [1],
]
DEC_CASES = []
for _g in GEOMS_DEC:
    for _dt in DTYPES:
        DEC_CASES += [(_g, _dt, 132, [n]) for n in LENS_B1]
        DEC_CASES += [(_g, _dt, grid, [n]) for grid in (66, 37) for n in (1, 257, 2047, 4096)]
        DEC_CASES += [(_g, _dt, grid, ls) for grid in (132, 66, 37) for ls in LENSETS]


def _dec_id(c):
    g, dt, grid, lens = c
    ls = f"len{lens[0]}" if len(lens) == 1 else f"b{len(lens)}-" + "-".join(map(str, lens[:4]))
    return f"{g}-{str(dt)[6:]}-g{grid}-{ls}"


class Decode:
    """Operands of one s2s_decode_attention call: a cache of B + 1 slots [slots, 2, MAX_POS, KVH hd] whose rows at and
    past each session's len are NaN, sessions on slots in reverse order (slot B stays unused)."""

    def __init__(self, geom, dt, grid, lens):
        self.H, self.KVH, self.hd = GEOMS_DEC[geom]
        self.geom, self.dt, self.grid, self.lens = geom, dt, grid, list(lens)
        self.B = len(lens)
        self.assoc_b = _assoc_b(lens)
        self.slots = [self.B - 1 - b for b in range(self.B)]
        self.kv = torch.full((self.B + 1, 2, MAX_POS, self.KVH * self.hd), float("nan"), dtype=dt, device="cuda")

    def keys(self, b):    # [2, len, KVH, hd] views of session b's K and V rows
        return self.kv[self.slots[b], :, : self.lens[b]].view(2, self.lens[b], self.KVH, self.hd)

    def run(self, E, q):
        out, plan = E.decode_attention(q, self.kv, self.slots, self.lens, self.H, self.KVH, grid=self.grid,
                                       assoc_b=self.assoc_b)
        assert plan == _plan_of(self.geom, self.lens, self.grid, self.assoc_b)
        return out, plan

    def check_bound(self, q, out):
        g = self.H // self.KVH
        worst = 0.0
        for b in range(self.B):
            kb, vb = self.keys(b).double()                       # [len, KVH, hd]
            kb, vb = kb.repeat_interleave(g, 1), vb.repeat_interleave(g, 1)
            qb = q[b].double()                                   # [H, hd]
            s = torch.einsum("hc,jhc->hj", qb, kb)
            sab = torch.einsum("hc,jhc->hj", qb.abs(), kb.abs())
            w = torch.softmax(s, -1)
            ref = torch.einsum("hj,jhc->hc", w, vb)
            A = torch.einsum("hj,jhc->hc", w, vb.abs())
            ds = self.hd * 2.0 ** -24 * sab.amax(-1, keepdim=True)
            bound = (2 * ds + SMALL) * A + U16[self.dt] * ref.abs()
            worst = max(worst, ((out[b].double() - ref).abs() / bound).max().item())
        return worst


@pytest.mark.parametrize("case", DEC_CASES, ids=[_dec_id(c) for c in DEC_CASES])
def test_decode_attention_random_repeatable(E, case):
    D = Decode(*case)
    gen = torch.Generator(device="cuda").manual_seed(sum(D.lens) + D.grid)
    for b in range(D.B):
        D.kv[D.slots[b], :, : D.lens[b]] = torch.randn(2, D.lens[b], D.KVH * D.hd, device="cuda", generator=gen).to(D.dt)
    q = torch.randn(D.B, D.H, D.hd, device="cuda", generator=gen) * D.hd ** -0.5
    out, _ = D.run(E, q)
    out2, _ = D.run(E, q)
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)), "two runs differ"
    r = D.check_bound(q, out)
    _note("B (decode)", D.dt, r)
    assert r <= 1.0, f"error / bound {r:.3f}"


@pytest.mark.parametrize("case", DEC_CASES, ids=[_dec_id(c) for c in DEC_CASES])
def test_decode_attention_counting_exact(E, case):
    D = Decode(*case)
    gen = torch.Generator(device="cuda").manual_seed(len(D.lens))
    g_of_h = torch.arange(D.H) // (D.H // D.KVH)
    q = torch.zeros(D.B, D.H, D.hd, device="cuda")
    for mode in ("mod", "block"):
        want = []
        for b, n in enumerate(D.lens):
            j = torch.arange(n)[None, :]
            gg = torch.arange(D.KVH)[:, None]
            f = ((j + 7 * gg) if mode == "mod" else (j // 32 + gg)) % D.hd                  # [KVH, n]
            onehot = torch.nn.functional.one_hot(f, D.hd)                                   # [KVH, n, hd]
            D.kv[D.slots[b], 0, :n] = torch.randn(n, D.KVH * D.hd, device="cuda", generator=gen).to(D.dt)
            D.kv[D.slots[b], 1, :n] = onehot.permute(1, 0, 2).reshape(n, D.KVH * D.hd).to(D.dt).cuda()
            want.append(_exact_counts(onehot.sum(1)[g_of_h], torch.tensor([n]), D.dt))     # [H, hd]
        want = torch.stack(want)
        for rep in range(2):
            out = D.run(E, q)[0].cpu()
            bad = (out.view(torch.int16) != want.view(torch.int16)).nonzero()
            assert bad.numel() == 0, (f"{mode} run {rep}: {len(bad)} outputs differ from the exact count, first (session, "
                                      f"head, comp) {bad[0].tolist()}: {out[tuple(bad[0])].item()} vs "
                                      f"{want[tuple(bad[0])].item()}")


def _peak_targets(n, plan, n_max):
    """key 0, key n - 1, the block edges 32k - 1 / 32k and the split edges s * bps * 32 (and the key before) below n."""
    S = plan & 0x7F
    bps = -(-(-(-n_max // 32)) // S)
    t = {0, n - 1}
    for k in (1, n // 64, n // 32):
        t |= {32 * k - 1, 32 * k}
    for s in range(1, S):
        t |= {s * bps * 32 - 1, s * bps * 32}
    return sorted(x for x in t if 0 <= x < n)


@pytest.mark.parametrize("case", DEC_CASES, ids=[_dec_id(c) for c in DEC_CASES])
def test_decode_attention_peaks(E, case):
    D = Decode(*case)
    gen = torch.Generator(device="cuda").manual_seed(7 * len(D.lens) + D.grid)
    for b, n in enumerate(D.lens):
        codes = torch.stack([_unit_rows(n, D.hd, gen) for _ in range(D.KVH)], 1)        # [n, KVH, hd]
        D.kv[D.slots[b], 0, :n] = codes.reshape(n, D.KVH * D.hd).to(D.dt)
        D.kv[D.slots[b], 1, :n] = torch.randn(n, D.KVH * D.hd, device="cuda", generator=gen).to(D.dt)
    plan = _plan_of(D.geom, D.lens, D.grid, D.assoc_b)
    targets = [_peak_targets(n, plan, max(D.lens)) for n in D.lens]
    g_of_h = [h // (D.H // D.KVH) for h in range(D.H)]
    for rnd in range(max(-(-len(t) // D.H) for t in targets)):   # every target of every session, H per launch
        q = torch.empty(D.B, D.H, D.hd, device="cuda")
        for b in range(D.B):
            k16 = D.keys(b)[0].float()
            for h in range(D.H):
                t = targets[b][(rnd * D.H + h) % len(targets[b])]
                q[b, h] = ALPHA * k16[t, g_of_h[h]]
        out, _ = D.run(E, q)
        r = D.check_bound(q, out)
        _note("B (decode)", D.dt, r)
        assert r <= 1.0, f"round {rnd}: error / bound {r:.3f}"


def test_decode_attention_plan_coverage(E):
    """The cases above reach every plan the issue table names: CTA-level C1 ... C16, warp-level W1 and W >= 9, and
    sessions with empty splits; one launch per plan confirms the library chooses it."""
    seen, empty = {}, False
    for g, dt, grid, lens in DEC_CASES:
        p = _plan_of(g, lens, grid, _assoc_b(lens))
        seen.setdefault(p, (g, dt, grid, lens))
        empty |= _has_empty_split(p, lens)
    names = {_plan_name(p) for p in seen}
    need = {f"C{s}" for s in range(1, 17)} | {"W1"}
    assert need <= names, sorted(need - names)
    assert any(p & 0x80 and (p & 0x7F) >= 9 for p in seen), sorted(names)
    assert empty
    print("\ndecode attention plans covered:", " ".join(sorted(names, key=lambda s: (s[0], int(s[1:])))))
    for p, (g, dt, grid, lens) in seen.items():
        D = Decode(g, dt, grid, lens)
        q = torch.zeros(D.B, D.H, D.hd, device="cuda")
        for b, n in enumerate(lens):
            D.kv[D.slots[b], :, :n] = 0
        assert D.run(E, q)[1] == p


def test_decode_attention_rejects_bad_arguments(E):
    from speech_to_speech_b200._lib import S2SError
    kv = torch.zeros(2, 2, 64, 128, dtype=torch.float16, device="cuda")
    q = torch.zeros(1, 2, 128, device="cuda")
    for lens in ([0], [65]):
        with pytest.raises(S2SError, match="len"):
            E.decode_attention(q, kv, [0], lens, 2, 1)
    out, plan = E.decode_attention(q, kv, [1], [64], 2, 1, grid=37)
    assert plan == attn_plan(2, 2, 1, 37)
    assert bool((out == 0).all())
