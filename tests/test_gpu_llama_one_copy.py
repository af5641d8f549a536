"""GPU: the Llama family stores its projections and lm_head once, in the tiled layout the decode kernel streams, and the
prefill GEMMs read that layout (16-bit tiles, or FP8 codes expanded to dq(Q) in shared memory).

  * the tiled GEMM equals the row-major GEMM bit for bit (bf16), and the FP8 one equals the row-major GEMM over dq(Q);
  * tile_weights lays out and quantises exactly as include/s2s_b200.h and oracle/fp8_ref.py state;
  * device_bytes(): the weights are the embedding, the norms and ONE tiled copy of every matrix -- no row-major projections;
  * 2-layer slices of Qwen3-14B and Qwen3-32B: prefill + decode against the numpy oracle, FP8 against bf16 on dq(Q);
  * the weight format is fixed by the first bind; a tied lm_head equals an lm_head bound to a copy of the embedding."""
import numpy as np
import pytest
import torch

from oracle import fp8_ref as F, llama_ref as R, weights as W

pytestmark = pytest.mark.gpu
TOL = 0.2                                            # bfloat16 logits, tests/test_gpu_llama.py
FP8 = "float8_e4m3"
# 2-layer slices of Qwen/Qwen3-14B and Qwen/Qwen3-32B (config.json of each)
SLICES = {
    "qwen3-14b-2l": W.LlamaGeometry(5120, 2, 40, 8, 128, 17408, 151936, rope_theta=1000000.0, rms_eps=1e-6, qk_norm=True),
    "qwen3-32b-2l": W.LlamaGeometry(5120, 2, 64, 8, 128, 25600, 151936, rope_theta=1000000.0, rms_eps=1e-6, qk_norm=True),
}


@pytest.fixture(scope="module")
def E():
    from speech_to_speech_b200 import engine
    return engine


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy()


def untile(t, N, K, fp8=False):
    """the tiled layout -> row-major [N, K]: 16-bit values, or for FP8 the dequantised dq(Q) = Q * 2^e_n in bfloat16"""
    esz = 1 if fp8 else 2
    blocks = t[: N * K * esz].view(torch.float8_e4m3fn if fp8 else torch.bfloat16)
    rows = blocks.view(N // 8, K // 32, 8, 4, 8).permute(0, 2, 1, 3, 4).reshape(N, K)
    if not fp8:
        return rows
    scale = t[N * K: N * K + 4 * N].view(torch.float32)
    return (rows.float() * scale[:, None]).to(torch.bfloat16)


# ---- 1. the GEMM ------------------------------------------------------------------------------------------------
# (M, N, K, bias): every M of {1, 17, 64, 130, 512}, every K of {256, 4096, 14336, 25600}, N = 151936, and N on both sides
# of the 128-wide tile rule (tiles128 = N/128 * ceil(M/128) >= 132 SMs); K = 96 ends on half a 64-k block.
SHAPES = [
    (1, 4096, 4096, False),       # 64-wide
    (17, 6144, 256, True),        # 64-wide
    (64, 28672, 4096, True),      # 128-wide: 224 tiles
    (130, 5120, 25600, False),    # 64-wide: 80 tiles
    (512, 5120, 14336, True),     # 128-wide: 160 tiles
    (130, 8448, 4096, False),     # 128-wide: 132 tiles exactly
    (64, 151936, 4096, False),    # 128-wide, the Qwen3 lm_head
    (17, 16896, 25600, True),     # 128-wide: 132 tiles, long K
    (64, 128, 96, True),
]


@pytest.mark.parametrize("M,N,K,bias", SHAPES)
def test_tiled_gemm_equals_row_major_gemm_bitwise(E, M, N, K, bias):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    a = (torch.randn((M, K), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn((N, K), device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    b = torch.randn((N,), device="cuda", generator=g) if bias else None
    wt = E.tile_weights(w)
    assert torch.equal(untile(wt, N, K), w)
    for out in (torch.float32, torch.bfloat16):
        want = E.gemm(a, w, b, out_dtype=out)
        got = E.gemm_tiled(a, wt, N, bias=b, out_dtype=out)
        assert np.array_equal(_bits(got), _bits(want)), out
    del wt
    q = E.tile_weights(w, FP8)
    wd = untile(q, N, K, fp8=True)
    want = E.gemm(a, wd, b, out_dtype=torch.float32)
    got = E.gemm_tiled(a, q, N, FP8, bias=b, out_dtype=torch.float32)
    assert np.array_equal(_bits(got), _bits(want))
    torch.cuda.synchronize()


def test_tile_weights_fp8_matches_the_oracle(E):
    """codes and power-of-two row scales of tile_weights(w, FP8) = oracle/fp8_ref.py, including an all-zero row, a row at
    the exponent floor and rows with saturating and subnormal codes"""
    rng = np.random.default_rng(5)
    N, K = 256, 1024
    w = (rng.standard_normal((N, K)) * np.exp(rng.uniform(-8, 8, (N, 1)))).astype(np.float32)
    w[3] = 0.0
    w[4] *= 2.0 ** -120
    w = W.round_bf16(w)
    q = E.tile_weights(torch.from_numpy(w).cuda().to(torch.bfloat16), FP8)
    got = untile(q, N, K, fp8=True).float().cpu().numpy()
    assert np.array_equal(got.view(np.uint32), F.dq(w).view(np.uint32))
    assert E.tile_weights(torch.zeros((8, 64), dtype=torch.float16, device="cuda")).numel() == 8 * 64 * 2


# ---- 2. footprint ------------------------------------------------------------------------------------------------
def _tiled(N, K, fp8):
    return N * K + 4 * N if fp8 else 2 * N * K


def _weight_formula(g, fp8, n_tables=1):
    d, hd, f = g["d_model"], g["head_dim"], g["ffn"]
    qd, kvd = g["heads"] * hd, g["kv_heads"] * hd
    per_layer = (_tiled(qd + 2 * kvd, d, fp8) + _tiled(d, qd, fp8) + _tiled(2 * f, d, fp8) + _tiled(d, f, fp8)
                 + 2 * 4 * d + (2 * 4 * hd if g.get("qk_norm") else 0))
    head = _tiled(g["vocab"], d, fp8) if fp8 else n_tables * _tiled(g["vocab"], d, False)
    return n_tables * g["vocab"] * d * 2 + 4 * d + g["layers"] * per_layer + head


FOOTPRINTS = [("micro", None), ("micro", FP8), ("qwen3-micro", None), ("qwen3-micro", FP8), ("llama-3-8b-2l", None),
              ("llama-3-8b-2l", FP8), ("tied", None), ("tied", FP8), ("predictor", None)]


@pytest.mark.parametrize("name,fmt", FOOTPRINTS)
def test_device_bytes_hold_one_tiled_copy(E, name, fmt):
    g = W.LLAMA_GEOMETRIES["micro" if name == "tied" else "qwen3-micro" if name == "predictor" else name].to_dict()
    n_tables = 4 if name == "predictor" else 1
    if n_tables > 1:
        g["n_tables"] = n_tables
    sessions, positions = 2, 128
    eng = E.LlamaEngine(g, max_sessions=sessions, max_positions=positions, max_prefill=64, weight_dtype=fmt)
    try:
        if name == "tied":
            w = W.make_llama_weights(W.LLAMA_GEOMETRIES["micro"], 0)
            del w["lm_head.weight"]
            eng.load_state_dict(w)
        else:
            eng.init_random(0)
        weights, total = eng.device_bytes()
        assert weights == _weight_formula(g, fmt == FP8, n_tables)
        kv = sessions * g["layers"] * 2 * positions * g["kv_heads"] * g["head_dim"] * 2
        assert total - weights > kv
        if fmt == FP8:   # the workspace does not depend on the weight format
            ref = E.LlamaEngine(g, max_sessions=sessions, max_positions=positions, max_prefill=64)
            ref.init_random(0)
            rw, rt = ref.device_bytes()
            ref.close()
            assert rt - rw == total - weights
    finally:
        eng.close()


# ---- 3. Qwen3-14B / 32B slices -----------------------------------------------------------------------------------
def _slice_weights(g, seed):
    """random bfloat16 weights with make_llama_weights' scales, drawn with torch (fast at these sizes)"""
    gen = torch.Generator().manual_seed(seed)
    d, f, hd = g.d_model, g.ffn, g.head_dim
    qd, kvd = g.heads * hd, g.kv_heads * hd

    def nrm(shape, std):
        return (torch.randn(shape, generator=gen) * std).to(torch.bfloat16).float().numpy()

    w = {"model.embed_tokens.weight": nrm((g.vocab, d), 0.02), "lm_head.weight": nrm((g.vocab, d), 0.02),
         "model.norm.weight": 1.0 + nrm((d,), 0.1)}
    for i in range(g.layers):
        p = f"model.layers.{i}."
        w[p + "self_attn.q_proj.weight"] = nrm((qd, d), 2.0 / d ** 0.5)
        w[p + "self_attn.k_proj.weight"] = nrm((kvd, d), 2.0 / d ** 0.5)
        w[p + "self_attn.v_proj.weight"] = nrm((kvd, d), 0.8 / d ** 0.5)
        w[p + "self_attn.o_proj.weight"] = nrm((d, qd), 1.0 / d ** 0.5)
        w[p + "self_attn.q_norm.weight"] = 1.0 + nrm((hd,), 0.1)
        w[p + "self_attn.k_norm.weight"] = 1.0 + nrm((hd,), 0.1)
        w[p + "mlp.gate_proj.weight"] = nrm((f, d), 1.0 / d ** 0.5)
        w[p + "mlp.up_proj.weight"] = nrm((f, d), 1.0 / d ** 0.5)
        w[p + "mlp.down_proj.weight"] = nrm((d, f), 0.7 / f ** 0.5)
        w[p + "input_layernorm.weight"] = 1.0 + nrm((d,), 0.1)
        w[p + "post_attention_layernorm.weight"] = 1.0 + nrm((d,), 0.1)
    return w


def _dq_gpu(E, w):
    """W -> dq(q(W)) in place for every streamed matrix, through tile_weights (whose quantiser the oracle test pins)"""
    for n in [n for n in w if n.endswith("proj.weight")] + ["lm_head.weight"]:
        t = torch.from_numpy(w[n]).cuda().to(torch.bfloat16)
        w[n] = untile(E.tile_weights(t, FP8), *t.shape, fp8=True).float().cpu().numpy()


def _prefill_decode(eng, prompt, first, forced):
    eng.reset(0)
    nxt, logits = eng.prefill(0, prompt, return_logits=True)
    ids, _, lg = eng.decode([0], torch.tensor([first], dtype=torch.int32, device="cuda"), forced.shape[1],
                            forced=torch.from_numpy(forced).cuda(), return_logits=True)
    return int(nxt[0]), logits.cpu().numpy(), ids.cpu().numpy(), lg[:, 0].cpu().numpy()


@pytest.mark.parametrize("name", list(SLICES))
def test_qwen3_large_slices_prefill_and_decode(E, name):
    g = SLICES[name]
    w = _slice_weights(g, 11)
    prompt = np.random.default_rng(2).integers(0, g.vocab, 24).tolist()
    ref_ids, ref_lg = R.greedy_generate(w, g, np.array(prompt), 3, return_logits=True)
    forced = np.array([ref_ids[1:]], dtype=np.int32)
    kw = dict(max_sessions=1, max_positions=64, max_prefill=32)
    eng = E.LlamaEngine(g.to_dict(), **kw)
    try:
        eng.load_state_dict(w)
        _, logits, _, lg = _prefill_decode(eng, prompt, ref_ids[0], forced)
        assert np.abs(logits[-1] - ref_lg[0]).max() < TOL
        assert np.abs(lg - ref_lg[1:]).max() < TOL
        full = eng.max_decode_batch()
    finally:
        eng.close()
    a = E.LlamaEngine(g.to_dict(), weight_dtype=FP8, **kw)
    b = E.LlamaEngine(g.to_dict(), **kw)
    try:
        a.load_state_dict(w)
        _dq_gpu(E, w)
        b.load_state_dict(w)
        ra, rb = _prefill_decode(a, prompt, ref_ids[0], forced), _prefill_decode(b, prompt, ref_ids[0], forced)
        assert ra[0] == rb[0] and np.array_equal(ra[2], rb[2])
        assert np.array_equal(ra[1].view(np.uint32), rb[1].view(np.uint32)), "prefill logits"
        assert np.array_equal(ra[3].view(np.uint32), rb[3].view(np.uint32)), "decode logits"
        fp8_full = a.max_decode_batch()
    finally:
        a.close()
        b.close()
    lane = E.LlamaEngine(g.to_dict(), weight_dtype=FP8, lane=1, lanes=2, **kw)
    try:
        lane.init_random(0)
        half = lane.max_decode_batch()
    finally:
        lane.close()
    print(f"{name}: max_decode_batch full grid bf16 {full}, FP8 {fp8_full}; FP8 on a 66-CTA lane {half}")
    assert min(full, fp8_full, half) >= 1


# ---- 4. interface and tied head ----------------------------------------------------------------------------------
def test_weight_format_is_fixed_by_the_first_bind(E):
    from speech_to_speech_b200 import _lib
    g = W.LLAMA_GEOMETRIES["micro"]
    w = W.make_llama_weights(g, 0)
    eng = E.LlamaEngine(g.to_dict(), max_sessions=1, max_positions=64, max_prefill=16)
    try:
        assert eng.lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_FP8_E4M3) == 0
        assert eng.lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_BF16) == 0
        E._bind_all(eng.lib.s2s_llama_bind_tensor, eng.handle, {"model.norm.weight": w["model.norm.weight"]}, "llama")
        assert eng.lib.s2s_llama_set_weight_format(eng.handle, _lib.S2S_FP8_E4M3) == -1     # S2S_ERR_INVALID
        assert eng.weight_format() == _lib.S2S_BF16
        eng.load_state_dict(w)
        assert len(eng.generate([1, 2, 3], 4)) == 4
    finally:
        eng.close()


@pytest.mark.parametrize("fmt", [None, FP8], ids=["bf16", "fp8"])
def test_tied_head_equals_head_bound_to_the_embedding(E, fmt):
    g = W.LLAMA_GEOMETRIES["qwen3-micro"]
    w = W.make_llama_weights(g, 4)
    tied = {k: v for k, v in w.items() if k != "lm_head.weight"}
    untied = {**tied, "lm_head.weight": w["model.embed_tokens.weight"].copy()}
    prompt = np.random.default_rng(6).integers(0, g.vocab, 19).tolist()
    outs = []
    for weights in (tied, untied):
        eng = E.LlamaEngine(g.to_dict(), max_sessions=1, max_positions=64, max_prefill=32, weight_dtype=fmt)
        try:
            eng.load_state_dict(weights)
            eng.reset(0)
            nxt, logits = eng.prefill(0, prompt, return_logits=True)
            ids, _, lg = eng.decode([0], nxt, 8, return_logits=True)
            outs.append((logits.cpu().numpy(), ids.cpu().numpy(), lg.cpu().numpy()))
        finally:
            eng.close()
    for x, y in zip(*outs):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
