"""CPU: the numpy reference of the FP8 E4M3 weight storage (oracle/fp8_ref.py) against torch.float8_e4m3fn, and the two
properties the GPU tests rest on: dq(q(W)) is a bfloat16 matrix, and quantising it again changes none of its values."""
import numpy as np
import torch

from oracle import fp8_ref as F, weights as W


def _torch_codes(x):
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def test_every_code_decodes_like_torch():
    codes = np.array([c for c in range(256) if c & 0x7F != 0x7F], dtype=np.uint8)   # 0x7f / 0xff are NaN
    ref = torch.from_numpy(codes).view(torch.float8_e4m3fn).to(torch.float32).numpy()
    assert np.array_equal(F.e4m3_decode(codes), ref)
    assert np.array_equal(F.e4m3_encode(ref), codes)     # -0 keeps its sign bit
    assert F.CODE_VALUES[-1] == 448.0 and F.CODE_VALUES[1] == 2.0 ** -9


def test_rounding_equals_torch_on_codes_ties_and_subnormals():
    v = F.CODE_VALUES
    mid = (v[:-1] + v[1:]) / 2                                # every tie, subnormal ones included
    grid = np.concatenate([v, mid, np.nextafter(mid.astype(np.float32), 0), np.nextafter(mid.astype(np.float32), 1e9),
                           [2.0 ** -10, 2.0 ** -11, 1e-30, 0.0]])
    grid = np.concatenate([grid, -grid]).astype(np.float32)
    assert np.array_equal(F.e4m3_encode(grid), _torch_codes(grid))
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(200000) * np.exp2(rng.integers(-12, 9, 200000))).astype(np.float32)
    x = np.clip(x, -448, 448)
    assert np.array_equal(F.e4m3_encode(x), _torch_codes(x))


def test_saturation_is_finite():
    x = np.array([448.0, 449.0, 463.9, 464.0, 480.0, 1e6, 3e38, -448.0, -464.0, -1e6], dtype=np.float32)
    assert np.array_equal(F.e4m3_encode(x), _torch_codes(np.clip(x, -448, 448)))
    assert np.abs(F.e4m3_decode(F.e4m3_encode(x))).max() == 448.0


def test_row_exponent_is_the_smallest_that_fits():
    rng = np.random.default_rng(1)
    w = W.round_bf16((rng.standard_normal((300, 64)) * np.exp2(rng.integers(-20, 12, (300, 1)))).astype(np.float32))
    w[7] = 0.0
    w[8, :] = 0.0; w[8, 3] = 448.0                            # fits with e = 0 exactly
    w[9, :] = 0.0; w[9, 3] = 450.0                            # bf16 neighbour above 448: needs e = 1
    w = W.round_bf16(w)
    codes, e = F.quantize_rows(w)
    amax = np.abs(w).max(axis=1).astype(np.float64)
    assert e[7] == 0 and not codes[7].any()
    assert e[8] == 0 and e[9] == 1
    nz = amax > 0
    assert (amax[nz] * np.exp2(-e[nz].astype(np.float64)) <= 448).all()
    assert (amax[nz] * np.exp2(-(e[nz] - 1).astype(np.float64)) > 448).all()
    assert np.abs(F.e4m3_decode(codes)).max() <= 448


def test_dequantised_weights_are_bf16_and_requantise_to_themselves():
    g = W.LLAMA_GEOMETRIES["micro"]
    w = W.make_llama_weights(g, 0)
    d = F.dq_state_dict(w, g)
    changed = 0
    for name, a in w.items():
        b = d[name]
        if "proj" in name or name == "lm_head.weight":
            assert np.array_equal(W.round_bf16(b), b), name                   # exact in bfloat16
            # quantising again changes no value.  (A row whose maximum rounds down to 224 * 2^e gets the exponent e - 1 and
            # codes one exponent step up the second time: the same numbers.)
            c0, e0 = F.quantize_rows(a)
            c1, e1 = F.quantize_rows(b)
            assert np.array_equal(F.dequantize(c1, e1), b), name
            assert np.isin(e0 - e1, (0, 1)).all() and np.array_equal(c0[e0 == e1], c1[e0 == e1]), name
            assert np.abs(b - a).max() <= np.abs(a).max() / 16                # half a 3-bit mantissa step
            changed += int(not np.array_equal(a, b))
        else:
            assert b is a, name                                               # embedding and norm weights stay as bound
    assert changed == 7 * g.layers + 1
    assert np.array_equal(F.dq_state_dict(d, g)["lm_head.weight"], d["lm_head.weight"])


def test_row_scale_is_invariant_to_the_engine_row_order():
    """the engine permutes q/k rows and interleaves gate/up rows before it quantises: per-row scales do not care"""
    rng = np.random.default_rng(2)
    w = W.round_bf16(rng.standard_normal((64, 96)).astype(np.float32))
    perm = rng.permutation(64)
    assert np.array_equal(F.dq(w)[perm], F.dq(w[perm]))


def test_tied_head_is_quantised_from_the_embedding():
    g = W.LLAMA_GEOMETRIES["micro"]
    w = W.make_llama_weights(g, 0)
    del w["lm_head.weight"]
    d = F.dq_state_dict(w, g, tied=True)
    assert np.array_equal(d["lm_head.weight"], F.dq(w["model.embed_tokens.weight"]))
    assert d["model.embed_tokens.weight"] is w["model.embed_tokens.weight"]
    assert "lm_head.weight" not in F.dq_state_dict(w, g)
