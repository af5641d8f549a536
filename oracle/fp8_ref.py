"""numpy reference of the engine's FP8 E4M3 weight-only storage (speech_to_speech_b200/csrc/weight_tiles.cu).

Per row n of a matrix W[N, K] the integer exponent e_n is the smallest with max_k |W[n, k]| * 2^-e_n <= 448 (never below
MIN_EXP; 0 for an all-zero row); the code is Q[n, k] = e4m3(W[n, k] * 2^-e_n), round-to-nearest-even, saturating at +-448,
and dq(Q)[n, k] = Q[n, k] * 2^e_n.  E4M3 ("fn": no infinities, 0x7f / 0xff = NaN) has 3 mantissa bits, exponents 2^-6..2^8 and
subnormals down to 2^-9, so dq(Q) is exactly representable in bfloat16: an FP8 engine computes what the bf16 engine computes
from the weights dq_state_dict() returns.
"""
from __future__ import annotations

import numpy as np

E4M3_MAX = 448.0
MIN_EXP = -100   # keeps 2^-9 * 2^e_n a normal bfloat16 number


def _code_values() -> np.ndarray:
    """values of the non-negative finite codes 0x00..0x7e, ascending"""
    c = np.arange(0x7F)
    e, m = c >> 3, (c & 7).astype(np.float64)
    return np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * 2.0 ** (e - 7.0))


CODE_VALUES = _code_values()


def e4m3_encode(x: np.ndarray) -> np.ndarray:
    """float -> E4M3 codes (uint8): round to nearest, ties to even, magnitudes above 448 saturate to 448"""
    x = np.asarray(x, dtype=np.float64)
    a = np.minimum(np.abs(x), E4M3_MAX)
    _, ex = np.frexp(a)                                    # a = m * 2^ex, m in [0.5, 1): the leading bit is 2^(ex - 1)
    qe = np.maximum(ex - 1, -6) - 3                        # exponent of the rounding step (2^-9 for subnormals)
    q = np.rint(np.ldexp(a, -qe)).astype(np.int64)         # np.rint rounds half to even; q <= 16
    # q = 8 + mantissa (16: the next binade's first value) under the exponent field qe + 3 + 7; with the subnormal step
    # (qe = -9) the same expression is q itself, the subnormal code.  Zero has no leading bit (frexp gives ex = 0).
    code = np.where(q == 0, 0, (qe + 10) * 8 + q - 8)
    return (code | np.where(np.signbit(x), 0x80, 0)).astype(np.uint8)


def e4m3_decode(codes: np.ndarray) -> np.ndarray:
    codes = np.asarray(codes, dtype=np.uint8)
    v = CODE_VALUES[np.minimum(codes & 0x7F, 0x7E)]
    return np.where(codes & 0x80, -v, v).astype(np.float32)


def row_exponents(w: np.ndarray) -> np.ndarray:
    """e_n per row: amax = m * 2^x with m in [0.5, 1) and 448 = 0.875 * 2^9, so e_n = x - 9 if m <= 0.875 else x - 8"""
    amax = np.abs(np.asarray(w, dtype=np.float32)).max(axis=1)
    m, x = np.frexp(amax)
    e = np.where(m <= 0.875, x - 9, x - 8)
    return np.where(amax > 0, np.maximum(e, MIN_EXP), 0).astype(np.int32)


def quantize_rows(w: np.ndarray):
    """W[N, K] -> (codes uint8 [N, K], exponents int32 [N])"""
    e = row_exponents(w)
    return e4m3_encode(np.ldexp(np.asarray(w, dtype=np.float64), -e[:, None])), e


def dequantize(codes: np.ndarray, exponents: np.ndarray) -> np.ndarray:
    return np.ldexp(e4m3_decode(codes), np.asarray(exponents)[:, None]).astype(np.float32)


def dq(w: np.ndarray, block: int = 2048) -> np.ndarray:
    """dequantize(quantize_rows(W)), a block of rows at a time (the float64 temporaries of a 128256 x 4096 head are large)"""
    w = np.asarray(w, dtype=np.float32)
    return np.concatenate([dequantize(*quantize_rows(w[i:i + block])) for i in range(0, w.shape[0], block)], axis=0)


# The matrices the decode launch streams.  The engine quantises them as it stores them: q / k rows permuted so that
# rotate_half partners are adjacent, gate and up rows interleaved, q / k / v stacked.  The scale is per stored ROW and every
# one of these rearrangements only permutes or stacks whole rows, so quantising each checkpoint tensor row by row gives the
# same values.  The embedding table is a lookup, not a stream, and stays as bound -- also when the checkpoint ties lm_head to
# it (the engine quantises its own copy for lm_head): pass tied=True to get the lm_head the engine then uses.
_LAYER_MATRICES = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
                   "mlp.down_proj")


def dq_state_dict(weights, geom, tied: bool = False) -> dict:
    out = dict(weights)
    for i in range(geom.layers):
        for m in _LAYER_MATRICES:
            name = f"model.layers.{i}.{m}.weight"
            out[name] = dq(weights[name])
    if "lm_head.weight" in weights:
        out["lm_head.weight"] = dq(weights["lm_head.weight"])
    elif tied:
        out["lm_head.weight"] = dq(weights["model.embed_tokens.weight"])
    return out
