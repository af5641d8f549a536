"""CPU: the load-time weight layouts of csrc/weight_arena.cuh (RoPE row permutation, gate/up interleave, [N,K] -> [K][N]
transpose whole and as a column block of a shared matrix, the codec's convolution and transposed-convolution tap orders,
Whisper's conv reorder and q-scale fold) and the 16-bit conversions, byte for byte against numpy statements of the same
layouts.  A small host program built with nvcc runs the arena's layout step and places its bytes where bind_tensor uploads
them (no GPU needed); init_random's per-tensor seed is checked against FNV-1a computed here."""
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

F32, F16, BF16 = 0, 1, 2  # S2S_F32 / S2S_F16 / S2S_BF16
PLAIN, ROPE_PERM, INTERLEAVE, LINEAR, CONV, TCONV, CONV_ROWS = range(7)  # enum WeightLayout
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = tmp_path_factory.mktemp("weight_layouts") / "weight_layout_check"
    src = os.path.join(ROOT, "tests", "dev", "weight_layout_check.cu")
    build = subprocess.run([NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(out), src],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stderr[-2000:]
    return str(out)


def bf16_bits(x):
    """float32 -> bf16 bits, round to nearest even, every NaN -> 0x7fc0"""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[np.isnan(x)] = 0x7FC0
    return r


def source(rng, n, dtype, specials):
    """n seeded source elements as the raw array bind_tensor receives, and their float32 values"""
    if dtype == F32:
        a = rng.standard_normal(n).astype(np.float32)
        if specials:
            u = a.view(np.uint32)
            u[::5] = (u[::5] & 0xFFFF0000) | 0x8000              # exact bf16 ties
            u[0], u[5] = 0x3F808000, 0x3F818000                    # a tie that rounds down (even) and one that rounds up
            u[1], u[2], u[3] = 0x7FC00123, 0xFFC00000, 0x7F800000  # NaNs with payload / sign, +inf
        return a, a
    if dtype == F16:
        a = rng.standard_normal(n).astype(np.float16)
        return a, a.astype(np.float32)
    u = (rng.standard_normal(n).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    if specials:
        u[1] = 0x7FC1
    return u, (u.astype(np.uint32) << 16).view(np.float32)


def expected(layout, v, d0, d1, d2, p, ld):
    """numpy statement of each layout: destination shape (elements), the part of it the tensor fills, and its values"""
    ALL = slice(None)
    if layout == ROPE_PERM:   # rows (j, j + hd/2) of every head of p rows -> rows 2j, 2j + 1
        return (d0, d1), ALL, v.reshape(d0 // p, 2, p // 2, d1).transpose(0, 2, 1, 3).reshape(d0, d1)
    if layout == INTERLEAVE:  # gate (p = 0) / up (p = 1) rows interleaved in a [2 d0][d1] block
        return (2 * d0, d1), slice(p, None, 2), v.reshape(d0, d1)
    if layout == LINEAR:      # [N, K] -> [K][N], as columns [p, p + N) of [K][ld] when ld > 0
        return (d1, ld or d0), (ALL, slice(p, p + d0)), v.reshape(d0, d1).T
    if layout == CONV:        # [O, C, k] -> [k][C][O]
        return (d2, d1, d0), ALL, v.reshape(d0, d1, d2).transpose(2, 1, 0)
    if layout == TCONV:       # [C, O, k], stride p: k = p -> [C][p][O]; k = 2p -> tap 0 = W[..., p:], tap 1 = W[..., :p]
        w = v.reshape(d0, d1, d2)
        taps = [w[:, :, p:], w[:, :, :p]] if d2 == 2 * p else [w]
        return (len(taps), d0, p, d1), ALL, np.stack([t.transpose(0, 2, 1) for t in taps])
    if layout == CONV_ROWS:   # [O, C, k] -> [O][k][C]
        return (d0, d2, d1), ALL, v.reshape(d0, d1, d2).transpose(0, 2, 1)
    return (v.size,), ALL, v


# (id, layout, d0, d1, d2, p, ld, storage, scale): storage F32, or the 16-bit compute dtype the tensor is stored in
CASES = [
    ("plain_bf16", PLAIN, 37, 0, 0, 0, 0, BF16, 1.0),
    ("plain_f16", PLAIN, 37, 0, 0, 0, 0, F16, 1.0),
    ("plain_f32", PLAIN, 37, 0, 0, 0, 0, F32, 1.0),
    ("llama_rope_rows", ROPE_PERM, 24, 5, 0, 8, 0, BF16, 1.0),
    ("llama_rope_rows_f16", ROPE_PERM, 16, 3, 0, 16, 0, F16, 1.0),
    ("qwen3_rope_norm", ROPE_PERM, 8, 1, 0, 8, 0, F32, 1.0),
    ("llama_gate", INTERLEAVE, 6, 5, 0, 0, 0, BF16, 1.0),
    ("llama_up", INTERLEAVE, 6, 5, 0, 1, 0, BF16, 1.0),
    ("codec_linear", LINEAR, 6, 7, 0, 0, 0, F32, 1.0),
    ("codec_linear_block_first", LINEAR, 4, 7, 0, 0, 11, F32, 1.0),
    ("codec_linear_block_mid", LINEAR, 3, 7, 0, 4, 11, F32, 1.0),
    ("codec_linear_block_last", LINEAR, 4, 7, 0, 7, 11, F32, 1.0),
    ("tts_text_projection", LINEAR, 9, 4, 0, 0, 0, F32, 1.0),
    ("codec_conv7", CONV, 3, 4, 7, 0, 0, F32, 1.0),
    ("codec_conv1", CONV, 5, 4, 1, 0, 0, F32, 1.0),
    ("codec_tconv_k_eq_s", TCONV, 3, 4, 3, 3, 0, F32, 1.0),
    ("codec_tconv_k_eq_2s", TCONV, 3, 4, 6, 3, 0, F32, 1.0),
    ("whisper_conv_f16", CONV_ROWS, 4, 8, 3, 0, 0, F16, 1.0),
    ("whisper_conv_bf16", CONV_ROWS, 4, 8, 3, 0, 0, BF16, 1.0),
    ("whisper_q_fold_f16", PLAIN, 40, 0, 0, 0, 0, F16, 0.125),
    ("whisper_q_fold_bf16", PLAIN, 40, 0, 0, 0, 0, BF16, 0.125),
    ("whisper_q_bias_fold", PLAIN, 40, 0, 0, 0, 0, F32, 0.125),
    ("scale_before_rounding", PLAIN, 40, 0, 0, 0, 0, BF16, 0.7),
]


@pytest.mark.parametrize("src_dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_layout_matches_numpy(exe, tmp_path, case, src_dtype):
    name, layout, d0, d1, d2, p, ld, storage, scale = case
    n = d0 * max(d1, 1) * max(d2, 1)
    rng = np.random.default_rng([zlib.crc32(name.encode()), src_dtype])
    # NaN / tie bytes are compared exactly; float16 NaN payloads are not part of the contract
    raw, v = source(rng, n, src_dtype, specials=storage != F16)
    v = v * np.float32(scale)
    if storage != F32:
        v = bf16_bits(v) if storage == BF16 else v.astype(np.float16).view(np.uint16)
    shape, where, values = expected(layout, v, d0, d1, d2, p, ld)
    want = np.full(int(np.prod(shape)) * v.itemsize, SENTINEL, np.uint8)
    want.view(v.dtype).reshape(shape)[where] = values
    src_path, out_path = tmp_path / "src.bin", tmp_path / "out.bin"
    raw.tofile(src_path)
    r = subprocess.run([exe, str(layout), str(d0), str(d1), str(d2), str(p), str(ld), str(n), str(int(storage != F32)),
                        str(src_dtype), str(storage if storage != F32 else BF16), float(scale).hex(), str(want.size),
                        str(src_path), str(out_path)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    got = np.fromfile(out_path, np.uint8)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} bytes differ, first at byte {bad[:8]}"


def fnv1a(name):
    # the library's offset basis, not FNV's published 0xCBF29CE484222325: every init_random weight depends on it
    h = 0x14650FB0739D0383
    for b in name.encode():
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


@pytest.mark.parametrize("seed,name", [(0, "model.layers.0.mlp.gate_proj.weight"), (0x7A11, "model.norm.weight"),
                                       (2**64 - 1, "decoder.1.block.0.alpha"), (12345, "")])
def test_init_random_seed_is_fnv1a_of_the_name(exe, seed, name):
    r = subprocess.run([exe, "seed", str(seed), name], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    assert int(r.stdout) == seed ^ fnv1a(name)
