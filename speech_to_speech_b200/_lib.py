"""ctypes binding of libs2s_b200.so (C ABI: include/s2s_b200.h).  Fails loudly when the library is missing."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# S2S_LIB_PATH: developer aid (A/B of two builds); the product always loads the in-tree library
LIB_PATH = os.environ.get("S2S_LIB_PATH") or os.path.join(_HERE, "libs2s_b200.so")

S2S_F32, S2S_F16, S2S_BF16 = 0, 1, 2
S2S_FP8_E4M3 = 3  # weight storage only (s2s_llama_set_weight_format)
WEIGHT_FORMAT_CODES = {"float8_e4m3": S2S_FP8_E4M3}
DTYPE_CODES = {"float32": S2S_F32, "float16": S2S_F16, "bfloat16": S2S_BF16}

# every symbol include/s2s_b200.h declares (checked by tests/test_abi.py)
EXPORTED = [
    "s2s_init", "s2s_destroy", "s2s_set_sm_partition", "s2s_last_error", "s2s_launch_count", "s2s_allocated_bytes",
    "s2s_whisper_create", "s2s_whisper_destroy", "s2s_whisper_bind_tensor", "s2s_whisper_init_random",
    "s2s_whisper_finalize", "s2s_whisper_logmel", "s2s_whisper_encode", "s2s_whisper_decode",
    "s2s_whisper_detect_language", "s2s_whisper_transcribe", "s2s_whisper_set_trace", "s2s_whisper_max_decode_batch",
    "s2s_whisper_create_shared", "s2s_whisper_device_bytes",
    "s2s_gemm_ex", "s2s_tiled_weight_bytes", "s2s_tile_weights", "s2s_attention", "s2s_decode_attention", "s2s_decode_gemv",
    "s2s_norm_rows", "s2s_prefill_rope", "s2s_argmax_row",
    "s2s_llama_create", "s2s_llama_destroy", "s2s_llama_bind_tensor", "s2s_llama_init_random",
    "s2s_llama_finalize", "s2s_llama_session_reset", "s2s_llama_set_sampling", "s2s_llama_prefill", "s2s_llama_prefill_batch", "s2s_llama_decode", "s2s_llama_generate", "s2s_llama_set_trace", "s2s_llama_max_decode_batch",
    "s2s_llama_set_weight_format", "s2s_llama_weight_format", "s2s_llama_device_bytes", "s2s_llama_create_shared",
    "s2s_tts_postproc",
    "s2s_codec_create", "s2s_codec_destroy", "s2s_codec_bind_tensor", "s2s_codec_init_random", "s2s_codec_finalize",
    "s2s_codec_decode", "s2s_codec_samples", "s2s_codec_total_upsample", "s2s_codec_contract",
    "s2s_qwen3tts_create", "s2s_qwen3tts_destroy", "s2s_qwen3tts_bind_tensor", "s2s_qwen3tts_init_random",
    "s2s_qwen3tts_finalize", "s2s_qwen3tts_prefill", "s2s_qwen3tts_set_sampling", "s2s_qwen3tts_decode_frames",
    "s2s_qwen3tts_decode_frames_logits", "s2s_qwen3tts_decode_audio", "s2s_qwen3tts_decode_audio_batch",
    "s2s_qwen3tts_set_frames", "s2s_qwen3tts_frames", "s2s_qwen3tts_max_batch", "s2s_qwen3tts_codec", "s2s_qwen3tts_set_trace",
    "s2s_qwen3tts_create_shared", "s2s_qwen3tts_device_bytes",
]


class WhisperConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "d_model", "heads", "enc_layers", "dec_layers", "ffn", "n_mels", "vocab",
        "max_source_positions", "max_target_positions", "compute_dtype", "max_batch")]


class WhisperDecodeOpts(C.Structure):
    _fields_ = [
        ("prefix_h", C.POINTER(C.c_int32)), ("n_prefix", C.c_int32), ("max_new_tokens", C.c_int32),
        ("eos_id", C.c_int32), ("suppress_h", C.POINTER(C.c_int32)), ("n_suppress", C.c_int32),
        ("begin_suppress_h", C.POINTER(C.c_int32)), ("n_begin_suppress", C.c_int32),
        ("prefix_rows_h", C.POINTER(C.c_int32)),
    ]


class LlamaConfig(C.Structure):
    _fields_ = [
        ("d_model", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("ffn", C.c_int32), ("vocab", C.c_int32),
        ("rope_theta", C.c_float), ("rms_eps", C.c_float),
        ("compute_dtype", C.c_int32), ("max_sessions", C.c_int32), ("max_positions", C.c_int32),
        ("max_prefill", C.c_int32), ("qk_norm", C.c_int32), ("n_tables", C.c_int32),
    ]


class Sampling(C.Structure):
    _fields_ = [
        ("do_sample", C.c_int32), ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
        ("repetition_penalty", C.c_float), ("min_new_tokens", C.c_int32), ("n_eos", C.c_int32), ("eos_ids", C.c_int32 * 8),
        ("seed", C.c_uint64),
    ]


class CodecConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("codebook_size", "hidden", "heads", "kv_heads", "inter", "layers", "quantizers")] + [
        ("n_upsample_rates", C.c_int32), ("upsample_rates", C.c_int32 * 8),
        ("n_upsampling_ratios", C.c_int32), ("upsampling_ratios", C.c_int32 * 4),
        ("decoder_dim", C.c_int32), ("sliding_window", C.c_int32), ("rope_theta", C.c_float), ("rms_eps", C.c_float),
        ("max_frames", C.c_int32), ("max_batch", C.c_int32), ("precision", C.c_int32)]


class ConvArgs(C.Structure):
    """s2s_conv_args: one codec-decoder contraction (s2s_codec_contract)."""
    _fields_ = [
        ("x", C.c_void_p), ("ldx", C.c_int64), ("T_in", C.c_int32), ("x_row0", C.c_int32),
        ("x16", C.c_void_p),
        ("w", C.c_void_p), ("k", C.c_int32), ("dil", C.c_int32), ("C_in", C.c_int32), ("N", C.c_int32),
        ("bias", C.c_void_p), ("bias_mod", C.c_int32),
        ("act", C.c_int32),
        ("scale", C.c_void_p),
        ("resid", C.c_void_p), ("ldr", C.c_int64),
        ("y", C.c_void_p), ("ldy", C.c_int64), ("T_out", C.c_int32),
        ("t0", C.c_int32),
        ("batch", C.c_int32), ("x_bs", C.c_int64), ("y_bs", C.c_int64), ("r_bs", C.c_int64),
    ]


class GemmArgs(C.Structure):
    """s2s_gemm_args: one call of the prefill / encoder GEMM (s2s_gemm_ex)."""
    _fields_ = [
        ("a", C.c_void_p), ("a_row_stride", C.c_int64), ("a_batch_stride", C.c_int64),
        ("w", C.c_void_p), ("ldw", C.c_int64),
        ("w_layout", C.c_int32),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("batch", C.c_int32),
        ("bias", C.c_void_p), ("act", C.c_int32),
        ("out_h", C.c_void_p), ("ldo_h", C.c_int64),
        ("out_f", C.c_void_p), ("ldo_f", C.c_int64),
        ("resid", C.c_void_p), ("ld_resid", C.c_int64), ("resid_mode", C.c_int32),
        ("out_batch_rows", C.c_int64), ("out_row_offset", C.c_int64),
        ("head_major_rows", C.c_int32),
        ("dtype", C.c_int32), ("bn", C.c_int32),
    ]


class DecAttnArgs(C.Structure):
    """s2s_dec_attn_args: one decode attention phase by itself (s2s_decode_attention)."""
    _fields_ = [
        ("q", C.c_void_p), ("kv", C.c_void_p), ("max_pos", C.c_int32),
        ("slots_h", C.POINTER(C.c_int32)), ("lens_h", C.POINTER(C.c_int32)), ("B", C.c_int32),
        ("heads", C.c_int32), ("kv_heads", C.c_int32), ("hd", C.c_int32), ("dtype", C.c_int32),
        ("grid", C.c_int32), ("assoc_b", C.c_int32), ("out", C.c_void_p),
        ("qk_norm", C.c_int32), ("kraw", C.c_void_p), ("q_norm", C.c_void_p), ("k_norm", C.c_void_p), ("rope", C.c_void_p),
        ("eps", C.c_float), ("qn_out", C.c_void_p),
    ]


class DecGemvProj(C.Structure):
    """s2s_dec_gemv_proj: one projection of an s2s_decode_gemv call."""
    _fields_ = [
        ("w", C.c_void_p), ("N", C.c_int32), ("K", C.c_int32), ("bias", C.c_void_p),
        ("input", C.c_int32),
        ("x16", C.c_void_p), ("kc", C.c_int32),
        ("xf", C.c_void_p), ("norm", C.c_int32), ("norm_w", C.c_void_p), ("norm_b", C.c_void_p), ("eps", C.c_float),
        ("rg", C.c_int32),
        ("parts", C.c_void_p), ("n_parts", C.c_int32), ("add_bias", C.c_void_p), ("x_out", C.c_void_p),
        ("staged", C.c_void_p),
        ("mode", C.c_int32),
        ("out", C.c_void_p), ("ldo", C.c_int32), ("out_h", C.c_void_p), ("ldh", C.c_int32),
        ("kv0", C.c_void_p), ("kv_which", C.c_int64), ("kv_batch", C.c_int64), ("d", C.c_int32),
        ("pos", C.c_void_p), ("slot", C.c_void_p), ("kv_slot", C.c_int64), ("kv_ld", C.c_int32), ("rope", C.c_void_p),
        ("hd", C.c_int32), ("q_rows", C.c_int32), ("k_rows", C.c_int32),
        ("q_scale", C.c_float), ("kraw", C.c_void_p),
        ("suppress", C.c_void_p), ("first_step", C.c_int32), ("logits_out", C.c_void_p), ("logits_ld", C.c_int64),
        ("argmax_out", C.c_void_p),
        ("head_plan", C.c_int32), ("x_cluster_stride", C.c_int64), ("out_cluster_stride", C.c_int64),
    ]


class DecGemvArgs(C.Structure):
    """s2s_dec_gemv_args: 1..3 decode projections in one launch (s2s_decode_gemv)."""
    _fields_ = [("proj", DecGemvProj * 3), ("n_proj", C.c_int32)] + [(n, C.c_int32) for n in (
        "B", "dtype", "weight_format", "llama", "grid", "slots", "prefetch", "use_plans", "drain", "cluster", "heads")]


class Qwen3TTSConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "d_model", "layers", "heads", "kv_heads", "head_dim", "ffn", "vocab",
        "cp_layers", "cp_heads", "cp_kv_heads", "cp_head_dim", "cp_ffn", "cp_vocab", "n_groups", "text_vocab", "text_hidden")] + [
        ("rope_theta", C.c_float), ("rms_eps", C.c_float)] + [(n, C.c_int32) for n in (
            "compute_dtype", "max_sessions", "max_positions", "max_text",
            "codec_eos", "codec_nothink", "codec_think_bos", "codec_think_eos", "codec_pad", "codec_bos",
            "tts_bos", "tts_eos", "tts_pad", "im_start", "assistant", "newline")] + [("codec", CodecConfig)]


class S2SError(RuntimeError):
    pass


_lib = None


def load() -> C.CDLL:
    """Load the shared library.  No fallback: a missing build is an ImportError (the reference's
    backend_registry turns ImportError into an actionable install hint, S/backend_registry.py:184-193)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  speech_to_speech_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    lib.s2s_last_error.restype = C.c_char_p
    lib.s2s_launch_count.restype = C.c_int64
    lib.s2s_launch_count.argtypes = [C.c_void_p, C.c_int]
    lib.s2s_init.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.s2s_destroy.argtypes = [C.c_void_p]
    lib.s2s_set_sm_partition.argtypes = [C.c_void_p, C.c_int32]
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    lib.s2s_allocated_bytes.argtypes = [C.POINTER(i64)]
    lib.s2s_whisper_create.argtypes = [vp, C.POINTER(WhisperConfig), C.POINTER(vp)]
    lib.s2s_whisper_destroy.argtypes = [vp]
    lib.s2s_whisper_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_whisper_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_whisper_finalize.argtypes = [vp]
    lib.s2s_whisper_create_shared.argtypes = [vp, vp, C.POINTER(WhisperConfig), C.POINTER(vp)]
    lib.s2s_whisper_device_bytes.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.s2s_whisper_logmel.argtypes = [vp, vp, i64, C.POINTER(i32), i32, vp, vp]
    lib.s2s_whisper_encode.argtypes = [vp, vp, i32, vp, vp]
    lib.s2s_whisper_decode.argtypes = [vp, C.POINTER(WhisperDecodeOpts), i32, vp, vp, vp, vp, vp]
    lib.s2s_whisper_detect_language.argtypes = [vp, i32, C.POINTER(i32), i32, i32, vp, vp]
    lib.s2s_whisper_transcribe.argtypes = [vp, C.POINTER(WhisperDecodeOpts), vp, i64, C.POINTER(i32), i32, vp, vp, vp]
    lib.s2s_whisper_set_trace.argtypes = [vp, vp, i32]
    lib.s2s_whisper_max_decode_batch.argtypes = [vp]
    lib.s2s_whisper_max_decode_batch.restype = i32
    lib.s2s_gemm_ex.argtypes = [vp, C.POINTER(GemmArgs), vp]
    lib.s2s_tiled_weight_bytes.argtypes = [i32, i32, i32]
    lib.s2s_tiled_weight_bytes.restype = i64
    lib.s2s_tile_weights.argtypes = [vp, vp, i32, i32, i32, vp, vp]
    lib.s2s_attention.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i64, i64, i64, i64, f32, i32, i32, vp]
    lib.s2s_decode_attention.argtypes = [vp, C.POINTER(DecAttnArgs), C.POINTER(i32), vp]
    lib.s2s_decode_gemv.argtypes = [vp, C.POINTER(DecGemvArgs), C.POINTER(i32), vp]
    lib.s2s_norm_rows.argtypes = [vp, vp, vp, vp, f32, i64, i32, vp, vp, i32, vp]
    lib.s2s_prefill_rope.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, i32, vp, vp, f32, vp, vp, i32, vp]
    lib.s2s_argmax_row.argtypes = [vp, vp, i32, vp, vp]
    lib.s2s_llama_create.argtypes = [vp, C.POINTER(LlamaConfig), C.POINTER(vp)]
    lib.s2s_llama_destroy.argtypes = [vp]
    lib.s2s_llama_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_llama_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_llama_finalize.argtypes = [vp]
    lib.s2s_llama_create_shared.argtypes = [vp, vp, C.POINTER(LlamaConfig), C.POINTER(vp)]
    lib.s2s_llama_set_weight_format.argtypes = [vp, i32]
    lib.s2s_llama_weight_format.argtypes = [vp]
    lib.s2s_llama_weight_format.restype = i32
    lib.s2s_llama_device_bytes.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.s2s_llama_session_reset.argtypes = [vp, i32]
    lib.s2s_llama_set_sampling.argtypes = [vp, i32, C.POINTER(Sampling)]
    lib.s2s_llama_prefill.argtypes = [vp, i32, C.POINTER(i32), i32, vp, vp, vp]
    lib.s2s_llama_prefill_batch.argtypes = [vp, C.POINTER(i32), i32, C.POINTER(i32), C.POINTER(i32), vp, vp]
    lib.s2s_llama_decode.argtypes = [vp, C.POINTER(i32), i32, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.s2s_llama_generate.argtypes = [vp, i32, C.POINTER(i32), i32, i32, i32, vp, vp, vp]
    lib.s2s_llama_set_trace.argtypes = [vp, vp, i32]
    lib.s2s_llama_max_decode_batch.argtypes = [vp]
    lib.s2s_llama_max_decode_batch.restype = i32
    lib.s2s_tts_postproc.argtypes = [vp, vp, i32, vp, i32, vp, C.POINTER(i32), vp]
    lib.s2s_codec_create.argtypes = [vp, C.POINTER(CodecConfig), C.POINTER(vp)]
    lib.s2s_codec_destroy.argtypes = [vp]
    lib.s2s_codec_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_codec_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_codec_finalize.argtypes = [vp]
    lib.s2s_codec_decode.argtypes = [vp, vp, i32, i32, vp, C.POINTER(i32), vp, vp]
    lib.s2s_codec_samples.argtypes = [vp, i32]
    lib.s2s_codec_samples.restype = i32
    lib.s2s_codec_total_upsample.argtypes = [vp]
    lib.s2s_codec_total_upsample.restype = i32
    lib.s2s_codec_contract.argtypes = [vp, C.POINTER(ConvArgs), i32, vp]
    lib.s2s_qwen3tts_create.argtypes = [vp, C.POINTER(Qwen3TTSConfig), C.POINTER(vp)]
    lib.s2s_qwen3tts_destroy.argtypes = [vp]
    lib.s2s_qwen3tts_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_qwen3tts_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_qwen3tts_finalize.argtypes = [vp]
    lib.s2s_qwen3tts_create_shared.argtypes = [vp, vp, C.POINTER(Qwen3TTSConfig), C.POINTER(vp)]
    lib.s2s_qwen3tts_device_bytes.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.s2s_qwen3tts_prefill.argtypes = [vp, i32, C.POINTER(i32), i32, i32, vp]
    lib.s2s_qwen3tts_set_sampling.argtypes = [vp, i32, C.POINTER(Sampling), C.POINTER(Sampling)]
    lib.s2s_qwen3tts_decode_frames.argtypes = [vp, C.POINTER(i32), i32, i32, vp, vp, vp]
    lib.s2s_qwen3tts_decode_frames_logits.argtypes = [vp, C.POINTER(i32), i32, i32, vp, vp, vp, vp, vp]
    lib.s2s_qwen3tts_decode_audio.argtypes = [vp, i32, i32, i32, vp, C.POINTER(i32), vp]
    lib.s2s_qwen3tts_decode_audio_batch.argtypes = [vp, C.POINTER(i32), i32, i32, i32, vp, i64, C.POINTER(i32), vp]
    lib.s2s_qwen3tts_set_frames.argtypes = [vp, i32, i32]
    lib.s2s_qwen3tts_frames.argtypes = [vp, i32]
    lib.s2s_qwen3tts_frames.restype = i32
    lib.s2s_qwen3tts_max_batch.argtypes = [vp]
    lib.s2s_qwen3tts_max_batch.restype = i32
    lib.s2s_qwen3tts_set_trace.argtypes = [vp, i32, vp, i32]
    lib.s2s_qwen3tts_codec.argtypes = [vp]
    lib.s2s_qwen3tts_codec.restype = vp
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().s2s_last_error().decode(errors="replace")
        raise S2SError(f"{what} failed ({rc}): {msg}")


def i32_array(values):
    vals = [int(v) for v in values]
    return (C.c_int32 * max(1, len(vals)))(*vals), len(vals)
