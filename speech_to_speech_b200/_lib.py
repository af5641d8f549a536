"""ctypes binding of libs2s_b200.so (C ABI: include/s2s_b200.h).  Fails loudly when the library is missing."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# S2S_LIB_PATH: developer aid (A/B of two builds); the product always loads the in-tree library
LIB_PATH = os.environ.get("S2S_LIB_PATH") or os.path.join(_HERE, "libs2s_b200.so")

S2S_F32, S2S_F16, S2S_BF16 = 0, 1, 2
DTYPE_CODES = {"float32": S2S_F32, "float16": S2S_F16, "bfloat16": S2S_BF16}

# every symbol include/s2s_b200.h declares (checked by tests/test_abi.py)
EXPORTED = [
    "s2s_init", "s2s_destroy", "s2s_set_sm_partition", "s2s_last_error", "s2s_launch_count",
    "s2s_whisper_create", "s2s_whisper_destroy", "s2s_whisper_bind_tensor", "s2s_whisper_init_random",
    "s2s_whisper_finalize", "s2s_whisper_logmel", "s2s_whisper_encode", "s2s_whisper_decode",
    "s2s_whisper_detect_language", "s2s_whisper_transcribe", "s2s_whisper_set_trace", "s2s_whisper_max_decode_batch",
    "s2s_gemm", "s2s_attention",
    "s2s_llama_create", "s2s_llama_destroy", "s2s_llama_bind_tensor", "s2s_llama_init_random",
    "s2s_llama_finalize", "s2s_llama_session_reset", "s2s_llama_prefill", "s2s_llama_prefill_batch", "s2s_llama_decode", "s2s_llama_generate", "s2s_llama_set_trace", "s2s_llama_max_decode_batch",
    "s2s_tts_postproc",
    "s2s_codec_create", "s2s_codec_destroy", "s2s_codec_bind_tensor", "s2s_codec_init_random", "s2s_codec_finalize",
    "s2s_codec_decode", "s2s_codec_samples", "s2s_codec_total_upsample",
    "s2s_qwen3tts_create", "s2s_qwen3tts_destroy", "s2s_qwen3tts_bind_tensor", "s2s_qwen3tts_init_random",
    "s2s_qwen3tts_finalize", "s2s_qwen3tts_prefill", "s2s_qwen3tts_decode_frames", "s2s_qwen3tts_decode_audio", "s2s_qwen3tts_decode_audio_batch",
    "s2s_qwen3tts_set_frames", "s2s_qwen3tts_frames", "s2s_qwen3tts_max_batch", "s2s_qwen3tts_codec", "s2s_qwen3tts_set_trace",
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


class CodecConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("codebook_size", "hidden", "heads", "kv_heads", "inter", "layers", "quantizers")] + [
        ("n_upsample_rates", C.c_int32), ("upsample_rates", C.c_int32 * 8),
        ("n_upsampling_ratios", C.c_int32), ("upsampling_ratios", C.c_int32 * 4),
        ("decoder_dim", C.c_int32), ("sliding_window", C.c_int32), ("rope_theta", C.c_float), ("rms_eps", C.c_float),
        ("max_frames", C.c_int32), ("max_batch", C.c_int32), ("precision", C.c_int32)]


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
    lib.s2s_whisper_create.argtypes = [vp, C.POINTER(WhisperConfig), C.POINTER(vp)]
    lib.s2s_whisper_destroy.argtypes = [vp]
    lib.s2s_whisper_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_whisper_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_whisper_finalize.argtypes = [vp]
    lib.s2s_whisper_logmel.argtypes = [vp, vp, i64, C.POINTER(i32), i32, vp, vp]
    lib.s2s_whisper_encode.argtypes = [vp, vp, i32, vp, vp]
    lib.s2s_whisper_decode.argtypes = [vp, C.POINTER(WhisperDecodeOpts), i32, vp, vp, vp, vp, vp]
    lib.s2s_whisper_detect_language.argtypes = [vp, i32, C.POINTER(i32), i32, i32, vp, vp]
    lib.s2s_whisper_transcribe.argtypes = [vp, C.POINTER(WhisperDecodeOpts), vp, i64, C.POINTER(i32), i32, vp, vp, vp]
    lib.s2s_whisper_set_trace.argtypes = [vp, vp, i32]
    lib.s2s_whisper_max_decode_batch.argtypes = [vp]
    lib.s2s_whisper_max_decode_batch.restype = i32
    lib.s2s_gemm.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    lib.s2s_attention.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i64, i64, i64, i64, f32, i32, i32, vp]
    lib.s2s_llama_create.argtypes = [vp, C.POINTER(LlamaConfig), C.POINTER(vp)]
    lib.s2s_llama_destroy.argtypes = [vp]
    lib.s2s_llama_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_llama_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_llama_finalize.argtypes = [vp]
    lib.s2s_llama_session_reset.argtypes = [vp, i32]
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
    lib.s2s_qwen3tts_create.argtypes = [vp, C.POINTER(Qwen3TTSConfig), C.POINTER(vp)]
    lib.s2s_qwen3tts_destroy.argtypes = [vp]
    lib.s2s_qwen3tts_bind_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, i32]
    lib.s2s_qwen3tts_init_random.argtypes = [vp, C.c_uint64]
    lib.s2s_qwen3tts_finalize.argtypes = [vp]
    lib.s2s_qwen3tts_prefill.argtypes = [vp, i32, C.POINTER(i32), i32, i32, vp]
    lib.s2s_qwen3tts_decode_frames.argtypes = [vp, C.POINTER(i32), i32, i32, vp, vp, vp]
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
