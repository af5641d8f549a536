"""GPU post-processing for the reference's Qwen3-TTS slot.

Scope note (DESIGN.md "TTS"): the Qwen3-TTS talker / codec arithmetic lives in `faster-qwen3-tts`, which is absent
from the reference tree, this container and the wheelhouse, so its parity is unpinned and it is NOT rebuilt here.
What the reference itself computes per audio chunk -- `_resample_to_pipeline_sr` (scipy resample_poly 24 kHz ->
16 kHz) + `_to_int16` (speech_to_speech/TTS/qwen3_tts_handler.py:612-613, 674-680) -- is fused
into one CUDA kernel (`s2s_tts_postproc`), bit-exact against scipy.  `patch_handler_class()` swaps those two
methods on the reference's Qwen3TTSHandler, leaving `_stream`'s trim / 512-sample blocking (:695-749) untouched."""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import numpy as np

PIPELINE_SR = 16000


class TTSPostProcessor:
    def __init__(self, device: int = 0):
        import torch
        from scipy.signal import firwin
        from .. import _lib, engine as E
        self._torch, self._lib, self._E = torch, _lib.load(), E
        self.device = device
        self.ctx = E.get_context(device)
        h = (firwin(61, 1.0 / 3.0, window=("kaiser", 5.0)).astype(np.float32) * np.float32(2)).astype(np.float32)
        self.taps = torch.from_numpy(h).to(f"cuda:{device}")

    def __call__(self, audio24k: np.ndarray) -> np.ndarray:
        """f32[n] @ 24 kHz (host) -> int16[ceil(2n/3)] @ 16 kHz (host)."""
        torch, E = self._torch, self._E
        x = torch.from_numpy(np.ascontiguousarray(audio24k, dtype=np.float32)).to(f"cuda:{self.device}", non_blocking=True)
        n = x.numel()
        out = torch.empty(((2 * n + 2) // 3,), dtype=torch.int16, device=x.device)
        n_out = C.c_int32(0)
        E.check(self._lib.s2s_tts_postproc(self.ctx, E._ptr(x), n, E._ptr(self.taps), self.taps.numel(), E._ptr(out), C.byref(n_out),
                                           E._stream_ptr(self.device)), "s2s_tts_postproc")
        return out[: n_out.value].cpu().numpy()

    def to_int16_device(self, x24k):
        """Device in, device out (int16 cuda tensor): the kernel alone, for device-timed measurements."""
        torch, E = self._torch, self._E
        x = x24k.contiguous()
        n = x.numel()
        out = torch.empty(((2 * n + 2) // 3,), dtype=torch.int16, device=x.device)
        n_out = C.c_int32(0)
        E.check(self._lib.s2s_tts_postproc(self.ctx, E._ptr(x), n, E._ptr(self.taps), self.taps.numel(), E._ptr(out), C.byref(n_out),
                                           E._stream_ptr(self.device)), "s2s_tts_postproc")
        return out[: n_out.value]

    def from_device(self, x24k) -> np.ndarray:
        """f32[n] @ 24 kHz ALREADY ON THE DEVICE (the codec decoder's output) -> int16[ceil(2n/3)] @ 16 kHz (host): no H2D,
        and only int16 samples cross PCIe."""
        torch, E = self._torch, self._E
        x = x24k.contiguous()
        n = x.numel()
        out = torch.empty(((2 * n + 2) // 3,), dtype=torch.int16, device=x.device)
        n_out = C.c_int32(0)
        E.check(self._lib.s2s_tts_postproc(self.ctx, E._ptr(x), n, E._ptr(self.taps), self.taps.numel(), E._ptr(out), C.byref(n_out),
                                           E._stream_ptr(self.device)), "s2s_tts_postproc")
        return out[: n_out.value].cpu().numpy()


def patch_handler_class(handler_cls: Any, device: int = 0) -> Any:
    """Return a subclass of the reference's Qwen3TTSHandler whose resample + int16 conversion run on the GPU."""

    class B200Qwen3TTSHandler(handler_cls):  # type: ignore[misc, valid-type]
        _b200_post: Optional[TTSPostProcessor] = None
        _b200_pending_int16: Optional[np.ndarray] = None

        def _resample_to_pipeline_sr(self, audio: np.ndarray, sr: int) -> np.ndarray:
            if sr != 24000:
                return super()._resample_to_pipeline_sr(audio, sr)
            if self._b200_post is None:
                type(self)._b200_post = TTSPostProcessor(device)
            self._b200_pending_int16 = self._b200_post(audio)
            return audio  # placeholder; _to_int16 below returns the fused result

        def _to_int16(self, audio: np.ndarray) -> np.ndarray:
            if self._b200_pending_int16 is not None:
                out, self._b200_pending_int16 = self._b200_pending_int16, None
                return out
            return super()._to_int16(audio)

    return B200Qwen3TTSHandler
