"""speech_to_speech_b200 -- H100-native (sm_90a) engine behind huggingface/speech-to-speech's STT / LLM / TTS
handler slots.  The compute path is libs2s_b200.so (hand-written CUDA, C ABI in include/s2s_b200.h) bound
through ctypes; PyTorch is used only for device memory and streams.  There is no CPU fallback: importing the
engine without the built library, or running it without an H100, raises."""

__version__ = "0.1.0"
