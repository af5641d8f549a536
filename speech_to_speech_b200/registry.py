"""Registration of the H100 handlers in the reference's backend registry
(speech_to_speech/backend_registry.py:77-100 BackendSpec, :151-161 registry dicts, :206-233
`_simple_handler_factory`).  Two ways in, both leaving the registry module unmodified:

  register()            adds the specs "b200-whisper" (stt), "b200-transformers" (llm) and "b200-qwen3" (tts) next to the
                        built-in ones.
                        Must run before `module_arguments` / `s2s_pipeline` freeze the CLI `choices` from the dict
                        keys (SURVEY.md 8b), i.e. `import speech_to_speech_b200.registry as r; r.register()` first.
  install_overrides()   keeps the names `whisper` / `transformers` / `qwen3` and points their lazy factories at our
                        classes (the literal "registry unchanged" reading).
"""
from __future__ import annotations

from typing import Any

STT_MODULE, STT_CLASS = "speech_to_speech_b200.handlers.whisper_stt_handler", "B200WhisperSTTHandler"
LLM_MODULE, LLM_CLASS = "speech_to_speech_b200.handlers.language_model_handler", "B200LanguageModelHandler"
TTS_MODULE, TTS_CLASS = "speech_to_speech_b200.handlers.qwen3_tts_handler", "B200Qwen3TTSHandler"


def _registry():
    import importlib
    return importlib.import_module("speech_to_speech.backend_registry")


def register() -> dict[str, Any]:
    br = _registry()
    from speech_to_speech.arguments_classes.whisper_stt_arguments import WhisperSTTHandlerArguments
    specs = {}
    stt = br.BackendSpec(name="b200-whisper", kind="stt", config_type=WhisperSTTHandlerArguments,
                         create_handler=br._simple_handler_factory(STT_MODULE, STT_CLASS, attach_speculative_turns=True),
                         config_prefix="stt")
    br.STT_BACKENDS["b200-whisper"] = stt
    specs["b200-whisper"] = stt
    base = br.LLM_BACKENDS.get("transformers")
    if base is not None:
        import dataclasses

        def _create(ctx: Any, config: Any) -> Any:
            import importlib
            cls = getattr(importlib.import_module(LLM_MODULE), LLM_CLASS)
            return cls(ctx.stop_event, queue_in=ctx.queue_in, queue_out=ctx.queue_out,
                       setup_kwargs={**dict(config), "cancel_scope": ctx.cancel_scope, "speculative_turns": ctx.speculative_turns})

        llm = dataclasses.replace(base, name="b200-transformers", create_handler=_create)
        br.LLM_BACKENDS["b200-transformers"] = llm
        specs["b200-transformers"] = llm
    tts_base = br.TTS_BACKENDS.get("qwen3")
    if tts_base is not None:   # same config dataclass (Qwen3TTSHandlerArguments) and prefix; only the class the factory resolves
        import dataclasses
        tts = dataclasses.replace(tts_base, name="b200-qwen3", create_handler=_tts_factory(br))
        br.TTS_BACKENDS["b200-qwen3"] = tts
        specs["b200-qwen3"] = tts
    return specs


def _tts_factory(br: Any) -> Any:
    # the reference's qwen3 entry: setup_should_listen=True, context_kwargs=True (backend_registry.py:478-488)
    return br._simple_handler_factory(TTS_MODULE, TTS_CLASS, setup_should_listen=True, context_kwargs=True)


def _llm_factory() -> Any:
    def _create(ctx: Any, config: Any) -> Any:
        import importlib
        cls = getattr(importlib.import_module(LLM_MODULE), LLM_CLASS)
        cfg = dict(config)
        cfg.pop("is_vlm", None)   # the VLM branch of the reference's local-LLM factory is outside the built path
        return cls(ctx.stop_event, queue_in=ctx.queue_in, queue_out=ctx.queue_out,
                   setup_kwargs={**cfg, "cancel_scope": ctx.cancel_scope, "speculative_turns": ctx.speculative_turns})
    return _create


def install_overrides() -> None:
    br = _registry()
    import dataclasses
    spec = br.STT_BACKENDS["whisper"]
    br.STT_BACKENDS["whisper"] = dataclasses.replace(
        spec, create_handler=br._simple_handler_factory(STT_MODULE, STT_CLASS, attach_speculative_turns=True))
    if "transformers" in br.LLM_BACKENDS:
        br.LLM_BACKENDS["transformers"] = dataclasses.replace(br.LLM_BACKENDS["transformers"], create_handler=_llm_factory())
    if "qwen3" in br.TTS_BACKENDS:
        br.TTS_BACKENDS["qwen3"] = dataclasses.replace(br.TTS_BACKENDS["qwen3"], create_handler=_tts_factory(br))
