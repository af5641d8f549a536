"""B200LanguageModelHandler -- the reference's `transformers` LLM slot with prefill + decode on libs2s_b200.so.

Mirrors LanguageModelHandler (speech_to_speech/LLM/language_model.py:785-972): it implements the
two hooks the reference's BaseLanguageModelHandler leaves abstract, `_load_model(model_name, device, torch_dtype,
gen_kwargs)` (:217-224) and `_generate(chat, language_code, gen, ctx, runtime_config, response)` (:238-247), and
reuses the reference's own `_stream_tokens` / sentence batching / cancel logic unchanged (:309-560).  Where the
reference spawns a thread running `pipeline("text-generation")` with a TextIteratorStreamer (:883-888), we run
`s2s_llama_prefill` once and then `s2s_llama_decode` in short persistent launches, detokenising on the host between
launches, so cancellation is polled every `stream_chunk_tokens` tokens.  No CPU fallback.

`gen_kwargs["max_sessions"] = N` (N = number of pipeline units) makes all handler instances of the process with the same
(model, dtype, device) share ONE engine -- one copy of the weights, N KV-cache slots -- and merges the decode chunks of
concurrent sessions into one persistent launch through the SessionBatcher (`batcher.py`): the kernel serves up to
`engine.max_decode_batch()` sessions of different lengths per launch at the cost of one weight stream.

`gen_kwargs["share_weights"] = True` goes one step further with lanes: the engines of all lanes of a (model, dtype,
weight_dtype, device) read ONE copy of the weights (LlamaEngine.share) and the checkpoint is read once per process; each
lane keeps its own engine, KV-cache slots, batcher and stream."""
from __future__ import annotations

import contextlib
import logging
import os
import random
import threading
from typing import Any, Callable, Iterator, Optional, Sequence

from ..batcher import SessionBatcher, acquire_shared, assign_lane, forget_weight_source, release_shared, weight_source
from ..host import _stub_optional

logger = logging.getLogger(__name__)

LLAMA_GEOMETRIES = {
    "micro": dict(d_model=256, layers=2, heads=2, kv_heads=1, head_dim=128, ffn=512, vocab=2048),
    "qwen3-micro": dict(d_model=256, layers=2, heads=4, kv_heads=2, head_dim=64, ffn=512, vocab=2048, rope_theta=1000000.0,
                        rms_eps=1e-6, qk_norm=True),
    # the reference's default LLM (language_model_base_arguments.py:6-9): Qwen/Qwen3-4B-Instruct-2507
    "qwen3-4b": dict(d_model=2560, layers=36, heads=32, kv_heads=8, head_dim=128, ffn=9728, vocab=151936, rope_theta=5000000.0,
                     rms_eps=1e-6, qk_norm=True),
    "mini": dict(d_model=1024, layers=4, heads=8, kv_heads=2, head_dim=128, ffn=3584, vocab=32064),
    "llama-3-8b": dict(d_model=4096, layers=32, heads=32, kv_heads=8, head_dim=128, ffn=14336, vocab=128256,
                       rope_theta=500000.0, rms_eps=1e-5),
    # Qwen/Qwen3-14B and Qwen/Qwen3-32B (config.json): one weight copy makes them fit one H100, 32B in FP8 only
    "qwen3-14b": dict(d_model=5120, layers=40, heads=40, kv_heads=8, head_dim=128, ffn=17408, vocab=151936, rope_theta=1000000.0,
                      rms_eps=1e-6, qk_norm=True),
    "qwen3-32b": dict(d_model=5120, layers=64, heads=64, kv_heads=8, head_dim=128, ffn=25600, vocab=151936, rope_theta=1000000.0,
                      rms_eps=1e-6, qk_norm=True),
}


# GenerationConfig fields the device sampler does not implement, with the value at which they do nothing
_UNSUPPORTED_GENERATION = {"min_p": 0.0, "typical_p": 1.0, "epsilon_cutoff": 0.0, "eta_cutoff": 0.0, "num_beams": 1,
                           "no_repeat_ngram_size": 0}


def resolve_generation(gen_kwargs: dict, generation_config: Any = None) -> dict:
    """The token-choice options of a response, resolved the way transformers' generate() resolves them: its defaults
    (GenerationConfig._get_default_generation_params), overlaid by the checkpoint's generation_config, overlaid by gen_kwargs.
    Returns the keyword arguments of LlamaEngine.set_sampling (without eos_ids / seed).  Raises ValueError for what the
    kernels do not implement instead of silently decoding differently."""
    from transformers import GenerationConfig
    eff = dict(GenerationConfig._get_default_generation_params())
    if generation_config is not None:
        src = generation_config.to_dict() if hasattr(generation_config, "to_dict") else dict(generation_config)
        eff.update({k: v for k, v in src.items() if v is not None})
    eff.update({k: v for k, v in gen_kwargs.items() if v is not None})
    for k, off in _UNSUPPORTED_GENERATION.items():
        v = eff.get(k)
        if v is not None and v != off and not (k == "num_beams" and int(v) <= 1):
            raise ValueError(f"`{k}` (={v}) is not supported by B200LanguageModelHandler: its sampler implements repetition_penalty, "
                             f"min_new_tokens, temperature, top_k and top_p only")
    do_sample = bool(eff.get("do_sample") or False)
    temperature = float(eff.get("temperature") if eff.get("temperature") is not None else 1.0)
    top_k = int(eff.get("top_k") or 0)
    top_p = float(eff.get("top_p") if eff.get("top_p") is not None else 1.0)
    penalty = float(eff.get("repetition_penalty") if eff.get("repetition_penalty") is not None else 1.0)
    if do_sample and not temperature > 0.0:
        raise ValueError(f"`temperature` (={temperature}) has to be a strictly positive float, otherwise your next token scores will be "
                         "invalid. If you're looking for greedy decoding strategies, set `do_sample=False`.")
    if do_sample and not 0.0 < top_p <= 1.0:
        raise ValueError(f"`top_p` has to be a float > 0 and < 1, but is {top_p}")
    if do_sample and top_k < 0:
        raise ValueError(f"`top_k` has to be a strictly positive integer, but is {top_k}")
    if not penalty > 0.0:
        raise ValueError(f"`penalty` has to be a strictly positive float, but is {penalty}")
    return dict(do_sample=do_sample, temperature=temperature if do_sample else 1.0, top_k=top_k if do_sample else 0,
                top_p=top_p if do_sample else 1.0, repetition_penalty=penalty, min_new_tokens=int(eff.get("min_new_tokens") or 0))


class TokenStreamer:
    """Generation as an iterator of text fragments (the role TextIteratorStreamer plays in the reference)."""

    def __init__(self, engine: Any, decode_text: Callable[[Sequence[int]], str], eos_ids: Sequence[int], chunk: int = 8, slot: int = 0,
                 decode_chunk: Optional[Callable[[int, int, int, int], list]] = None, lock: Optional[Any] = None,
                 context: Optional[Callable[[], Any]] = None, prefill: Optional[Callable[..., int]] = None,
                 sampling: Optional[Callable[[], dict]] = None):
        import contextlib
        self._context = context or contextlib.nullcontext   # the lane's CUDA stream for this thread's GPU calls
        self._sampling = sampling   # -> LlamaEngine.set_sampling kwargs of the next response (None: leave the slot as it is)
        self.engine, self.decode_text, self.eos_ids, self.chunk, self.slot = engine, decode_text, set(int(e) for e in eos_ids), max(1, chunk), slot
        self.generated: list[int] = []
        self._po = self._ro = 0   # incremental detokenisation window
        # decode_chunk(slot, first_token, n, eos) -> ids: the shared-engine path routes it through the session batcher;
        # lock serialises prefill on a shared engine (one thread per engine handle at a time)
        self._decode_chunk = decode_chunk or self._decode_direct
        self._prefill = prefill   # shared engine: prompts of concurrent sessions are prefilled in one pass (bundle.prefill)
        self._lock = lock or threading.Lock()

    def _decode_direct(self, slot: int, tok: int, n: int, eos: int) -> list:
        import torch
        eng = self.engine
        first = torch.tensor([tok], dtype=torch.int32, device=f"cuda:{eng.device}")
        with self._lock, self._context():
            ids, lens = eng.decode([slot], first, n, eos_id=eos)
            return ids[0, : int(lens[0]) if int(lens[0]) > 0 else n].tolist()

    def _fresh_text(self) -> str:
        """Incremental detokenisation: decode only the window [previous chunk | new tokens] instead of the whole reply every
        chunk (O(n * window), not O(n^2)); the previous chunk is context for correct spacing / byte merges."""
        toks = self.generated
        before = self.decode_text(toks[self._po:self._ro]) if self._ro > self._po else ""
        now = self.decode_text(toks[self._po:])
        if len(now) > len(before) and not now.endswith("\ufffd"):
            self._po, self._ro = self._ro, len(toks)
            return now[len(before):]
        return ""

    def stream(self, prompt_ids: Sequence[int], max_new_tokens: int, should_stop: Callable[[], bool] = lambda: False) -> Iterator[str]:
        eng = self.engine
        max_prefill = eng.cfg.max_prefill
        max_pos = int(getattr(eng, "max_positions", 1 << 30))
        prompt_ids = list(prompt_ids) or [0]          # an empty prompt still needs one position to predict from
        # one session must never make a shared launch fail (llama.cu rejects len + n_steps > max_positions for the whole batch):
        # keep the tail of an over-long prompt and cap the reply at what the KV slot can still hold
        room = max_pos - 2
        if len(prompt_ids) > room - 1:
            logger.warning("LLM prompt of %d tokens exceeds the %d-position KV slot: keeping the last %d", len(prompt_ids), max_pos, room - 1)
            prompt_ids = prompt_ids[-(room - 1):]
        max_new_tokens = max(1, min(int(max_new_tokens), room - len(prompt_ids)))
        nxt = None
        sampling = self._sampling() if self._sampling is not None else None
        if self._prefill is not None:
            tok = int(self._prefill(self.slot, prompt_ids, sampling) if sampling is not None else self._prefill(self.slot, prompt_ids))
        else:
            with self._lock, self._context():
                eng.reset(self.slot)
                if sampling is not None:
                    eng.set_sampling(self.slot, **sampling)
                for o in range(0, len(prompt_ids), max_prefill):
                    nxt, _ = eng.prefill(self.slot, list(prompt_ids[o:o + max_prefill]))
                tok = int(nxt[0])
        self.generated = []
        self._po = self._ro = 0
        eos_for_kernel = next(iter(self.eos_ids)) if len(self.eos_ids) == 1 else -1
        while len(self.generated) < max_new_tokens:
            if tok in self.eos_ids:
                break
            self.generated.append(tok)
            piece = self._fresh_text()
            if piece:
                yield piece
            if should_stop() or len(self.generated) >= max_new_tokens:
                break
            n = min(self.chunk, max_new_tokens - len(self.generated))
            out = self._decode_chunk(self.slot, tok, n, eos_for_kernel)
            stop = False
            for t in out[:-1]:
                if t in self.eos_ids:
                    stop = True
                    break
                self.generated.append(t)
            if stop or not out:
                break
            tok = out[-1]
        if self.generated:   # flush the tail (tokens appended by the last launch before EOS / budget end)
            before = self.decode_text(self.generated[self._po:self._ro]) if self._ro > self._po else ""
            now = self.decode_text(self.generated[self._po:])
            if len(now) > len(before):
                yield now[len(before):]


class _LlamaBundle:
    """One engine shared by the handler instances of a process: KV-cache slots handed out per handler, prefill serialised
    by a lock, decode chunks of concurrent sessions merged into one launch by the SessionBatcher."""

    def __init__(self, engine: Any, tokenizer: Any, eos_ids: list, max_sessions: int, batch_wait_s: float, lane: int = 0, lanes: int = 1,
                 batch_gap_s: Optional[float] = None, generation_config: Any = None):
        self.engine, self.tokenizer, self.eos_ids = engine, tokenizer, eos_ids
        self.generation_config = generation_config   # the checkpoint's (None for random weights)
        self.lane, self.lanes = lane, lanes
        self.lock = threading.Lock()
        self._free = list(range(max_sessions))
        mb = max(1, min(int(engine.max_decode_batch()), max_sessions))
        self.batcher = SessionBatcher(self._run_batch, mb, batch_wait_s, "s2s-llm-batcher",
                                      thread_context=self.lane_context, idle_gap_s=batch_gap_s) if max_sessions > 1 else None

    def lane_context(self):
        """The lane's CUDA stream as the calling thread's current stream (engine.lane_context; a no-op for one lane)."""
        if self.lanes <= 1:
            return contextlib.nullcontext()
        from .. import engine as E
        return E.lane_context(self.engine.device, self.lane, self.lanes)

    def acquire_slot(self) -> int:
        with self.lock:
            if not self._free:
                raise RuntimeError("all KV-cache slots of the shared LLM engine are in use (raise max_sessions)")
            return self._free.pop(0)

    def release_slot(self, slot: int) -> None:
        with self.lock:
            self._free.append(slot)

    def _run_prefill(self, items: list) -> list:
        """items: (slot, prompt ids[, set_sampling kwargs]).  Each slot is reset and gets its token choice first.  Fresh prompts that fit one pass together are prefilled by ONE s2s_llama_prefill_batch
        call (one pass over the weights for all of them); the rest go one by one, over-long prompts in max_prefill chunks."""
        eng = self.engine
        cap = int(eng.cfg.max_prefill)
        out: list = [None] * len(items)
        with self.lock, self.lane_context():
            group: list = []
            rows = 0

            def flush() -> None:
                nonlocal group, rows
                if len(group) > 1:
                    nxt = eng.prefill_batch([items[i][0] for i in group], [items[i][1] for i in group]).tolist()
                    for i, t in zip(group, nxt):
                        out[i] = int(t)
                elif group:
                    i = group[0]
                    nx = None
                    for o in range(0, len(items[i][1]), cap):
                        nx, _ = eng.prefill(items[i][0], list(items[i][1][o:o + cap]))
                    out[i] = int(nx[0])
                group, rows = [], 0
            for i, it in enumerate(items):
                slot, ids = it[0], it[1]
                eng.reset(slot)
                if len(it) > 2 and it[2] is not None:
                    eng.set_sampling(slot, **it[2])
                if len(ids) > cap:
                    flush()
                    group = [i]
                    flush()
                    continue
                if rows + len(ids) > cap or len(group) >= 16:
                    flush()
                group.append(i)
                rows += len(ids)
            flush()
        return out

    def prefill(self, slot: int, ids: Sequence[int], sampling: Optional[dict] = None) -> int:
        """Reset the session, set its token choice (under the lock, on the lane's stream) and run its prompt; concurrent
        sessions' prompts share one pass over the weights."""
        if self.batcher is None:
            return self._run_prefill([(slot, list(ids), sampling)])[0]
        return self.batcher.call(("prefill",), (slot, list(ids), sampling))

    def _run_batch(self, key: tuple, items: list) -> list:
        import torch
        if key and key[0] == "prefill":
            return self._run_prefill(items)
        n, eos = key
        slots = [it[0] for it in items]
        with self.lock, self.lane_context():
            first = torch.tensor([it[1] for it in items], dtype=torch.int32, device=f"cuda:{self.engine.device}")
            ids, lens = self.engine.decode(slots, first, n, eos_id=eos)
            ids, lens = ids.tolist(), lens.tolist()
        return [row[: (ln if ln > 0 else n)] for row, ln in zip(ids, lens)]

    def decode_chunk(self, slot: int, tok: int, n: int, eos: int) -> list:
        if self.batcher is None:
            return self._run_batch((n, eos), [(slot, tok)])[0]
        return self.batcher.call((n, eos), (slot, tok))

    def close(self) -> None:
        if self.batcher is not None:
            self.batcher.close()
        self.engine.close()

    def share(self, lane: int, lanes: int, max_sessions: int, max_positions: int, batch_wait_s: float,
              batch_gap_s: Optional[float]) -> "_LlamaBundle":
        """A bundle for another lane whose engine reads this bundle's weights (LlamaEngine.share), same tokenizer and EOS ids."""
        engine = self.engine.share(lane, lanes, max_sessions=max_sessions, max_positions=max_positions)
        return _LlamaBundle(engine, self.tokenizer, self.eos_ids, max_sessions, batch_wait_s, lane, lanes, batch_gap_s,
                            self.generation_config)


def geometry_from_hf_config(c: Any, max_positions: int) -> dict:
    """Engine geometry from a transformers config, REJECTING everything the kernels do not implement instead of loading
    it and producing silently wrong logits: model families other than Llama / Mistral / Qwen3, RoPE scaling (Llama-3.1+
    `rope_scaling={"rope_type": "llama3", ...}`, linear, dynamic, yarn), attention / MLP biases, a sliding window shorter than
    the KV slot, MoE variants."""
    mt = getattr(c, "model_type", None)
    if mt not in ("llama", "mistral", "qwen3"):
        raise ValueError(f"B200LanguageModelHandler supports Llama / Mistral / Qwen3 checkpoints (got model_type={mt!r})")
    rope = getattr(c, "rope_parameters", None) or getattr(c, "rope_scaling", None) or {}
    rtype = (rope.get("rope_type") or rope.get("type") or "default") if isinstance(rope, dict) else "default"
    if rtype != "default":
        raise ValueError(f"rope scaling {rtype!r} is not implemented by the sm_90a RoPE table (plain theta^(-2j/hd) only)")
    theta = float((rope.get("rope_theta") if isinstance(rope, dict) else None) or getattr(c, "rope_theta", 10000.0))
    for flag in ("attention_bias", "mlp_bias"):
        if getattr(c, flag, False):
            raise ValueError(f"{flag}=True is not implemented (projections are bias-free in the built path)")
    sw = getattr(c, "sliding_window", None)
    if sw is not None and getattr(c, "use_sliding_window", True) and int(sw) < int(max_positions):
        raise ValueError(f"sliding_window={sw} < max_positions={max_positions}: windowed attention is not implemented")
    heads = int(c.num_attention_heads)
    return dict(d_model=int(c.hidden_size), layers=int(c.num_hidden_layers), heads=heads, kv_heads=int(c.num_key_value_heads),
                head_dim=int(getattr(c, "head_dim", None) or c.hidden_size // heads), ffn=int(c.intermediate_size),
                vocab=int(c.vocab_size), rope_theta=theta, rms_eps=float(c.rms_norm_eps), qk_norm=(mt == "qwen3"))


def _reference_base():
    """The reference's BaseLanguageModelHandler when importable (nltk stubbed like the reference's own tests do)."""
    try:
        _stub_optional("nltk")
        from speech_to_speech.LLM.language_model import BaseLanguageModelHandler
        return BaseLanguageModelHandler
    except Exception:
        return None


_Base = _reference_base()


class _StandaloneBase:
    """Used only where the reference package is absent (e.g. the GPU test box): owns the load hook and exposes
    `generate_text_stream`; the reference-side request lifecycle (Chat, LLMResponseChunk, cancel scopes) needs the
    reference package and is exercised by tests/test_handlers.py with it present."""

    def __init__(self, model_name: str, device: str = "cuda", torch_dtype: str = "bfloat16", gen_kwargs: Optional[dict] = None):
        self.device = device
        self._load_model(model_name, device, torch_dtype, dict(gen_kwargs or {}))


class B200LanguageModelHandler(_Base if _Base is not None else _StandaloneBase):  # type: ignore[misc]
    backend = "transformers"

    def _load_model(self, model_name: str, device: str, torch_dtype: str, gen_kwargs: dict[str, Any]) -> None:
        if not str(device).startswith("cuda"):
            raise ValueError(f"B200LanguageModelHandler runs on CUDA (sm_90a) only, got device={device!r}; there is no CPU fallback")
        from .. import engine as E
        dev = int(device.split(":")[1]) if ":" in device else 0
        self.gen_kwargs = dict(gen_kwargs)
        seed = self.gen_kwargs.pop("seed", None)
        # one 64-bit sampling seed per response, drawn from a generator seeded by gen_kwargs["seed"] (OS entropy when absent)
        self._seed_rng = random.Random(int(seed) if seed is not None else int.from_bytes(os.urandom(8), "little"))
        self.stream_chunk_tokens = int(self.gen_kwargs.pop("stream_chunk_tokens", 8))
        max_pos = int(self.gen_kwargs.pop("max_positions", 4096))
        max_sessions = max(1, int(self.gen_kwargs.pop("max_sessions", 1)))
        batch_wait_s = float(self.gen_kwargs.pop("batch_wait_ms", 6.0)) / 1000.0   # upper bound of the batch window
        gap_ms = float(self.gen_kwargs.pop("batch_gap_ms", 0.6))                     # a batch leaves once arrivals pause this long
        batch_gap_s = gap_ms / 1000.0 if gap_ms > 0 else None
        # SM partition: the handler instances of lane i share lane i's engine (engine.get_context; INTEGRATION.md section 4)
        lanes = max(1, int(self.gen_kwargs.pop("lanes", 1)))
        lane = self.gen_kwargs.pop("lane", None)
        if lane is None:   # not pinned by the caller: units join the lanes round-robin in construction order
            lane = assign_lane(("llama", model_name, dev), lanes)
        lane = int(lane) % lanes
        # weight-only FP8 for the decode launch's projections (engine.LlamaEngine; INTEGRATION.md): off unless asked for
        weight_dtype = self.gen_kwargs.pop("weight_dtype", None)
        if weight_dtype not in (None, "float8_e4m3"):
            raise ValueError(f"weight_dtype={weight_dtype!r}: supported values are None (weights stored as torch_dtype) and 'float8_e4m3'")
        fmt = {"weight_dtype": weight_dtype} if weight_dtype else {}
        # one weight copy for all lanes of the model (LlamaEngine.share): off unless asked for
        share_weights = bool(self.gen_kwargs.pop("share_weights", False))

        def load() -> _LlamaBundle:
            if model_name.startswith("random:"):
                parts = model_name.split(":")
                geom = LLAMA_GEOMETRIES[parts[1]]
                engine = E.LlamaEngine(geom, dtype=torch_dtype, max_sessions=max_sessions, max_positions=max_pos, max_prefill=512, device=dev, lane=lane, lanes=lanes, **fmt)
                engine.init_random(int(parts[2]) if len(parts) > 2 else 0)
                return _LlamaBundle(engine, _IdTokenizer(geom["vocab"]), [geom["vocab"] - 1], max_sessions, batch_wait_s, lane, lanes, batch_gap_s)
            # the checkpoint is read before the weights are loaded so that unsupported options fail fast
            from transformers import AutoModelForCausalLM, AutoTokenizer, GenerationConfig
            try:
                ckpt_gen = GenerationConfig.from_pretrained(model_name)
            except OSError:
                ckpt_gen = None
            resolve_generation(self.gen_kwargs, ckpt_gen)
            tokenizer = AutoTokenizer.from_pretrained(model_name)
            hf = AutoModelForCausalLM.from_pretrained(model_name)
            c = hf.config
            geom = geometry_from_hf_config(c, max_pos)
            engine = E.LlamaEngine(geom, dtype=torch_dtype, max_sessions=max_sessions, max_positions=max_pos, max_prefill=512, device=dev, lane=lane, lanes=lanes, **fmt)
            engine.load_state_dict(hf.state_dict())
            eos = hf.generation_config.eos_token_id
            eos_ids = list(eos) if isinstance(eos, (list, tuple)) else [int(eos)]
            del hf
            return _LlamaBundle(engine, tokenizer, eos_ids, max_sessions, batch_wait_s, lane, lanes, batch_gap_s, ckpt_gen)

        self._weights_key = ("llama", model_name, torch_dtype, weight_dtype, dev) if share_weights else None

        def build() -> _LlamaBundle:
            if self._weights_key is None:
                return load()
            return weight_source(self._weights_key, load,
                                 lambda src: src.share(lane, lanes, max_sessions, max_pos, batch_wait_s, batch_gap_s))

        if model_name.startswith("random:"):
            resolve_generation(self.gen_kwargs)
        self._shared_key = ("llama", model_name, torch_dtype, weight_dtype, dev, max_sessions, max_pos, lane, lanes) if max_sessions > 1 else None
        self.bundle = acquire_shared(self._shared_key, build, self._close_bundle) if self._shared_key else build()
        self.engine, self.tokenizer, self.eos_ids = self.bundle.engine, self.bundle.tokenizer, self.bundle.eos_ids
        self.sampling = resolve_generation(self.gen_kwargs, getattr(self.bundle, "generation_config", None))
        self.slot = self.bundle.acquire_slot()
        self.streamer = TokenStreamer(self.engine, lambda ids: self.tokenizer.decode(list(ids), skip_special_tokens=True),
                                      self.eos_ids, self.stream_chunk_tokens, slot=self.slot, decode_chunk=self.bundle.decode_chunk,
                                      lock=self.bundle.lock, context=self.bundle.lane_context, prefill=self.bundle.prefill,
                                      sampling=self.next_sampling)

    def next_sampling(self) -> dict:
        """LlamaEngine.set_sampling kwargs of the next response: the resolved options, the model's EOS ids (for
        min_new_tokens) and a fresh 64-bit seed."""
        return dict(self.sampling, eos_ids=list(self.eos_ids)[:8], seed=self._seed_rng.getrandbits(64))

    def generate_text_stream(self, prompt_ids: Sequence[int], max_new_tokens: Optional[int] = None,
                             should_stop: Callable[[], bool] = lambda: False) -> Iterator[str]:
        n = int(max_new_tokens or self.gen_kwargs.get("max_new_tokens", 1024))
        return self.streamer.stream(prompt_ids, n, should_stop)

    def setup(self, **kwargs: Any) -> None:  # type: ignore[override]
        """LanguageModelHandler.setup (S/LLM/language_model.py:795-798): base setup, then warm up so that the first user turn
        does not pay for cudaFuncSetAttribute and the cooperative-launch cold start."""
        super().setup(**kwargs)
        self.warmup()

    def _prompt_ids(self, chat_messages: Any) -> list:
        """What the reference feeds the model (:846-848, :885): the chat template rendered with the generation prompt and
        `enable_thinking=False`, then tokenised the way `pipeline("text-generation")` tokenises a string prompt."""
        tok = self.tokenizer
        if isinstance(tok, _IdTokenizer):
            return list(tok.apply_chat_template(chat_messages, tokenize=True, add_generation_prompt=True))
        text = tok.apply_chat_template(chat_messages, tokenize=False, add_generation_prompt=True, enable_thinking=False)
        ids = tok(text)["input_ids"]
        return list(ids[0]) if ids and isinstance(ids[0], (list, tuple)) else list(ids)

    # -- reference hook (S/LLM/language_model.py:832-892) -----------------------------------------
    def _generate(self, chat: Any, language_code: Optional[str], gen: Optional[int], ctx: Any, runtime_config: Any = None,
                  response: Any = None) -> Iterator[Any]:
        chat_messages = chat.to_transformers_chat()
        counted = self.tokenizer.apply_chat_template(chat_messages, tokenize=True)   # the reference's prompt-token count (:842-844)
        ctx.input_tokens += len(counted if isinstance(counted, list) else counted["input_ids"])
        prompt_ids = self._prompt_ids(chat_messages)
        aborted = threading.Event()
        if getattr(ctx, "prefetch_transaction", None) is not None:   # speculative prefetch discarded -> stop at the next chunk (:879-880)
            ctx.prefetch_transaction.register_abort(aborted.set)
        check = getattr(self, "_check_stop", None)
        stop = (lambda: aborted.is_set() or bool(check(gen, ctx))) if check else aborted.is_set
        token_iter = self.generate_text_stream(prompt_ids, should_stop=stop)
        yield from self._stream_tokens(token_iter, gen, language_code, ctx, runtime_config, response)

    def warmup(self) -> None:
        for _ in self.generate_text_stream([1, 2, 3, 4], max_new_tokens=4):
            pass

    def _close_bundle(self, bundle: _LlamaBundle) -> None:
        if getattr(self, "_weights_key", None) is not None:   # never handed out as a weight source once closing
            forget_weight_source(self._weights_key, bundle)
        bundle.close()

    def cleanup(self) -> None:
        bundle = getattr(self, "bundle", None)
        if bundle is None:
            return
        self.bundle = None
        bundle.release_slot(self.slot)
        if self._shared_key is not None:
            release_shared(self._shared_key)  # the last handler of the process closes the shared engine
        else:
            self._close_bundle(bundle)


class _IdTokenizer:
    """Stand-in tokenizer for random-init models: token i <-> the text "<i> "."""

    def __init__(self, vocab: int):
        self.vocab = vocab

    def decode(self, ids: Sequence[int], skip_special_tokens: bool = True) -> str:
        return "".join(f"<{int(i)}> " for i in ids)

    def encode(self, text: str) -> list[int]:
        return [int(t.strip("<> ")) % self.vocab for t in text.split() if t.strip("<> ").isdigit()]

    def apply_chat_template(self, messages: Any, tokenize: bool = True, add_generation_prompt: bool = True, **kw: Any):
        ids: list[int] = []
        for m in messages:
            ids += self.encode(str(m.get("content", ""))) or [1]
        return ids if tokenize else " ".join(f"<{i}>" for i in ids)
