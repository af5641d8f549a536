"""Minimal mirror of the reference's stage runtime for machines without the upstream speech_to_speech package.

Same constructor, hook names and loop semantics as the reference BaseHandler
(S/baseHandler.py:24-187): `setup(*setup_args, **setup_kwargs)` runs in the constructor, `run()` pulls from
`queue_in` with a 0.1 s timeout, feeds `process(item)` (a generator), pushes every yielded output to
`queue_out`, swallows + logs exceptions raised by `process`, stops on the PIPELINE_END sentinel or `stop_event`,
then calls `cleanup()` and forwards the sentinel.  Message types carry the fields the hot path reads/writes
(S/pipeline/messages.py:45-78, 137-223)."""
from __future__ import annotations

import logging
from dataclasses import dataclass, field
from queue import Empty, Queue
from threading import Event
from time import perf_counter
from typing import Any, Iterator, Optional

import numpy as np

logger = logging.getLogger(__name__)

PIPELINE_END = b"__PIPELINE_END__"
AUDIO_RESPONSE_DONE = b"__AUDIO_RESPONSE_DONE__"


@dataclass
class VADAudio:
    audio: np.ndarray
    runtime_config: Any = None
    mode: Optional[str] = None  # "progressive" | "final" | None
    turn_id: Optional[str] = None
    turn_revision: Optional[int] = None
    processing_delay_s: float = 0.0
    created_at_s: float = field(default_factory=perf_counter)


@dataclass
class PartialTranscription:
    text: str
    turn_id: Optional[str] = None
    turn_revision: Optional[int] = None


@dataclass
class Transcription:
    text: str
    language_code: Optional[str] = None
    turn_id: Optional[str] = None
    turn_revision: Optional[int] = None
    speech_stopped_at_s: Optional[float] = None


@dataclass
class TTSInput:
    text: str
    language_code: Optional[str] = None
    cancel_generation: Optional[int] = None
    response_key: Optional[str] = None
    turn_id: Optional[str] = None
    turn_revision: Optional[int] = None
    speech_stopped_at_s: Optional[float] = None
    runtime_config: Any = None
    prefetch_transaction: Any = None


@dataclass
class EndOfResponse:
    cancel_generation: Optional[int] = None
    response_key: Optional[str] = None
    error: Optional[str] = None


class BaseHandler:
    def __init__(self, stop_event: Event, queue_in: Queue, queue_out: Queue, setup_args: tuple = (),
                 setup_kwargs: dict | None = None) -> None:
        self.stop_event = stop_event
        self.queue_in = queue_in
        self.queue_out = queue_out
        self.pipeline_index = None
        self.setup(*setup_args, **(setup_kwargs or {}))
        self._times: list[float] = []

    def setup(self, *args: Any, **kwargs: Any) -> None:
        pass

    def process(self, item: Any) -> Iterator[Any]:
        raise NotImplementedError

    def should_process_input(self, item: Any) -> bool:
        return True

    def should_emit_output(self, output: Any) -> bool:
        return True

    def before_emit_output(self, output: Any) -> None:
        pass

    def output_for_queue(self, output: Any, source_input: Any) -> Any:
        return output

    def run(self) -> None:
        while not self.stop_event.is_set():
            try:
                item = self.queue_in.get(timeout=0.1)
            except Empty:
                continue
            if isinstance(item, bytes) and item == PIPELINE_END:
                break
            if not self.should_process_input(item):
                continue
            start = perf_counter()
            try:
                for out in self.process(item):
                    if not self.should_emit_output(out):
                        start = perf_counter()
                        continue
                    self._times.append(perf_counter() - start)
                    self.before_emit_output(out)
                    self.queue_out.put(self.output_for_queue(out, item))
                    start = perf_counter()
            except Exception as e:  # same policy as the reference: log, drop the item, keep the stage alive
                logger.error("%s: Error in process(): %s: %s", type(self).__name__, type(e).__name__, e, exc_info=True)
        self.cleanup()
        self.queue_out.put(PIPELINE_END)

    @property
    def last_time(self) -> float:
        return self._times[-1]

    def cleanup(self) -> None:
        pass

    def on_session_end(self) -> None:
        pass


class BaseSTTHandler(BaseHandler):
    """The reference adds speculative-turn stale filtering here (S/STT/base_stt_handler.py:24-128); without a
    SpeculativeTurnTracker every input is current, which is what this mirror implements."""

    speculative_turns = None
