"""Session batcher: concurrent conversation sessions share ONE engine (one copy of the weights) per GPU and their
requests are merged into one launch.

Why (SURVEY.md §8f rank 1): the reference gives every pipeline unit its own handler threads and its own model copy
(`s2s_pipeline.py:554-565`, `--num_pipelines`, `arguments_classes/module_arguments.py:85-93`), so N sessions cost
N weight sets and N independent per-token weight streams.  On the GPU path the decode kernel processes up to 16
sessions per persistent launch at almost the cost of one (the batch is the m dimension of the tensor-core tile,
csrc/decode_common.cuh): measured 1030 concurrent real-time Whisper-small sessions per GPU at 16 per launch
against 121 one at a time.  The batcher is the host piece that makes that reachable from the handler slots:

  handler thread (one per session, unchanged reference threading)      batcher thread (one per engine)
      fut = batcher.submit(key, item)   ------------------------------>   collect items with the same key for at
      ids = fut.result()                <------------------------------   most `max_wait_s` or until `max_batch`,
                                                                          run_batch(key, items) once, scatter

Dispatch policy: a key's batch goes out when it is full (`max_batch`), when its oldest request has waited `max_wait_s`, or --
with `idle_gap_s` set -- as soon as no further request has arrived for `idle_gap_s`.  Sessions that share launches resubmit in
a burst (they all receive the previous launch's results at the same instant), so "the burst is over" is the signal that the
batch is as full as it is going to get: a lone session waits one gap (a fraction of a millisecond) instead of the whole window,
and under load the window can be long enough for every session's request without costing latency when they are all there.

`key` groups requests that may share a launch (the decoder prompt / generation options are per launch in the C ABI:
`s2s_whisper_transcribe` takes one `s2s_whisper_decode_opts`).  Requests with different keys are never mixed; they
are served in arrival order of their first element.  Exceptions raised by `run_batch` are delivered to every future
of that batch -- inside the reference's stage loop that means "log and drop the item" (`baseHandler.py:162-163`).
"""
from __future__ import annotations

import threading
import time
from collections import OrderedDict
from concurrent.futures import Future
from typing import Any, Callable, Hashable, List, Optional, Sequence, Tuple


class SessionBatcher:
    def __init__(self, run_batch: Callable[[Hashable, List[Any]], Sequence[Any]], max_batch: int = 16,
                 max_wait_s: float = 0.004, name: str = "s2s-batcher",
                 thread_context: Optional[Callable[[], Any]] = None, idle_gap_s: Optional[float] = None):
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self._run_batch = run_batch
        self.max_batch = int(max_batch)
        self.max_wait_s = float(max_wait_s)
        self.idle_gap_s = None if idle_gap_s is None else float(idle_gap_s)
        self._last_arrival = 0.0
        self._free_at = 0.0          # when the engine thread finished its last launch
        self._cv = threading.Condition()
        # key -> list of (item, future, t_arrival); OrderedDict keeps the arrival order of each key's oldest request
        self._pending: "OrderedDict[Hashable, List[Tuple[Any, Future, float]]]" = OrderedDict()
        self._closed = False
        self.batches_run = 0
        self.items_run = 0
        self.largest_batch = 0
        # a context manager factory entered once by the engine thread for its whole life (e.g. the lane's CUDA stream)
        self._thread_context = thread_context
        self._fatal: Optional[BaseException] = None
        self._thread = threading.Thread(target=self._loop, name=name, daemon=True)
        self._thread.start()

    # ---- producer side (handler threads) ----------------------------------------------------------------
    def submit(self, key: Hashable, item: Any) -> Future:
        fut: Future = Future()
        with self._cv:
            if self._closed:
                raise RuntimeError("SessionBatcher is closed")
            now = time.monotonic()
            self._pending.setdefault(key, []).append((item, fut, now))
            self._last_arrival = now
            self._cv.notify_all()
        return fut

    def call(self, key: Hashable, item: Any, timeout: Optional[float] = None) -> Any:
        return self.submit(key, item).result(timeout)

    # ---- consumer side (the one thread that talks to the engine) -----------------------------------------
    def _take(self) -> Optional[Tuple[Hashable, List[Tuple[Any, Future, float]]]]:
        """Block until a batch is due: the oldest key has max_batch items, or its oldest item waited max_wait_s."""
        with self._cv:
            while True:
                if self._pending:
                    key, items = next(iter(self._pending.items()))
                    # both clocks run only while the engine is free: requests that queued up behind a running launch must not
                    # leave the instant it ends -- the sessions of THAT launch are about to resubmit, and taking the queue
                    # as it stands locks two groups of sessions into alternating half-full launches
                    due = max(items[0][2], self._free_at) + self.max_wait_s
                    if self.idle_gap_s is not None:       # the burst of resubmissions is over: nothing new for idle_gap_s
                        due = min(due, max(items[-1][2], self._last_arrival, self._free_at) + self.idle_gap_s)
                    now = time.monotonic()
                    if len(items) >= self.max_batch or now >= due or self._closed:
                        batch = items[: self.max_batch]
                        rest = items[self.max_batch:]
                        del self._pending[key]
                        if rest:
                            self._pending[key] = rest  # re-queued behind the other keys
                        return key, batch
                    self._cv.wait(timeout=due - now)
                elif self._closed:
                    return None
                else:
                    self._cv.wait()

    def _loop(self) -> None:
        if self._thread_context is None:
            return self._serve()
        try:
            cm = self._thread_context()
            cm.__enter__()
        except BaseException as exc:   # the waiting handler threads must hear about it: every request fails with this error
            self._fatal = exc
            return self._serve()
        try:
            return self._serve()
        finally:
            cm.__exit__(None, None, None)

    def _serve(self) -> None:
        while True:
            taken = self._take()
            if taken is None:
                return
            key, batch = taken
            live = [(it, fut) for it, fut, _ in batch if fut.set_running_or_notify_cancel()]
            if not live:
                continue
            try:
                if self._fatal is not None:
                    raise RuntimeError(f"SessionBatcher engine thread could not enter its context: {self._fatal!r}")
                results = self._run_batch(key, [it for it, _ in live])
                if len(results) != len(live):
                    raise RuntimeError(f"run_batch returned {len(results)} results for {len(live)} items")
            except BaseException as exc:  # delivered to the waiting handler threads, never swallowed
                for _, fut in live:
                    fut.set_exception(exc)
                self._free_at = time.monotonic()
                continue
            self.batches_run += 1
            self.items_run += len(live)
            self.largest_batch = max(self.largest_batch, len(live))
            for (_, fut), res in zip(live, results):
                fut.set_result(res)
            self._free_at = time.monotonic()

    def close(self, timeout: float = 5.0) -> None:
        """Serve what is queued, then stop the thread."""
        with self._cv:
            self._closed = True
            self._cv.notify_all()
        self._thread.join(timeout)


# ---- lanes: which SM partition a new pipeline unit joins --------------------------------------------------------
_lane_counters: dict = {}


def assign_lane(group: Hashable, lanes: int) -> int:
    """Round-robin lane of the next handler of `group` (slot kind, model, device): unit k of a `--num_pipelines N` process lands
    on lane k mod lanes for each of its three handlers (they are constructed in unit order), so `max_sessions = ceil(N / lanes)`
    slots per lane suffice.  lanes <= 1 -> 0."""
    if lanes <= 1:
        return 0
    with _registry_lock:
        k = _lane_counters.get(group, 0)
        _lane_counters[group] = k + 1
    return k % lanes


# ---- engines shared between handler instances ------------------------------------------------------------------
class _Shared:
    def __init__(self, value: Any, closer: Callable[[Any], None]):
        self.value, self.closer, self.refs = value, closer, 0


_registry: dict = {}
_registry_lock = threading.Lock()


def acquire_shared(key: Hashable, factory: Callable[[], Any], closer: Callable[[Any], None]) -> Any:
    """One object per key for the whole process (e.g. one WhisperEngine + batcher per (model, dtype, device)),
    reference-counted: the first acquire builds it, the last release closes it."""
    with _registry_lock:
        ent = _registry.get(key)
        if ent is None:
            ent = _registry[key] = _Shared(factory(), closer)
        ent.refs += 1
        return ent.value


def release_shared(key: Hashable) -> None:
    with _registry_lock:
        ent = _registry.get(key)
        if ent is None:
            return
        ent.refs -= 1
        if ent.refs <= 0:
            del _registry[key]
            ent.closer(ent.value)
