"""Where the tests find the upstream huggingface/speech-to-speech source tree (its `src` directory).

The drop-in tests subclass, register into and drive the upstream handler classes themselves, so they need that tree.
It is looked up, in order, from
  1. the environment variable S2S_REFERENCE_SRC;
  2. a checkout named `reference` beside this repository or beside one of its parent directories (`<dir>/reference/src`).
`reference_src()` returns "" when none is found; the tests that need the tree then skip.
"""
from __future__ import annotations

import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _is_upstream_src(path: str) -> bool:
    return bool(path) and os.path.isfile(os.path.join(path, "speech_to_speech", "baseHandler.py"))


def reference_src() -> str:
    env = os.environ.get("S2S_REFERENCE_SRC", "")
    if env:
        return env if _is_upstream_src(env) else ""
    d = ROOT
    while True:
        parent = os.path.dirname(d)
        cand = os.path.join(parent, "reference", "src")
        if _is_upstream_src(cand):
            return cand
        if parent == d:
            return ""
        d = parent
