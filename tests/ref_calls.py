"""The compiled reference's answers as recorded data (tests/golden/ref_calls.pkl.xz).

Every test that compares with the compiled reference (oracle/_ref/libnpref.so) asks it through the `ref_oracle` fixture.
Where that library exists the fixture is the live RefOracle.  Elsewhere it is a Replay: the i-th call a test makes returns the
i-th answer the reference gave to that same test when it was recorded, so the comparison still runs against the reference's
own output.  The inputs of these tests are seeded, so a test asks the same questions in the same order every time; the
replay checks the method name of every call and fails on a test it holds no record for.

Recording: run the tests with NPH_REF_RECORD=<path> where the reference is built; the recorded calls of the tests that ran
are merged into the committed file and written to <path>.
"""
from __future__ import annotations

import copy
import lzma
import os
import pickle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_calls.pkl.xz")


def test_key(node) -> str:
    return f"{os.path.basename(str(node.fspath))}::{node.name}"


def load(path: str = GOLDEN) -> dict:
    if not os.path.exists(path):
        return {}
    with lzma.open(path, "rb") as f:
        return pickle.load(f)


def save(calls: dict, path: str) -> None:
    with lzma.open(path, "wb", preset=9) as f:
        pickle.dump(calls, f, protocol=4)


class Recorder:
    """Forwards every call to the live oracle and appends (name, answer) to `log`."""

    def __init__(self, target, log: list, prefix: str = ""):
        self._target, self._log, self._prefix = target, log, prefix

    def __getattr__(self, name):
        attr = getattr(self._target, name)
        if name == "lib":
            return Recorder(attr, self._log, "lib.")
        if not callable(attr):
            return attr

        def call(*args, **kwargs):
            try:
                out = attr(*args, **kwargs)
            except Exception as ex:
                self._log.append((self._prefix + name, ex))
                raise
            self._log.append((self._prefix + name, copy.deepcopy(out)))
            return out
        return call


class Replay:
    """Answers a test's calls, in order, from the record of that test."""

    def __init__(self, key: str, log: list, prefix: str = "", pos: list | None = None):
        self._key, self._log, self._prefix = key, log, prefix
        self._pos = pos if pos is not None else [0]

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        if name == "lib":
            return Replay(self._key, self._log, "lib.", self._pos)

        def call(*args, **kwargs):
            i = self._pos[0]
            if i >= len(self._log):
                raise AssertionError(f"{self._key}: call {i} ({self._prefix}{name}) is beyond the {len(self._log)} recorded calls")
            want, out = self._log[i]
            if want != self._prefix + name:
                raise AssertionError(f"{self._key}: call {i} is {self._prefix}{name}, the record has {want}")
            self._pos[0] = i + 1
            if isinstance(out, Exception):
                raise out
            return copy.deepcopy(out)
        return call
