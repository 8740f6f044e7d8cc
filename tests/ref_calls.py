"""The compiled reference's answers as recorded data (tests/golden/ref_calls.pkl.xz).

Every test that compares with the compiled reference (oracle/_ref/libnpref.so) asks it through the `ref_oracle` fixture.
Where that library exists the fixture is the live RefOracle.  Elsewhere it is a Replay: the i-th call a test makes returns the
i-th answer the reference gave to that same test when it was recorded, so the comparison still runs against the reference's
own output.  The inputs of these tests are seeded, so a test asks the same questions in the same order every time; the
replay checks the method name of every call and fails on a test it holds no record for.

Recording: run the tests with NPH_REF_RECORD=<path> where the reference is built; the recorded calls of the tests that ran
are merged into the committed file and written to <path>.

The edge suites (test_*_edges_oracle.py) keep the reference's answers per case instead, in one CaseRecord per suite
(tests/golden/ref_*_edges.pkl.xz), keyed by a fingerprint of each case's inputs so that the GPU suites can look them up
too (case_answers).  A suite may ask another reference library (the tail callers' oracle/_ref/libnpref_polya.so and
libnpref_polyi.so) by giving case_fixture its own `ref`.  NPH_REF_CASES_RECORD=<dir> pytest <edge suites> writes a new record of
every suite that ran to <dir>.
"""
from __future__ import annotations

import copy
import lzma
import os
import pickle
import signal

import numpy as np
import pytest

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = os.path.join(GOLDEN_DIR, "ref_calls.pkl.xz")
ASSERTS = "asserts"


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


def forked(fn):
    """fn() in a forked child: its pickled result, or ASSERTS if the child died of SIGABRT (the reference aborts the process
    on a failed assert)"""
    rd, wr = os.pipe()
    pid = os.fork()
    if pid == 0:
        os.close(rd)
        try:
            data = pickle.dumps(fn())
            with os.fdopen(wr, "wb") as f:
                f.write(data)
        finally:
            os._exit(0)
    os.close(wr)
    with os.fdopen(rd, "rb") as f:
        data = f.read()
    _, st = os.waitpid(pid, 0)
    if os.WIFSIGNALED(st) and os.WTERMSIG(st) == signal.SIGABRT:
        return ASSERTS
    assert os.WIFEXITED(st) and data, f"reference child ended with status {st}"
    return pickle.loads(data)


def same(a, b) -> bool:
    """a equals b bit for bit, through tuples, lists, numpy arrays and numpy scalars"""
    if isinstance(a, (tuple, list)) or isinstance(b, (tuple, list)):
        return isinstance(a, (tuple, list)) and isinstance(b, (tuple, list)) and len(a) == len(b) and all(map(same, a, b))
    if isinstance(a, (np.ndarray, np.generic)) or isinstance(b, (np.ndarray, np.generic)):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return type(a) is type(b) and a == b


class CaseRecord:
    """The compiled reference's answers to one edge suite's cases, kept in tests/golden/<name> as {key: [row per case]}, a row
    being (fingerprint of the case's inputs, answer), or (fingerprint, *answer) where a suite's rows are flat.  Three modes:
      record  NPH_REF_CASES_RECORD=<dir>: every case is asked of the reference, which must exist and export every entry point
              in `needs`, and the rows are written to <dir>/<name> at the end of the module;
      live    the reference exists and exports `needs`: every case is asked of it, and the fingerprints and answers must equal
              the record's, so a stale record fails here and not only where it is replayed;
      replay  otherwise (no library, or one built from an older harness): the record's answers, whose fingerprints must equal
              the cases'."""

    def __init__(self, name: str, needs=(), ref=None):
        """ref: where the suite asks another library than oracle/_ref/libnpref.so, a callable returning its live handle, or
        None where that library is not built"""
        self.path = os.path.join(GOLDEN_DIR, name)
        out = os.environ.get("NPH_REF_CASES_RECORD")
        if ref is None:
            from oracle.oracle_py import RefOracle
            self.live = RefOracle() if RefOracle.available() else None
            if self.live is not None and not all(self.live.has(e) for e in needs):
                self.live = None
            what = f"the compiled reference (oracle/_ref/libnpref.so) exporting {list(needs)}"
        else:
            self.live = ref()
            what = f"the compiled reference {getattr(ref, '__doc__', None) or ''}".rstrip()
        if out and self.live is None:
            pytest.fail(f"NPH_REF_CASES_RECORD needs {what}")
        self.out = os.path.join(out, name) if out else None
        self.rows = {} if out else load(self.path)

    def answers(self, key: str, fingerprints: list, ask, skip: dict | None = None, fork: bool = False, flat: bool = False) -> list:
        """The reference's answer to every case, in order.  ask(i) asks the live reference about case i; while recording with
        `fork` it runs in a forked child, and a child the reference aborts answers ASSERTS.  `skip` maps the cases never sent
        to the reference to the answer recorded for them."""
        skip = skip or {}
        n = len(fingerprints)
        if self.live is not None:
            got = [skip[i] if i in skip else forked(lambda i=i: ask(i)) if fork and self.out else ask(i) for i in range(n)]
            if self.out:
                self.rows[key] = [(fp, *a) if flat else (fp, a) for fp, a in zip(fingerprints, got)]
                return got
        rows = self.rows.get(key)
        assert rows is not None and len(rows) == n, f"no recorded reference answers for {key} ({self.path}); re-record"
        want = []
        for i, (fp, *a) in enumerate(rows):
            assert fp == fingerprints[i], f"{key}, case {i}: inputs differ from the recorded ones; re-record"
            want.append(tuple(a) if flat else a[0])
        if self.live is None:
            got = [skip.get(i, want[i]) for i in range(n)]
        bad = [i for i in range(n) if not same(got[i], want[i])]
        assert not bad, f"{key}: the reference's answers to cases {bad[:5]} ({len(bad)} in all) differ from the record {self.path}"
        return got

    @property
    def recording(self) -> bool:
        return self.out is not None


def case_fixture(name: str, needs=(), ref=None):
    """a module-scoped fixture holding the CaseRecord of tests/golden/<name>; while recording it writes the record at the end"""
    def fixture():
        rec = CaseRecord(name, needs, ref)
        yield rec
        if rec.out:
            os.makedirs(os.path.dirname(rec.out), exist_ok=True)
            save(rec.rows, rec.out)
    return pytest.fixture(scope="module")(fixture)


def case_answers(name: str, key: str) -> dict:
    """{fingerprint: answer} of the rows recorded under `key` in tests/golden/<name>"""
    rows = load(os.path.join(GOLDEN_DIR, name)).get(key)
    assert rows is not None, f"no recorded reference answers for {key} (tests/golden/{name})"
    return {fp: (tuple(a) if len(a) > 1 else a[0]) for fp, *a in rows}
