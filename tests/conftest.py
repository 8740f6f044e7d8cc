import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def port_oracle():
    from oracle.oracle_py import PortOracle
    return PortOracle()


@pytest.fixture(scope="session")
def _ref_session():
    """(live RefOracle or None, recorded calls, record path or None); see tests/ref_calls.py"""
    from oracle.oracle_py import RefOracle
    from tests import ref_calls
    path = os.environ.get("NPH_REF_RECORD")
    live = RefOracle() if RefOracle.available() else None
    if path and live is None:
        pytest.fail("NPH_REF_RECORD needs the compiled reference (oracle/_ref/libnpref.so)")
    calls = ref_calls.load()
    yield live, calls, path
    if path:
        ref_calls.save(calls, path)


@pytest.fixture
def ref_oracle(request, _ref_session):
    """The compiled reference: live where oracle/_ref/libnpref.so exists, else its recorded answers for this test."""
    from tests import ref_calls
    live, calls, path = _ref_session
    key = ref_calls.test_key(request.node)
    if path:
        calls[key] = []
        return ref_calls.Recorder(live, calls[key])
    if live is not None:
        return live
    if key not in calls:
        pytest.fail(f"no recorded reference answers for {key} (tests/golden/ref_calls.pkl.xz)")
    return ref_calls.Replay(key, calls[key])


@pytest.fixture(scope="session")
def engine():
    """One context on cuda:0 through the C ABI. No fallback: a missing library or device is an error."""
    from nanopolish_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()
