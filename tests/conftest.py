import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a; run with -m gpu)")
    # tests/test_emulated_gpu_suite.py re-runs the gpu-marked parity tests on the CPU box in a child pytest whose
    # package is pointed at the emulated build of the library (tests/simt/library_emul.cc). Test infrastructure only:
    # the variable is read here, never by the package.
    emulated = os.environ.get("AMB_TEST_EMULATED_LIB")
    if emulated:
        from gr_air_modes_b200 import _lib
        _lib.LIB_PATH, _lib._lib = emulated, None


@pytest.fixture(scope="session")
def port():
    from oracle import cpu_oracle
    return cpu_oracle.Port()


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference's answers, from tests/golden/ref_calls.json.gz (tests/ref_golden.py). AMB_RECORD_REF=1:
    from the live reference objects (oracle/_ref), and the record is rewritten at the end of the session."""
    from ref_golden import GoldenRef
    if not os.environ.get("AMB_RECORD_REF"):
        yield GoldenRef()
        return
    from oracle import cpu_oracle
    if not cpu_oracle.ref_available():
        pytest.fail("AMB_RECORD_REF: oracle/_ref is not built (it needs the reference sources)")
    rec = GoldenRef(cpu_oracle.Ref())
    yield rec
    rec.save()


@pytest.fixture(scope="session")
def ref_py():
    """The reference's Python modules' answers, from tests/golden/ref_python.json.gz (tests/ref_golden.py).
    AMB_RECORD_REF=1: from the live modules, and the record is rewritten at the end of the session."""
    from ref_golden import PythonRecord
    rec = PythonRecord(live=bool(os.environ.get("AMB_RECORD_REF")))
    yield rec
    if rec.live:
        rec.save()
