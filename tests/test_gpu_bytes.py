"""GPU: the byte and scalar harness (tests/device/bytes_harness.cu, built by build() with the library's flags) on the case list of
tests/bytes_cases.py against hashlib, hmac, Python integers and the oracles.  test_bytes_emulation.py checks the same list on
the host-compiled twin, so a case that fails here only is a code-generation finding; a failure names the operation, the
launch, the case class, the lane and the input."""
import ctypes
import os

import pytest

import bytes_cases as bc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness():
    so = os.path.join(ROOT, "tests", "device", "libbytes_harness.so")
    assert os.path.exists(so), f"{so} is missing: build() compiles it"
    return ctypes.CDLL(so)


@pytest.mark.parametrize("op", bc.OPS)
def test_bytes_ops_on_the_device(harness, op):
    failures = bc.run_all(harness, "device", [op])
    assert not failures, "\n".join(failures)


def test_case_counts(capsys):
    """prints the number of cases per (operation, class)"""
    counts = bc.case_counts()
    with capsys.disabled():
        print(f"\n{sum(counts.values())} cases")
        for op in bc.OPS:
            print(f"{op}: " + ", ".join(f"{cls} {n}" for (o, cls), n in counts.items() if o == op))
