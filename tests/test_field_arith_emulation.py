"""CPU tests: the field harness (tests/device/field_harness.cu) compiled by g++ with the emulated carry chains of ptx.cuh, on the
full case list of tests/field_cases.py against Python integers.  test_gpu_field_arith.py runs the same list on the three device
builds, so a case that passes here and fails there is a code-generation difference, not a limb-algorithm one."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import field_cases as fc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "device", "field_harness.cu")


@pytest.fixture(scope="module")
def twin():
    so = os.path.join(EMU, "libemul_field_harness.so")
    newest = max([os.path.getmtime(SRC)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cuh")])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", "-x", "c++", SRC,
                        "-o", so], check=True)
    return ctypes.CDLL(so)


def run_batches(lib, batches):
    failures = []
    for b in batches:
        got = fc.call(lib, b.kind, b.target, b.opcode, b.alias, b.inp, len(b.operands), b.out_words)
        count, msgs = fc.mismatches(b, got)
        if count:
            failures.append(f"{count} wrong: " + "\n  ".join(msgs))
    return failures


@pytest.mark.parametrize("field", [f.name for f in fc.FIELDS])
def test_field_operations_match_python(twin, field):
    failures = run_batches(twin, fc.fp_batches(field))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("tower", list(fc.TOWERS))
def test_tower_operations_match_the_oracles(twin, tower):
    failures = run_batches(twin, fc.tw_batches(tower))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("tower", list(fc.TOWERS))
def test_frobenius_is_the_power_p_k(twin, tower):
    """the device map against x^(p^k) by square-and-multiply (the tower tests use the oracle's conjugate-and-twist form)"""
    tw = fc.TOWERS[tower]
    for A, k, want in fc.frobenius_by_power(tower):
        inp = fc.pack(A + [0] * 12, tw.n)
        got = fc.call(twin, "tw", tower, fc.TW_OPS.index(f"f12_frob{k}"), 0, inp, 1, 12 * tw.n + 1)
        assert fc.unpack(got[:12 * tw.n], tw.n) == want, (tower, k, [hex(x) for x in A])


def test_case_volume():
    """the grid holds every edge pair and 2000 random cases per binary operation; one launch per field has 64K inversions"""
    for f in fc.FIELDS:
        batches = fc.fp_batches(f.name)
        E = fc.edges(f)
        mul = next(b for b in batches if b.op == "mul" and b.alias == 0)
        assert len(mul.operands) >= len(E) ** 2 + 2000
        assert max(len(b.operands) for b in batches if b.op == "inv") >= 65536
        assert {f.p - 1, f.p - 2, 0, 1, (f.p + 1) // 2} <= set(E)
