"""GPU: the field harness (tests/device/field_harness.cu) in its three device builds -- the library's compact layout, the same with
the by-reference Fp2 product, and the inlined layout -- on the case list of tests/field_cases.py, case by case against Python
integers.  test_field_arith_emulation.py checks the same list on the host-emulated twin, so together they assert device ==
emulation for every case; a failure names the field or tower, the operation, the aliasing, the layout and the operands."""
import ctypes
import os

import pytest

import field_cases as fc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUTS = ["compact", "byref", "inlined"]


@pytest.fixture(scope="module", params=LAYOUTS)
def harness(request):
    so = os.path.join(ROOT, "tests", "device", f"libfield_harness_{request.param}.so")
    assert os.path.exists(so), f"{so} is missing: build() compiles it"
    return request.param, ctypes.CDLL(so)


def check(harness, batches):
    layout, lib = harness
    failures = []
    for b in batches:
        got = fc.call(lib, b.kind, b.target, b.opcode, b.alias, b.inp, len(b.operands), b.out_words)
        count, msgs = fc.mismatches(b, got)
        if count:
            failures.append(f"[{layout}] {count} of {len(b.operands)} wrong:\n  " + "\n  ".join(msgs))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("field", [f.name for f in fc.FIELDS])
def test_field_operations_on_the_device(harness, field):
    check(harness, fc.fp_batches(field))


@pytest.mark.parametrize("tower", list(fc.TOWERS))
def test_tower_operations_on_the_device(harness, tower):
    check(harness, fc.tw_batches(tower))


@pytest.mark.parametrize("tower", list(fc.TOWERS))
def test_frobenius_is_the_power_p_k_on_the_device(harness, tower):
    layout, lib = harness
    tw = fc.TOWERS[tower]
    for A, k, want in fc.frobenius_by_power(tower):
        got = fc.call(lib, "tw", tower, fc.TW_OPS.index(f"f12_frob{k}"), 0, fc.pack(A + [0] * 12, tw.n), 1, 12 * tw.n + 1)
        assert fc.unpack(got[:12 * tw.n], tw.n) == want, (layout, tower, k, [hex(x) for x in A])


def test_case_counts(harness, capsys):
    """prints the number of cases per (field or tower, operation, layout)"""
    layout, _ = harness
    with capsys.disabled():
        for name in [f.name for f in fc.FIELDS]:
            counts = {}
            for b in fc.fp_batches(name):
                counts[b.op] = counts.get(b.op, 0) + len(b.operands)
            print(f"\n[{layout}] {name}: " + ", ".join(f"{k} {v}" for k, v in counts.items()), end="")
        for name in fc.TOWERS:
            counts = {}
            for b in fc.tw_batches(name):
                counts[b.op] = counts.get(b.op, 0) + len(b.operands)
            print(f"\n[{layout}] {name}: " + ", ".join(f"{k} {v}" for k, v in counts.items()), end="")
