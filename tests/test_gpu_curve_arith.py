"""GPU: the curve harness (tests/device/curve_harness.cu) in its three device builds -- the library's compact layout, the same with
the by-reference Fp2 product (the layout b2k_g2.cu builds the G2 formulas in), and the inlined layout -- on the case list of
tests/curve_cases.py against the oracles.  test_curve_arith_emulation.py checks the same list on the host-emulated twin, so a
case that fails here only is a code-generation finding; a failure names the group, the operation, the aliasing, the layout and
the operands.  One more test drives the GLV split's boundary scalars through the library's own entry points."""
import ctypes
import os

import pytest

import curve_cases as cc
from kyber_b200 import workload as wl
from oracle import bls12381 as o

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUTS = ["compact", "byref", "inlined"]


@pytest.fixture(scope="module", params=LAYOUTS)
def harness(request):
    so = os.path.join(ROOT, "tests", "device", f"libcurve_harness_{request.param}.so")
    assert os.path.exists(so), f"{so} is missing: build() compiles it"
    return request.param, ctypes.CDLL(so)


# the inlined build holds the BLS12-381 G1 family only (curve_harness.cu: the group the library compiles in that layout)
LAYOUT_FAMILIES = {"inlined": ["w_bls381_g1"]}


@pytest.mark.parametrize("family", cc.families())
def test_curve_operations_on_the_device(harness, family):
    layout, lib = harness
    if family not in LAYOUT_FAMILIES.get(layout, cc.families()):
        pytest.skip(f"the {layout} build does not hold {family}")
    failures = cc.run_family(lib, family, layout, device=True)
    assert not failures, "\n".join(failures)


def test_case_counts(harness, capsys):
    """prints the number of cases per (family, operation, layout)"""
    layout, _ = harness
    counts = cc.case_counts(device=True)
    with capsys.disabled():
        for fam in cc.families():
            print(f"\n[{layout}] {fam}: " + ", ".join(f"{op} {n}" for (f, op), n in counts.items() if f == fam), end="")


def test_glv_boundary_scalars_through_the_abi(engine):
    """bls12381_g1_mul_batch and bls12381_g1_msm on the split's edge scalars, with the endomorphism split on and off: every product
    and the sum are the oracle's"""
    ks = cc.GLV_EDGES + [0, 1, 2, o.R - 1, o.R - 2, o.R - cc.X2 // 2, o.R - cc.X2 // 2 - 1, cc.X2 // 2 - 1]
    ks += [q * cc.X2 + cc.X2 // 2 + d for q in (1, 3, (1 << 126) + 5) for d in (-1, 0, 1)]
    ks = [k % o.R for k in ks]
    a = wl.prng_scalars("b2k/curve-glv-points", len(ks), o.R)
    pts = [o.g1_mul(x) for x in a]
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    sb = wl.scalars_to_bytes(ks)
    want_mul = b"".join(o.g1_compress(o.g1_mul(k * x % o.R)) for k, x in zip(ks, a))
    want_msm = o.g1_compress(o.g1_mul(wl.dot_mod(ks, a, o.R)))
    for glv in (True, False):
        engine.set_msm_glv(glv)
        try:
            got_mul = engine.bls12381_g1_mul_batch(sb, pb)
            got_msm = engine.bls12381_g1_msm(sb, pb)
        finally:
            engine.set_msm_glv(True)
        for i in range(len(ks)):
            assert got_mul[48 * i:48 * (i + 1)] == want_mul[48 * i:48 * (i + 1)], (glv, hex(ks[i]))
        assert got_msm == want_msm, glv
