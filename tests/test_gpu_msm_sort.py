"""GPU parity of the MSM's bucket sort (kyber_b200/csrc/msm_sort.cuh) at sizes where it runs the paths that the 2000-pair sets of
test_gpu_msm_curves.py never reach: partition tiles by the hundred, bin-sort tiles that share one coarse bin, and buckets millions
of entries deep.  BLS12-381 G1 at 2^20 pairs (GLV split on, through the chunked host-buffer front end, and off), BLS12-381 G2 and
bn254 G1 at 2^16, each with uniform scalars, one (s, P) repeated n times, and 128-bit BDN factors; expected values from the
oracle (tests/msm_cases.py)."""
import pytest

import msm_cases as mc

pytestmark = pytest.mark.gpu

ENTRY = {
    "bls12381_g1": ("b2k_bls12381_g1_msm", "b2k_bls12381_g1_mul_batch_affine"),
    "bls12381_g2": ("b2k_bls12381_g2_msm", "b2k_bls12381_g2_mul_batch_affine"),
    "bn254_g1": ("b2k_bn254_g1_msm", "b2k_bn254_g1_mul_batch"),
}
CASES = [("bls12381_g1", 1 << 20), ("bls12381_g2", 1 << 16), ("bn254_g1", 1 << 16)]
SETS = ("uniform", "equal", "bdn128")


@pytest.fixture(scope="module")
def operands(engine):
    """per group: multipliers A and the operands A_i G from the engine's fixed-base batch, a few re-checked against the oracle"""
    out = {}
    for group, n in CASES:
        g = mc.GROUPS[group]
        a = mc.multipliers(g, n)
        pts = engine.call_host(ENTRY[group][1], n, mc.scalars_to_bytes(a), g.gen * n, g.in_bytes * n)
        for i in (0, 1, n - 1):
            assert pts[g.in_bytes * i:g.in_bytes * (i + 1)] == g.operand(g.mul(a[i])), (group, i)
        out[group] = (a, pts)
    return out


@pytest.mark.parametrize("set_name", SETS)
@pytest.mark.parametrize("group,n", CASES)
def test_msm_sort_large(engine, operands, group, n, set_name):
    g = mc.GROUPS[group]
    A, base = operands[group]
    a, s = mc.build_set(g, set_name, n, A)
    if set_name == "equal":                       # one operand n times
        pts = base[:g.in_bytes] * n
    else:
        pts = base
    want = g.expected(a, s)
    sb = mc.scalars_to_bytes(s)
    glv_modes = (True, False) if group == "bls12381_g1" else (True,)
    try:
        for glv in glv_modes:
            engine.set_msm_glv(glv)
            got = engine.call_host(ENTRY[group][0], n, sb, pts, g.out_bytes)
            assert got == want, (group, n, set_name, glv)
    finally:
        engine.set_msm_glv(True)
