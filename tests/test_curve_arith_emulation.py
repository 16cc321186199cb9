"""CPU tests: the curve harness (tests/device/curve_harness.cu) compiled by g++ with the emulated carry chains of ptx.cuh, on the
full case list of tests/curve_cases.py against the oracles.  test_gpu_curve_arith.py runs the same list on the three device
builds, so a case that passes here and fails there is a code-generation difference, not a formula one."""
import ctypes
import os
import subprocess

import pytest

import curve_cases as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "device", "curve_harness.cu")


@pytest.fixture(scope="module")
def twin():
    so = os.path.join(EMU, "libemul_curve_harness.so")
    newest = max([os.path.getmtime(SRC)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", "-x", "c++", SRC,
                        "-o", so], check=True)
    return ctypes.CDLL(so)


@pytest.mark.parametrize("family", cc.families())
def test_curve_operations_match_the_oracles(twin, family):
    failures = cc.run_family(twin, family, "host", device=False)
    assert not failures, "\n".join(failures)


REQUIRED = {
    "w_bls381_g1": set(cc.W_OPS) - {"jac_psi", "clear_cofactor"},
    "w_bls381_g2": set(cc.W_OPS) - {"glv_split", "scalar_mul_glv", "fp_from_64_bytes"},
    "xmd": set(cc.XMD_OPS),
    "ed": set(cc.ED_OPS),
}
GENERIC = set(cc.W_OPS[:cc.W_OPS.index("jac_mul_xabs")])


def test_case_counts(capsys):
    """every operation of the issue's list has cases in every family that has it; prints the count per (family, operation)"""
    counts = cc.case_counts(device=True)
    for fam in cc.families():
        want = REQUIRED.get(fam, GENERIC)
        have = {op for (f, op) in counts if f == fam}
        assert want <= have, (fam, sorted(want - have))
    with capsys.disabled():
        for fam in cc.families():
            print(f"\n{fam}: " + ", ".join(f"{op} {n}" for (f, op), n in counts.items() if f == fam), end="")


def test_operand_classes_are_present():
    """the binary operations see P + P and P + (-P) at different scales, infinity in each slot, and a Jacobian infinity other
    than (1, 1, 0); the edwards25519 lists hold the 8-torsion, the 19 non-canonical y and the identity with the sign bit"""
    for name in cc.GROUPS:
        g = cc.GROUPS[name]
        add = next(b for b in cc.w_batches(name) if b.op == "jac_add" and b.alias == 0)
        ops = [c.operands for c in add.cases]
        assert any(a == b and a != "inf" and s == "rescaled" for a, b, s in ops)
        assert any(a != "inf" and b != "inf" and cc.fmt(g.neg(eval_pt(a, g))) == b for a, b, _ in ops[:40])
        assert any(a == "inf" for a, _, _ in ops) and any(b == "inf" for _, b, _ in ops) and ("inf", "inf", "rescaled") in ops
        one = g.F.enc(g.F.one)
        E4 = 4 * g.F.n * g.F.deg
        assert any(c.row[2 * E4:3 * E4] == bytes(E4) and c.row[:E4] != one for c in add.cases)
    assert len(cc.ed_torsion()) == 8 and len(set(cc.ed_torsion())) == 8
    encs = cc.ed_bytes_cases(__import__("random").Random(0))
    ys = {int.from_bytes(e, "little") & ((1 << 255) - 1) for e in encs}
    assert {cc.ed.P + j for j in range(19)} <= ys
    assert (1 | (1 << 255)).to_bytes(32, "little") in encs


def eval_pt(s, g):
    """the point a failure message prints, back as a tuple (only for the operand-class check above)"""
    for P in cc.pools(g.name)[0] + cc.pools(g.name)[1] + cc.pools(g.name)[2]:
        if cc.fmt(P) == s:
            return P
    return None


def test_glv_split_restatement_recombines():
    """the Python restatement the device split is compared with: k = +-k1 +- k2 x^2 (mod r), |k1| <= x^2 / 2, k2 < 2^128"""
    for b in cc.w_batches("bls381_g1"):
        if b.op != "glv_split":
            continue
        for c in b.cases:
            k = int(c.operands[0], 16)
            k1, k2, n1, n2 = cc.glv_split(k)
            assert ((-1) ** n1 * k1 + (-1) ** n2 * k2 * cc.X2 - k) % cc.o.R == 0, hex(k)
            assert 2 * k1 <= cc.X2 and k2 < 1 << 128
