"""CPU: the restatement of the reference's Point.Mul (geScalarMult, ge.go:443-502) that the edwards25519 MSM tests use as
their expected value: equal to the plain product below 2^255, different exactly where the top digit exceeds 8, and still
reproducing the reference's Diffie-Hellman KAT (examples/dh_test.go:17-49)."""
import random

import pytest

from oracle import ed25519 as ed
import ed25519_msm_cases as cases


def _b(k: int) -> bytes:
    return k.to_bytes(32, "little")


POINTS = [ed.BASE, ed.scalar_mult(987654321), ed.decode(cases.T8), ed.decode(cases.mixed_point(5)), ed.decode(cases.ZERO)]


def test_equals_the_plain_product_below_2_255():
    rng = random.Random(11)
    ks = [0, 1, 2, 8, 9, 15, 16, ed.L - 1, ed.L, ed.L + 1, (1 << 252) - 1, 1 << 252, (1 << 255) - 1]
    ks += [rng.getrandbits(255) for _ in range(40)]
    for k in ks:
        assert cases.top_digit(k) <= 8
        for pt in POINTS:
            assert cases.ge_scalar_mult(_b(k), pt) == ed.scalar_mult(k, pt), hex(k)


@pytest.mark.parametrize("e63", [9, 16])
def test_a_top_digit_above_8_is_dropped(e63):
    rng = random.Random(e63)
    ks = [k for k in cases.crafted_high_scalars(rng) if cases.top_digit(k) == e63]
    assert ks
    for k in ks:
        assert k >= 1 << 255
        for pt in POINTS[:4]:
            got = cases.ge_scalar_mult(_b(k), pt)
            assert got == ed.scalar_mult(k - (e63 << 252) + 8 * ed.L, pt)
            assert got == ed.scalar_mult(cases.effective_scalar(k), pt)
        assert cases.ge_scalar_mult(_b(k), ed.BASE) != ed.scalar_mult(k, ed.BASE), hex(k)


def test_0x8f_with_and_without_a_carry_into_nibble_62():
    rng = random.Random(3)
    without = (0x8f << 248) | rng.getrandbits(236)              # nibble 61 < 8: nothing carries into nibble 62
    with_c = (0x8f << 248) | (0xf0 << 240) | rng.getrandbits(236)
    assert cases.nibbles(_b(without))[62] == -1 and cases.nibbles(_b(with_c))[62] == 0
    for k in (without, with_c):
        assert cases.top_digit(k) == 9
        got = cases.ge_scalar_mult(_b(k), ed.BASE)
        assert got == ed.scalar_mult((k - (9 << 252)) % (8 * ed.L), ed.BASE)
        assert got != ed.scalar_mult(k, ed.BASE)


def test_closed_form_top_digit_matches_the_carry_pass():
    rng = random.Random(4)
    for k in cases.crafted_high_scalars(rng) + [rng.getrandbits(256) for _ in range(2000)] + [0, (1 << 256) - 1]:
        assert cases.top_digit_fast(k) == cases.top_digit(k), hex(k)


def test_top_digit_8_is_kept():
    for k in cases.crafted_high_scalars(random.Random(8)):
        if cases.top_digit(k) == 8:
            assert cases.ge_scalar_mult(_b(k), POINTS[1]) == ed.scalar_mult(k, POINTS[1])
            assert cases.effective_scalar(k) == k


def test_reference_dh_kat_through_ge_scalar_mult():
    rng = ed.Blake2Xb(b"")
    a, b = ed.pick_scalar(rng), ed.pick_scalar(rng)
    A = cases.ge_scalar_mult(a, ed.BASE)
    B = cases.ge_scalar_mult(b, ed.BASE)
    s1, s2 = cases.ge_scalar_mult(a, B), cases.ge_scalar_mult(b, A)
    assert s1 == s2
    assert ed.encode(s1).hex() == "80ea238cacfdab279626970bba18c69083c7751865dec4c6434bff4351282847"


def test_identity_and_the_all_zero_encoding():
    assert cases.IDENTITY == bytes([1]) + bytes(31)
    z = ed.decode(cases.ZERO)
    assert z is not None and z != ed.IDENT
    assert ed.scalar_mult(4, z) == ed.IDENT and ed.scalar_mult(2, z) != ed.IDENT
