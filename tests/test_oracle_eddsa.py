"""CPU: the Ed25519 oracle (oracle/eddsa.py) against the reference's fixtures -- RFC 8032, sign.input, Wycheproof, the byte
vectors of eddsa_test.go and the small-order list of const.go."""
import pytest

from oracle import ed25519 as ed
from oracle import eddsa as oe
import eddsa_cases as cases

NAME_TO_CODE = {v: k for k, v in oe.ERR_NAMES.items()}


def test_oracle_signs_rfc8032_and_sign_input_to_the_fixture_bytes():
    vecs = cases.rfc8032() + cases.sign_input()
    assert len(vecs) == 5 + 1024
    for seed, pk, msg, sig in vecs:
        assert oe.keygen(seed)[2] == pk
        assert oe.sign(seed, msg) == sig


def test_verify_accepts_every_valid_vector():
    for _, pk, msg, sig in cases.rfc8032() + cases.sign_input():
        assert oe.verify_with_checks(pk, msg, sig) == oe.OK


def test_verify_agrees_with_wycheproof():
    wp = cases.wycheproof()
    assert len(wp) == 150 and sum(v for *_, v in wp) == 88
    for tc, pk, msg, sig, valid in wp:
        assert (oe.verify_with_checks(pk, msg, sig) == oe.OK) == valid, tc


def test_inline_vectors_give_the_error_their_test_expects():
    inl = cases.inline()
    assert len(inl) == 6
    for name, pk, msg, sig, expect in inl:
        assert oe.verify_with_checks(pk, msg, sig) == NAME_TO_CODE[expect], name


def test_small_order_encodings_derived_from_the_curve_equal_the_reference_list():
    derived = [y.to_bytes(32, "little") for y in oe.small_order_ys()]
    assert sorted(derived) == sorted(cases.weak_keys())
    t8 = oe.order8_point()
    assert ed.scalar_mult(8, t8) == ed.IDENT and ed.scalar_mult(4, t8) != ed.IDENT


@pytest.mark.parametrize("kind", ["non-canonical", "no sqrt", "small order"])
def test_crafted_point_rejections_map_to_their_codes(kind):
    codes = {"non-canonical": (oe.R_NOT_CANONICAL, oe.PK_NOT_CANONICAL), "no sqrt": (oe.R_INVALID, oe.PK_INVALID),
             "small order": (oe.R_SMALL_ORDER, oe.PK_SMALL_ORDER)}[kind]
    seen = 0
    for name, pk, msg, sig in cases.crafted():
        if kind in name:
            assert oe.verify_with_checks(pk, msg, sig) == codes[0 if name.startswith("R ") else 1], name
            seen += 1
    assert seen >= 4


def test_cofactorless_equation():
    got = [(oe.verify_with_checks(pk, msg, sig), h8) for _, pk, msg, sig, h8 in cases.cofactor_cases()]
    assert any(h8 == 0 for _, h8 in got) and sum(h8 != 0 for _, h8 in got) >= 8
    for code, h8 in got:
        assert code == (oe.OK if h8 == 0 else oe.NOT_EQUAL)
