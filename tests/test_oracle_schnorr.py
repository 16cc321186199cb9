"""CPU: the sign/schnorr oracle (tests/schnorr_oracle.py) against the properties the device code relies on."""
import hashlib

import pytest

from oracle import bls12381 as bls
from oracle import eddsa as oe
import schnorr_cases as cases
import schnorr_oracle as so


def test_edwards25519_signatures_pass_the_pinned_eddsa_verifier():
    """sign/schnorr and sign/eddsa accept the same signatures on edwards25519 (TestEdDSACompatibility)"""
    n = 0
    for name, pk, msg, sig in cases.ed_cases():
        st = so.verify_with_checks("ed25519", pk, msg, sig)
        if st == oe.OK:
            assert oe.verify_with_checks(pk, msg, sig) == oe.OK, name
            n += 1
        if oe.verify_with_checks(pk, msg, sig) == oe.OK:
            assert st == oe.OK, name
    assert n >= 15


@pytest.mark.parametrize("group", so.GROUPS)
def test_honest_signatures_verify_and_lengths_are_refused(group):
    for name, pk, msg, sig in cases.cases(group):
        if name.startswith("honest"):
            assert so.verify_with_checks(group, pk, msg, sig) == (oe.OK if group == "ed25519" else so.OK), name
    want = oe.SIG_LENGTH if group == "ed25519" else so.LENGTH
    for name, pk, msg, sig in cases.length_cases(group):
        assert so.verify_with_checks(group, pk, msg, sig) == want, name


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_every_status_occurs_and_the_order_is_the_references(group):
    st = {name: so.verify_with_checks(group, pk, msg, sig) for name, pk, msg, sig in cases.cases(group)}
    assert set(st.values()) == {so.OK, so.R_BAD, so.S_BAD, so.PK_BAD, so.INVALID}
    assert st["s + r"] == so.S_BAD                     # malleability: s + r is refused by mod.Int's range check
    assert st["R bad and s >= r"] == so.R_BAD          # R before s
    assert st["s >= r and key bad"] == so.S_BAD        # s before the key
    for name, _ in cases.bad_encodings(group):
        assert st["R: " + name] == so.R_BAD and st["key: " + name] == so.PK_BAD and st["R and key: " + name] == so.R_BAD
    assert st["R, s, key = O, 0, O"] == so.OK and st["key infinity"] == so.OK and st["R infinity"] == so.OK
    assert st["s = r - 1, key infinity, R = -B"] == so.OK


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_decodable_encodings_are_their_own_re_encoding(group):
    """why the device may hash the input bytes of R and the key instead of MarshalTo: every accepted encoding re-encodes
    to itself, and every case that reaches the equation hashes to the same challenge either way"""
    decode = so._BLS[group][0]
    pl = so.POINT_LEN[group]
    n = 0
    for name, pk, msg, sig in cases.cases(group):
        for enc in (pk, sig[:pl]):
            try:
                pt = decode(enc)
            except ValueError:
                continue
            assert so.encode(group, pt) == enc, name
            n += 1
    assert n > 80


def test_challenge_reduction_is_big_endian_mod_r():
    for i in range(200):
        d = hashlib.sha512(b"%d" % i).digest()
        assert so.reduce_be(d) == int.from_bytes(d, "big") % bls.R
    assert so.reduce_be(b"\xff" * 64) == (2 ** 512 - 1) % bls.R
    assert so.reduce_be((bls.R * 2 ** 256).to_bytes(64, "big")) == 0
