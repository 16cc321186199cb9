"""CPU: static checks on the Go adapters' sign/schnorr bindings (go/pairing/bls12381/b200/schnorr.go and
go/group/edwards25519/b200/schnorr.go; no Go toolchain in the image): the entry points and status constants they use exist in
include/b2kyber.h, both BLS12-381 groups and edwards25519 are bound, the reference's error strings
(sign/schnorr/schnorr.go:89-183) are present, and the build tag is set."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLS = os.path.join(ROOT, "go", "pairing", "bls12381", "b200", "schnorr.go")
ED = os.path.join(ROOT, "go", "group", "edwards25519", "b200", "schnorr.go")
HDR = os.path.join(ROOT, "include", "b2kyber.h")


def _declared(hdr, sym):
    return re.search(r"\bint %s\(" % sym, hdr) or re.search(r"\b%s\b\s*=" % sym, hdr)


def test_bls_entry_points_and_statuses_are_bound():
    src, hdr = open(BLS).read(), open(HDR).read()
    for fn in ("b2k_bls12381_g1_schnorr_verify", "b2k_bls12381_g2_schnorr_verify"):
        assert "C.%s(" % fn in src, fn
        assert _declared(hdr, fn), fn
    for fn in ("b2k_bls12381_g1_schnorr_verify_dev", "b2k_bls12381_g2_schnorr_verify_dev"):
        assert _declared(hdr, fn), fn
    for st in ("B2K_SCHNORR_OK", "B2K_SCHNORR_R", "B2K_SCHNORR_S", "B2K_SCHNORR_PK"):
        assert "C." + st in src, st
    for st, v in (("B2K_SCHNORR_OK", 0), ("B2K_SCHNORR_R", 1), ("B2K_SCHNORR_S", 2), ("B2K_SCHNORR_PK", 3), ("B2K_SCHNORR_INVALID", 4)):
        assert re.search(r"\b%s = %d\b" % (st, v), hdr), st


def test_edwards25519_uses_the_eddsa_kernel():
    src, hdr = open(ED).read(), open(HDR).read()
    assert "C.b2k_ed25519_verify(" in src and _declared(hdr, "b2k_ed25519_verify")
    assert "case C.B2K_ED_OK:" in src and "case C.B2K_ED_NOT_EQUAL:\n\t\t\terrs[i] = errSchnorrInvalid" in src
    # statuses 1-7: the reference on the host for that signature
    assert "default:\n\t\t\terrs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i])" in src


def test_signatures_and_reference_errors():
    for path in (BLS, ED):
        src = open(path).read()
        assert src.startswith("//go:build b200"), path
        assert re.search(r"\bfunc SchnorrVerifyWithChecksBatch\(g kyber\.Group, pubs, msgs, sigs \[\]\[\]byte\) \[\]error", src)
        assert re.search(r"\bfunc SchnorrVerifyBatch\(g kyber\.Group, pubs \[\]kyber\.Point, msgs, sigs \[\]\[\]byte\) \[\]error", src)
        assert 'errors.New("schnorr: invalid signature")' in src
        assert '"schnorr: signature of invalid length %d instead of %d"' in src
        assert '"error unmarshalling public key: %w"' in src
    src = open(BLS).read()
    assert 'errors.New("schnorr: error unmarshalling public key")' in src
    assert "case C.B2K_SCHNORR_R, C.B2K_SCHNORR_S:\n\t\t\terrs[i] = schnorr.VerifyWithChecks(g, pubs[i], msgs[i], sigs[i])" in src
    assert "case C.B2K_SCHNORR_PK:\n\t\t\terrs[i] = errSchnorrPK" in src
