"""CPU: static checks on the Go adapter's sign/bdn binding (go/pairing/bls12381/b200/bdn.go; no Go toolchain in the image): the
entry points and status constants it uses exist in include/b2kyber.h, both schemes are bound, statuses map to the reference's
error strings (sign/bls/bls.go:82-96), and the build tag is present."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "go", "pairing", "bls12381", "b200", "bdn.go")


def test_bdn_entry_points_are_bound():
    src = open(SRC).read()
    hdr = open(os.path.join(ROOT, "include", "b2kyber.h")).read()
    for fn in ("b2k_bls12381_g2_bdn_terms", "b2k_bls12381_g1_bdn_terms", "b2k_bls12381_g2_bdn_aggregate_keys",
               "b2k_bls12381_g1_bdn_aggregate_keys", "b2k_bls12381_bdn_verify_g1sig", "b2k_bls12381_bdn_verify_g2sig"):
        assert "C.%s(" % fn in src, fn
        assert re.search(r"\bint %s\(" % fn, hdr), fn
    for st in ("B2K_BDN_OK", "B2K_BDN_SIG", "B2K_ERR_POINT"):
        assert "C." + st in src
        assert re.search(r"\b%s\b\s*=" % st, hdr) or re.search(r"#define %s\b" % st, hdr)
    assert re.search(r"\bfunc BDNTerms\(publics \[\]kyber\.Point\) \(\*BDNRoster, error\)", src)
    assert re.search(r"\bfunc AggregatePublicKeysBatch\(r \*BDNRoster, masks \[\]\[\]byte\) \(\[\]kyber\.Point, error\)", src)
    assert re.search(r"\bfunc VerifyBatch\(r \*BDNRoster, masks \[\]\[\]byte, msgs \[\]\[\]byte, sigs \[\]\[\]byte\) \(\[\]error, error\)", src)
    assert src.startswith("//go:build b200")


def test_statuses_carry_the_reference_s_errors():
    src = open(SRC).read()
    assert 'errors.New("bls: unmarshalling signature point")' in src
    assert 'errors.New("bls: invalid signature")' in src
    body = src[src.index("func VerifyBatch"):]
    assert "case C.B2K_BDN_SIG:\n\t\t\terrs[k] = errBDNSig" in body
    assert "default:\n\t\t\terrs[k] = errBDNInvalid" in body
    # the signature group's default domain separation tags
    assert "sigLen, dst := 48, domainG1" in body and "sigLen, dst = 96, domainG2" in body
