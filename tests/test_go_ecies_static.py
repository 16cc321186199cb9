"""CPU: static checks on the Go adapter's ECIES binding (go/group/edwards25519/b200/ecies.go; no Go toolchain in the image): both
entry points and their status constants exist in include/b2kyber.h and are bound, the errors carry the reference's messages
(encrypt/ecies/ecies.go:87, crypto/cipher's GCM Open and the point decoding), the host-side length order is the reference's,
and the build tag is present."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "go", "group", "edwards25519", "b200")
SRC = os.path.join(PKG, "ecies.go")


def test_ecies_entry_points_are_bound():
    src = open(SRC).read()
    hdr = open(os.path.join(ROOT, "include", "b2kyber.h")).read()
    for fn in ("b2k_ed25519_ecies_decrypt", "b2k_ed25519_ecies_encrypt"):
        assert "C.%s(" % fn in src
        assert re.search(r"\bint %s\(" % fn, hdr)
    for st in ("B2K_ECIES_OK", "B2K_ECIES_POINT", "B2K_ECIES_AUTH", "B2K_ECIES_MAX_LEN"):
        assert "C." + st in src
        assert re.search(r"#define %s\b" % st, hdr)
    assert re.search(r"\bfunc ECIESDecryptBatch\(private kyber\.Scalar, ctxts \[\]\[\]byte\) \(\[\]\[\]byte, \[\]error\)", src)
    assert re.search(r"\bfunc ECIESEncryptBatch\(publics \[\]kyber\.Point, msgs \[\]\[\]byte\) \(\[\]\[\]byte, error\)", src)
    assert "Scalar().Pick(rnd)" in src and "random.New()" in src
    assert src.startswith("//go:build b200")


def test_errors_and_host_checks_are_the_reference_s():
    src = open(SRC).read()
    pkg = "".join(open(os.path.join(PKG, f)).read() for f in os.listdir(PKG) if f.endswith(".go"))
    assert 'errors.New("invalid ecies cipher")' in src
    assert 'errors.New("cipher: message authentication failed")' in src
    assert 'errInvalidPoint = errors.New("invalid Ed25519 curve point")' in pkg
    body = src[src.index("func ECIESDecryptBatch"):src.index("func ECIESEncryptBatch")]
    short, tag, cap = body.index("len(c) < 32"), body.index("len(c) < 48"), body.index("B2K_ECIES_MAX_LEN")
    assert short < tag < cap                                       # the reference's order: point length, then GCM's tag check
    # 32..47 bytes: R is decoded before the short body fails Open, as ecies.Decrypt does (ecies.go:84-90)
    short_case = body[tag:cap]
    assert short_case.index("UnmarshalBinary(c[:32])") < short_case.index("errOpen")
    # the private key is a kyber.Scalar: it is used as it is (un unwraps points only)
    assert "un(private)" not in src and "private.MarshalBinary()" in body
    # every returned ciphertext is its own copy, not a window into the staging buffer
    assert "append([]byte{}, cb[" in src
    assert "ecies.Decrypt(eciesSuite" in body and "ecies.Encrypt(eciesSuite" in src
