"""CPU: static checks on the Go adapter's BLS12-381 ECIES binding (go/pairing/bls12381/b200/ecies.go; no Go toolchain in the
image): the four entry points and the status constants exist in include/b2kyber.h and are bound, the errors are the reference's
(encrypt/ecies/ecies.go: "invalid ecies cipher", kilic's UnmarshalBinary error, crypto/cipher's GCM Open) in its order, r is
picked on the host as the reference picks it, and the build tag is set."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "go", "pairing", "bls12381", "b200", "ecies.go")
HDR = os.path.join(ROOT, "include", "b2kyber.h")


def test_entry_points_and_statuses_are_bound():
    src, hdr = open(SRC).read(), open(HDR).read()
    for g in (1, 2):
        for op in ("decrypt", "encrypt"):
            fn = f"b2k_bls12381_g{g}_ecies_{op}"
            assert "C.%s(" % fn in src, fn
            assert re.search(r"\bint %s\(" % fn, hdr), fn
    for st in ("B2K_ECIES_OK", "B2K_ECIES_POINT", "B2K_ECIES_AUTH", "B2K_ECIES_MAX_LEN"):
        assert "C." + st in src, st
        assert re.search(r"#define %s\b" % st, hdr), st
    assert src.startswith("//go:build b200")


def test_signatures_and_reference_errors():
    src = open(SRC).read()
    assert re.search(r"\bfunc ECIESDecryptBatch\(g kyber\.Group, private kyber\.Scalar, ctxts \[\]\[\]byte\) \(\[\]\[\]byte, \[\]error\)", src)
    assert re.search(r"\bfunc ECIESEncryptBatch\(g kyber\.Group, publics \[\]kyber\.Point, msgs \[\]\[\]byte\) \(\[\]\[\]byte, error\)", src)
    assert 'errors.New("invalid ecies cipher")' in src
    assert 'errors.New("cipher: message authentication failed")' in src
    body = src[src.index("func ECIESDecryptBatch"):src.index("func ECIESEncryptBatch")]
    short, tag, cap = body.index("len(c) < pl:"), body.index("len(c) < pl+16"), body.index("B2K_ECIES_MAX_LEN")
    assert short < tag < cap                                       # the reference's order: point length, R, then GCM's tag
    assert body[tag:cap].index("UnmarshalBinary(c[:pl])") < body[tag:cap].index("errECIESOpen")
    # status POINT: kilic's own error, from the reference's UnmarshalBinary on the host
    assert "case C.B2K_ECIES_POINT:\n\t\t\t\terrs[i] = g.Point().UnmarshalBinary(ctxts[i][:pl])" in body
    assert "case C.B2K_ECIES_AUTH:\n\t\t\t\terrs[i] = errECIESOpen" in body
    assert "g.Scalar().Pick(rnd)" in src and "random.New()" in src
    assert "ecies.Decrypt(g, private, c, sha256.New)" in body and "ecies.Encrypt(g, publics[i], m, sha256.New)" in src
    assert "append([]byte{}, cb[" in src                            # every result is its own copy
