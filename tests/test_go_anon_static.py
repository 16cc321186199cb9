"""CPU: static checks on the Go adapter's ring signature binding (go/group/edwards25519/b200/anon.go; no Go toolchain in the
image): the entry point and its three status constants exist in include/b2kyber.h and are bound, the errors carry the
reference's messages (sign/anon/sig.go:243 and the Tag's point decoding), and the build tag is present."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "go", "group", "edwards25519", "b200")
SRC = os.path.join(PKG, "anon.go")


def test_anon_entry_point_is_bound():
    src = open(SRC).read()
    hdr = open(os.path.join(ROOT, "include", "b2kyber.h")).read()
    assert "C.b2k_ed25519_anon_verify(" in src
    assert re.search(r"\bint b2k_ed25519_anon_verify\(", hdr)
    for st in ("B2K_ANON_OK", "B2K_ANON_INVALID", "B2K_ANON_POINT"):
        assert "C." + st in src
        assert re.search(r"\b%s = \d" % st, hdr)
    assert re.search(r"\bfunc AnonVerifyBatch\(msgs \[\]\[\]byte, anonymitySet anon\.Set, linkScope \[\]byte, sigs \[\]\[\]byte\)", src)
    assert src.startswith("//go:build b200")


def test_errors_are_the_reference_messages():
    src = open(SRC).read()
    pkg = "".join(open(os.path.join(PKG, f)).read() for f in os.listdir(PKG) if f.endswith(".go"))
    assert 'errors.New("invalid signature")' in src
    assert "errInvalidPoint" in src and 'errInvalidPoint = errors.New("invalid Ed25519 curve point")' in pkg
    assert "io.EOF" in src and "io.ErrUnexpectedEOF" in src
