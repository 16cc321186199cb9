"""CPU: static checks on the Go adapter's shuffle bindings (go/group/edwards25519/b200/shuffle.go; no Go toolchain in the image):
both shuffle entry points of include/b2kyber.h are bound, the status constants are all mapped, and the per-shuffle errors carry
the reference's messages (shuffle/simple.go:250, shuffle/pair.go:302 and :308)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "go", "group", "edwards25519", "b200", "shuffle.go")


def test_shuffle_entry_points_are_bound():
    src = open(SRC).read()
    hdr = open(os.path.join(ROOT, "include", "b2kyber.h")).read()
    for name in ("b2k_ed25519_shuffle_verify", "b2k_ed25519_shuffle_sequence_verifiable"):
        assert "C.%s(" % name in src
        assert re.search(r"\bint %s\(" % name, hdr)
    for st in ("B2K_SHUFFLE_OK", "B2K_SHUFFLE_SIMPLE", "B2K_SHUFFLE_PAIR"):
        assert "C." + st in src
    assert re.search(r"\bfunc HashVerifyShuffles\(", src) and re.search(r"\bfunc GetSequenceVerifiable\(", src)
    assert src.startswith("//go:build b200")


def test_errors_are_the_reference_messages():
    src = open(SRC).read()
    assert 'errors.New("incorrect SimpleShuffleProof")' in src
    assert 'errors.New("invalid PairShuffleProof")' in src
