"""CPU: the IBE restatement (oracle/ibe.py) against the reference's behaviour -- the drand timelock interop vector, round trips on
both groups, the reference's negative tests (encrypt/ibe/ibe_test.go) and an H3 that needs more than one candidate."""
import random

import pytest

from oracle import bls12381 as o
from oracle import ibe

TLOCK_BEACON = bytes.fromhex(
    "86ecea71376e78abd19aaf0ad52f462a6483626563b1023bd04815a7b953da888c74f5bf6ee672a5688603ab310026230522898f33f23a7de363c66f90ffd49e"
    "c77ebf7f6c1478a9ecd6e714b4d532ab43d044da0a16fed13b4791d7fc999e2b")
TLOCK_U = bytes.fromhex("a5ddec5fa76795d5a28f0869e6a620248c94c112beb8135b11d5614a2b6845c5a4128e3dfe4328d7a6e70b2dea3d7f25")
TLOCK_V = bytes.fromhex("89f0e6cf2b27371017dddeff43ab2263")
TLOCK_W = bytes.fromhex("d767e14f5e3e1738a6c50725c4f0d1b6")


def multi_iteration_case(min_iter: int = 2):
    """(sigma, msg, iterations): the first seeded 16-byte pair whose H3 rejects at least one candidate."""
    rng = random.Random(7)
    while True:
        sigma, msg = rng.randbytes(16), rng.randbytes(16)
        r, it = ibe.h3_iterations(sigma, msg)
        if it >= min_iter:
            return sigma, msg, it


def test_tlock_vector():
    """TestBackwardsInteropWithTypescript (ibe_test.go:202-245, skipped in the reference: "Typescript library not yet updated").
    Steps 1-2 of DecryptCCAonG1 recover deadbeef..., which pins the GT bytes; the rP check of step 3 does not hold for this U
    under the reference's H3 (r Base != U for the scalar H3 derives), so the full decryption reports an invalid proof."""
    U, key = o.g1_decompress(TLOCK_U), o.g2_decompress(TLOCK_BEACON)
    sigma = bytes(a ^ b for a, b in zip(TLOCK_V, ibe.h2(o.gt_to_bytes(ibe.pair(U, key)), 16)))
    msg = bytes(a ^ b for a, b in zip(TLOCK_W, ibe.h4(sigma, 16)))
    assert msg.hex() == "deadbeef" * 4
    assert o.g1_mul(ibe.h3(sigma, msg)) != U
    assert ibe.decrypt_cca_g1(TLOCK_BEACON, TLOCK_U, TLOCK_V, TLOCK_W) == (bytes(16), ibe.PROOF)


@pytest.mark.parametrize("group", [1, 2])
@pytest.mark.parametrize("n", [0, 1, 12, 32])
def test_round_trip(group, n):
    rng = random.Random(100 * group + n)
    ident = b"round-%d" % n
    master, priv = ibe.keypair(group, rng.randrange(1, o.R), ident)
    msg, sigma = rng.randbytes(n), rng.randbytes(n)
    enc = ibe.encrypt_cca_g1 if group == 1 else ibe.encrypt_cca_g2
    dec = ibe.decrypt_cca_g1 if group == 1 else ibe.decrypt_cca_g2
    U, V, W = enc(master, ident, msg, sigma)
    assert len(U) == 48 * group and len(V) == len(W) == n
    assert dec(priv, U, V, W) == (msg, ibe.OK)
    # a key for another identity does not decrypt
    _, other = ibe.keypair(group, rng.randrange(1, o.R), b"another id")
    if n:
        assert dec(other, U, V, W) == (bytes(n), ibe.PROOF)


@pytest.mark.parametrize("group", [1, 2])
def test_reference_negative_cases(group):
    """ibe_test.go: V or W replaced by "somenonsense" -> invalid proof."""
    rng = random.Random(30 + group)
    ident = b"ibe test"
    master, priv = ibe.keypair(group, rng.randrange(1, o.R), ident)
    msg = b"hello world!"                               # 12 bytes, the length of "somenonsense"
    enc = ibe.encrypt_cca_g1 if group == 1 else ibe.encrypt_cca_g2
    dec = ibe.decrypt_cca_g1 if group == 1 else ibe.decrypt_cca_g2
    U, V, W = enc(master, ident, msg, rng.randbytes(12))
    assert dec(priv, U, b"somenonsense", W) == (bytes(12), ibe.PROOF)
    assert dec(priv, U, V, b"somenonsense") == (bytes(12), ibe.PROOF)
    assert dec(priv, U, V, W) == (msg, ibe.OK)


def test_h3_needs_several_candidates():
    sigma, msg, it = multi_iteration_case()
    assert it >= 2
    r, it2 = ibe.h3_iterations(sigma, msg)
    assert it2 == it and r < o.R
    # the rejected candidates really are >= r
    import hashlib
    buf = hashlib.sha256(b"IBE-H3" + sigma + msg).digest()
    for i in range(1, it):
        h = bytearray(hashlib.sha256(i.to_bytes(2, "little") + buf).digest())
        h[0] >>= 1
        assert int.from_bytes(h, "big") >= o.R
    rng = random.Random(5)
    master, priv = ibe.keypair(1, rng.randrange(1, o.R), b"id")
    U, V, W = ibe.encrypt_cca_g1(master, b"id", msg, sigma)
    assert U == o.g1_compress(o.g1_mul(r))
    assert ibe.decrypt_cca_g1(priv, U, V, W) == (msg, ibe.OK)


def test_u_that_does_not_decode_or_is_infinity():
    rng = random.Random(9)
    master, priv = ibe.keypair(1, rng.randrange(1, o.R), b"id")
    U, V, W = ibe.encrypt_cca_g1(master, b"id", b"0123456789ab", rng.randbytes(12))
    assert ibe.decrypt_cca_g1(priv, bytes(48), V, W) == (bytes(12), ibe.POINT)          # no compression flag
    assert ibe.decrypt_cca_g1(priv, o.g1_compress(None), V, W) == (bytes(12), ibe.PROOF)


def test_pairing_matches_the_python_reference_convention():
    rng = random.Random(3)
    p, q = o.g1_mul(rng.randrange(1, o.R)), o.g2_mul(rng.randrange(1, o.R))
    assert ibe.pair(p, q) == o.pairing_reference(p, q)
