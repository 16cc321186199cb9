"""CPU: the BLS12-381 ECIES restatement (tests/ecies_bls12381_oracle.py) against an independent implementation of its symmetric
half, the `cryptography` package's HKDF-SHA256 and AES-256-GCM, on the 48- and 96-byte ikm of G1 and G2 points; its point
encodings against the ZCash deserialisation fixtures' rules (oracle/bls12381.py); and round trips on G1 and G2.  The reference
has no ECIES vector on BLS12-381."""
import random

import pytest
from cryptography.hazmat.primitives import hashes
from cryptography.hazmat.primitives.ciphers.aead import AESGCM
from cryptography.hazmat.primitives.kdf.hkdf import HKDF

from oracle import bls12381 as bls
import ecies_bls12381_oracle as eb

R = bls.R


def sb(k: int) -> bytes:
    return k.to_bytes(32, "big")


def independent_encrypt(group, pub_pt, r: int, msg: bytes) -> bytes:
    """R || AESGCM(key, nonce).encrypt(msg), key || nonce = HKDF-SHA256(dh, salt None, info None) of the `cryptography` package"""
    dh = eb.compress(group, eb.mul(group, r, pub_pt) if pub_pt is not None else None)
    k = HKDF(algorithm=hashes.SHA256(), length=44, salt=None, info=None).derive(dh)
    return eb.compress(group, eb.mul(group, r)) + AESGCM(k[:32]).encrypt(k[32:], msg, None)


@pytest.mark.parametrize("group", eb.GROUPS)
def test_symmetric_half_against_cryptography(group):
    rng = random.Random(group)
    for n in (0, 1, 15, 16, 17, 32, 1000):
        priv = rng.randrange(R)
        pub = eb.public(group, sb(priv))
        r = rng.randrange(R)
        msg = rng.randbytes(n)
        st, ct = eb.encrypt(group, pub, sb(r), msg)
        assert st == eb.OK
        assert ct == independent_encrypt(group, eb.decode(group, pub)[1], r, msg)
        assert eb.decrypt(group, sb(priv), ct) == (eb.OK, msg)
    # the identity as dh: ikm = 0xC0 || 0...
    inf = eb.compress(group, None)
    st, ct = eb.encrypt(group, inf, sb(5), b"share")
    k = HKDF(algorithm=hashes.SHA256(), length=44, salt=None, info=None).derive(inf)
    assert st == eb.OK and ct[eb.POINT_LEN[group]:] == AESGCM(k[:32]).encrypt(k[32:], b"share", None)


@pytest.mark.parametrize("group", eb.GROUPS)
def test_point_encodings(group):
    """compress / decode: infinity is 0xC0 || 0..., k G decodes back to itself, and the flags follow the ZCash rules"""
    pl = eb.POINT_LEN[group]
    assert eb.compress(group, None) == bytes([0xC0]) + bytes(pl - 1)
    assert eb.decode(group, bytes([0xC0]) + bytes(pl - 1)) == (True, None)
    for k in (1, 2, R - 1, 12345):
        b = eb.compress(group, eb.mul(group, k))
        assert b[0] & 0x80 and not b[0] & 0x40
        assert eb.decode(group, b) == (True, eb.mul(group, k))
    assert eb.decode(group, bytes([0xE0]) + bytes(pl - 1)) == (False, None)      # infinity with the sign flag
    assert eb.decode(group, bytes(pl)) == (False, None)                          # compression flag clear


@pytest.mark.parametrize("group", eb.GROUPS)
def test_round_trips_and_failures(group):
    rng = random.Random(10 + group)
    pl = eb.POINT_LEN[group]
    for priv in (0, 1, R - 1, rng.randrange(R)):
        pub = eb.public(group, sb(priv))
        for r in (0, 1, R - 1, rng.randrange(R)):
            msg = rng.randbytes(33)
            st, ct = eb.encrypt(group, pub, sb(r), msg)
            assert st == eb.OK and len(ct) == pl + 33 + 16
            assert eb.decrypt(group, sb(priv), ct) == (eb.OK, msg)
            bad = ct[:-1] + bytes([ct[-1] ^ 1])
            assert eb.decrypt(group, sb(priv), bad) == (eb.AUTH, bytes(33))
    st, ct = eb.encrypt(group, bytes(pl), sb(3), b"abc")
    assert (st, ct) == (eb.POINT, bytes(pl + 3 + 16))
    assert eb.decrypt(group, sb(3), bytes(pl) + bytes(19)) == (eb.POINT, bytes(3))
