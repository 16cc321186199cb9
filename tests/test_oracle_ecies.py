"""CPU: the ECIES restatement (oracle/ecies.py) pinned to FIPS-197 C.3 and, independently, to OpenSSL through the
`cryptography` package's AESGCM and HKDF; both ECIES directions round-trip, and the scalar rule is geScalarMult's."""
import random

import pytest

from oracle import ecies as ec
from oracle import ed25519 as ed

LENGTHS = [0, 1, 15, 16, 17, 31, 32, 33, 100, 4096]


def test_fips197_c3():
    key = bytes(range(32))
    pt = bytes.fromhex("00112233445566778899aabbccddeeff")
    assert ec.aes256_encrypt_block(key, pt) == bytes.fromhex("8ea2b7ca516745bfeafc49904b496089")


def test_sbox_is_a_permutation_with_the_known_ends():
    assert sorted(ec.SBOX) == list(range(256))
    assert ec.SBOX[0x00] == 0x63 and ec.SBOX[0x01] == 0x7c and ec.SBOX[0x53] == 0xed and ec.SBOX[0xff] == 0x16


def test_gcm_against_openssl():
    aead = pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead")
    rng = random.Random(1)
    for n in LENGTHS:
        key, nonce, msg = rng.randbytes(32), rng.randbytes(12), rng.randbytes(n)
        ct = aead.AESGCM(key).encrypt(nonce, msg, None)
        assert ec.gcm_seal(key, nonce, msg) == ct, n
        assert ec.gcm_open(key, nonce, ct) == msg
        bad = bytearray(ct)
        bad[rng.randrange(len(bad))] ^= 1 << rng.randrange(8)
        assert ec.gcm_open(key, nonce, bytes(bad)) is None


def test_hkdf_against_openssl():
    hk = pytest.importorskip("cryptography.hazmat.primitives.kdf.hkdf")
    hashes = pytest.importorskip("cryptography.hazmat.primitives.hashes")
    rng = random.Random(2)
    for n in (1, 32, 44, 64, 100):
        secret = rng.randbytes(32)
        want = hk.HKDF(algorithm=hashes.SHA256(), length=n, salt=None, info=None).derive(secret)
        assert ec.hkdf_sha256(secret, n) == want


def test_round_trip_and_the_wire_layout():
    rng = random.Random(3)
    for n in (0, 1, 32, 33, 1000):
        priv = rng.randbytes(32)
        pub = ec.mul(priv)
        r, msg = rng.randbytes(32), rng.randbytes(n)
        st, ct = ec.encrypt(pub, r, msg)
        assert st == ec.OK and len(ct) == 32 + n + 16 and ct[:32] == ec.mul(r)
        assert ec.decrypt(priv, ct) == (ec.OK, msg)
        bad = bytearray(ct)
        bad[32 + rng.randrange(n + 16)] ^= 0x80
        assert ec.decrypt(priv, bytes(bad)) == (ec.AUTH, bytes(n))


def test_scalars_are_read_as_point_mul_reads_them():
    rng = random.Random(4)
    P = ed.decode(ec.mul(rng.randbytes(32)))
    for k in [0, 1, ed.L, (1 << 256) - 1, 0x8f << 248, 0x80 << 248, rng.getrandbits(256)]:
        b = k.to_bytes(32, "little")
        e63 = ec.top_digit(k)
        eff = k - (e63 << 252) if e63 > 8 else k
        assert ec.mul(b, P) == ed.encode(ed.scalar_mult(eff % (8 * ed.L), P))
    assert ec.top_digit((1 << 256) - 1) == 16 and ec.top_digit(0x80 << 248) == 8


def test_points_decode_like_frombytes():
    priv = bytes(range(32))
    st, ct = ec.encrypt(bytes(32), b"\x07" * 32, b"share")     # all-zero bytes: the point of order 4
    assert st == ec.OK and ec.decrypt(priv, ct)[0] == ec.AUTH
    bad = next(bytes([i]) + bytes(31) for i in range(2, 256) if ed.decode(bytes([i]) + bytes(31)) is None)
    assert ec.encrypt(bad, b"\x07" * 32, b"x")[0] == ec.POINT
    assert ec.decrypt(priv, bad + bytes(17)) == (ec.POINT, bytes(1))
