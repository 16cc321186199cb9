"""ECIES on edwards25519 with SHA-256, restated from the reference (encrypt/ecies/ecies.go:23-131), in plain Python:
AES-256 (FIPS-197), GCM (SP 800-38D, 12-byte nonce, 16-byte tag, no AAD), HKDF-SHA256 (RFC 5869) and both ECIES functions over
oracle/ed25519.py.

  Encrypt(P, r, msg) = R || AES-GCM_k(nonce, msg),  R = r B, dh = r P, k || nonce = HKDF(dh.MarshalBinary(), nil, nil)[0:44]
  Decrypt(priv, ct)  = GCM Open under HKDF(priv R) of ct[32:], R = FromBytes(ct[:32])

Scalars are the raw 32 little-endian bytes, multiplied as geScalarMult / geScalarMultBase multiply them (ed25519.point_mul: the
plain integer, except that a top signed digit e63 above 8 selects nothing).  TEST INFRASTRUCTURE."""
from __future__ import annotations
import hashlib
import hmac

from . import ed25519 as ed
from .ed25519 import effective_scalar, top_digit          # noqa: F401 (the digit rule, shared with Point.Mul)

OK, POINT, AUTH = 0, 1, 2               # B2K_ECIES_* of include/b2kyber.h
MAX_LEN = 1 << 16


# ---- AES-256 -----------------------------------------------------------------------------------------------------------------
def _gmul(a: int, b: int) -> int:
    r = 0
    for _ in range(8):
        if b & 1:
            r ^= a
        a = ((a << 1) ^ (0x11b if a & 0x80 else 0)) & 0xff
        b >>= 1
    return r


def _sbox_entry(x: int) -> int:
    inv = 0 if x == 0 else next(y for y in range(1, 256) if _gmul(x, y) == 1)
    s = inv
    for k in range(1, 5):
        s ^= ((inv << k) | (inv >> (8 - k))) & 0xff
    return s ^ 0x63


SBOX = [_sbox_entry(x) for x in range(256)]


def aes256_round_keys(key: bytes) -> list:
    assert len(key) == 32
    w = [list(key[4 * i:4 * i + 4]) for i in range(8)]
    rcon = 1
    for i in range(8, 60):
        t = list(w[i - 1])
        if i % 8 == 0:
            t = [SBOX[b] for b in t[1:] + t[:1]]
            t[0] ^= rcon
            rcon = _gmul(rcon, 2)
        elif i % 8 == 4:
            t = [SBOX[b] for b in t]
        w.append([a ^ b for a, b in zip(w[i - 8], t)])
    return [bytes(sum(w[4 * r:4 * r + 4], [])) for r in range(15)]


def aes256_encrypt_block(key: bytes, block: bytes, rks=None) -> bytes:
    rks = rks or aes256_round_keys(key)
    s = [b ^ k for b, k in zip(block, rks[0])]
    for r in range(1, 15):
        s = [SBOX[b] for b in s]
        s = [s[q + 4 * ((c + q) % 4)] for c in range(4) for q in range(4)]          # ShiftRows (column-major state)
        if r != 14:
            m = []
            for c in range(4):
                a = s[4 * c:4 * c + 4]
                m += [_gmul(a[0], 2) ^ _gmul(a[1], 3) ^ a[2] ^ a[3], a[0] ^ _gmul(a[1], 2) ^ _gmul(a[2], 3) ^ a[3],
                      a[0] ^ a[1] ^ _gmul(a[2], 2) ^ _gmul(a[3], 3), _gmul(a[0], 3) ^ a[1] ^ a[2] ^ _gmul(a[3], 2)]
            s = m
        s = [b ^ k for b, k in zip(s, rks[r])]
    return bytes(s)


# ---- GCM ---------------------------------------------------------------------------------------------------------------------
_R = 0xe1 << 120


def _gf128_mul(x: int, y: int) -> int:
    z, v = 0, y
    for i in range(128):
        if (x >> (127 - i)) & 1:
            z ^= v
        v = (v >> 1) ^ (_R if v & 1 else 0)
    return z


def _ghash(h: int, data: bytes) -> int:
    x = 0
    padded = data + bytes(-len(data) % 16)
    for o in range(0, len(padded), 16):
        x = _gf128_mul(x ^ int.from_bytes(padded[o:o + 16], "big"), h)
    return _gf128_mul(x ^ (len(data) * 8), h)                    # length block: len(A) = 0 || len(C) in bits


def _ctr(rks, nonce: bytes, data: bytes) -> bytes:
    out = bytearray()
    for i in range(0, len(data), 16):
        ks = aes256_encrypt_block(b"", nonce + (2 + i // 16).to_bytes(4, "big"), rks)
        out += bytes(a ^ b for a, b in zip(data[i:i + 16], ks))
    return bytes(out)


def gcm_seal(key: bytes, nonce: bytes, msg: bytes) -> bytes:
    rks = aes256_round_keys(key)
    h = int.from_bytes(aes256_encrypt_block(b"", bytes(16), rks), "big")
    c = _ctr(rks, nonce, msg)
    s = _ghash(h, c) ^ int.from_bytes(aes256_encrypt_block(b"", nonce + b"\x00\x00\x00\x01", rks), "big")
    return c + s.to_bytes(16, "big")


def gcm_open(key: bytes, nonce: bytes, ct: bytes):
    """the plaintext, or None when the tag does not match (cipher: message authentication failed)"""
    if len(ct) < 16:
        return None
    rks = aes256_round_keys(key)
    h = int.from_bytes(aes256_encrypt_block(b"", bytes(16), rks), "big")
    c, tag = ct[:-16], ct[-16:]
    s = _ghash(h, c) ^ int.from_bytes(aes256_encrypt_block(b"", nonce + b"\x00\x00\x00\x01", rks), "big")
    if s.to_bytes(16, "big") != tag:
        return None
    return _ctr(rks, nonce, c)


# ---- HKDF-SHA256 -------------------------------------------------------------------------------------------------------------
def hkdf_sha256(secret: bytes, length: int, salt: bytes = None, info: bytes = b"") -> bytes:
    prk = hmac.new(salt or bytes(32), secret, hashlib.sha256).digest()
    out, t, i = b"", b"", 1
    while len(out) < length:
        t = hmac.new(prk, t + info + bytes([i]), hashlib.sha256).digest()
        out += t
        i += 1
    return out[:length]


# ---- ECIES -------------------------------------------------------------------------------------------------------------------
def mul(scalar_le: bytes, point=None) -> bytes:
    """Point.Mul(s, P).MarshalBinary() for a decoded point (None = the base point)"""
    return ed.point_mul(scalar_le, None if point is None else ed.encode(point))


def derive(dh: bytes):
    k = hkdf_sha256(dh, 44)
    return k[:32], k[32:44]


def encrypt(pub: bytes, r: bytes, msg: bytes):
    """(status, ciphertext): ecies.Encrypt with the ephemeral scalar r; the ciphertext is zero unless OK"""
    P = ed.decode(pub)
    if P is None:
        return POINT, bytes(32 + len(msg) + 16)
    key, nonce = derive(mul(r, P))
    return OK, mul(r) + gcm_seal(key, nonce, msg)


def decrypt(priv: bytes, ct: bytes):
    """(status, message) of ecies.Decrypt for a ciphertext of at least 48 bytes; the message is zero unless OK"""
    assert len(ct) >= 48
    zero = bytes(len(ct) - 48)
    R = ed.decode(ct[:32])
    if R is None:
        return POINT, zero
    key, nonce = derive(mul(priv, R))
    m = gcm_open(key, nonce, ct[32:])
    return (AUTH, zero) if m is None else (OK, m)
