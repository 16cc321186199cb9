"""CPU ORACLE (test infrastructure, NOT product code) -- ECIES on BLS12-381 with keys on G1 or on G2 and SHA-256, restated
from the reference (encrypt/ecies/ecies.go:23-131) over oracle/ecies.py's AES-256, GCM and HKDF-SHA256 and oracle/bls12381.py's
group arithmetic and ZCash codecs.

  Encrypt(P, r, msg) = R || AES-GCM_k(nonce, msg),  R = r G, dh = r P, k || nonce = HKDF(dh.MarshalBinary(), nil, nil)[0:44]
  Decrypt(priv, ct)  = GCM Open under HKDF((priv R).MarshalBinary()) of ct[PL:], R = UnmarshalBinary(ct[:PL])

PL = 48 on G1 and 96 on G2 (kilic/g1.go:119-124, g2.go:118-123).  Scalars are mod.Int bytes: 32 bytes big-endian, below r.
The point codecs are those the reference's ZCash deserialisation fixtures pin; the symmetric half is checked against the
`cryptography` package in tests/test_oracle_ecies_bls12381.py."""
from __future__ import annotations

from oracle import bls12381 as bls
from oracle import ecies as ec

OK, POINT, AUTH = ec.OK, ec.POINT, ec.AUTH
MAX_LEN = ec.MAX_LEN
GROUPS = (1, 2)
POINT_LEN = {1: 48, 2: 96}


def _decode(group: int, b: bytes):
    """UnmarshalBinary with the subgroup check; raises ValueError"""
    if group == 1:
        pt = bls.g1_decompress(b, subgroup_check=False)
        if pt is not None and not bls.g1_in_subgroup_fast(pt):
            raise ValueError("not in G1")
        return pt
    pt = bls.g2_decompress(b, subgroup_check=False)
    if pt is not None and not bls.g2_in_subgroup_fast(pt):
        raise ValueError("not in G2")
    return pt


def decode(group: int, b: bytes):
    """(ok, point): point None is infinity"""
    try:
        return True, _decode(group, b)
    except ValueError:
        return False, None


def compress(group: int, pt) -> bytes:
    return bls.g1_compress(pt) if group == 1 else bls.g2_compress(pt)


def mul(group: int, k: int, pt=None):
    """k pt, pt None = the generator"""
    if group == 1:
        return bls.g1_mul(k, bls.G1 if pt is None else pt)
    return bls.g2_mul(k, bls.G2 if pt is None else pt)


def public(group: int, priv: bytes) -> bytes:
    return compress(group, mul(group, _scalar(priv)))


def _scalar(b: bytes) -> int:
    k = int.from_bytes(b, "big")
    assert len(b) == 32 and k < bls.R
    return k


def derive(dh: bytes):
    k = ec.hkdf_sha256(dh, 44)
    return k[:32], k[32:44]


def encrypt(group: int, pub: bytes, r: bytes, msg: bytes):
    """(status, ciphertext): ecies.Encrypt with the ephemeral scalar r; the ciphertext is zero unless OK"""
    pl = POINT_LEN[group]
    ok, P = decode(group, pub)
    if not ok:
        return POINT, bytes(pl + len(msg) + 16)
    k = _scalar(r)
    key, nonce = derive(compress(group, mul(group, k, P) if P is not None else None))
    return OK, compress(group, mul(group, k)) + ec.gcm_seal(key, nonce, msg)


def decrypt(group: int, priv: bytes, ct: bytes):
    """(status, message) of ecies.Decrypt for a ciphertext of at least PL + 16 bytes; the message is zero unless OK"""
    pl = POINT_LEN[group]
    assert len(ct) >= pl + 16
    zero = bytes(len(ct) - pl - 16)
    ok, R = decode(group, ct[:pl])
    if not ok:
        return POINT, zero
    key, nonce = derive(compress(group, mul(group, _scalar(priv), R) if R is not None else None))
    m = ec.gcm_open(key, nonce, ct[pl:])
    return (AUTH, zero) if m is None else (OK, m)
