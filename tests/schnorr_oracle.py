"""CPU ORACLE (test infrastructure, NOT product code) -- sign/schnorr Sign and VerifyWithChecks, restated line by line for
BLS12-381 keys on G1, on G2, and edwards25519.

Restates, from the in-tree reference:
  Sign              sign/schnorr/schnorr.go:28-58: k random, R = k B, h = hash(public, R, msg), s = k + h private
  VerifyWithChecks  sign/schnorr/schnorr.go:89-165 -> verify_with_checks(), in the reference's order:
    1 len(sig) != PointLen + ScalarLen                        -> LENGTH (host only)
    2 R.UnmarshalBinary                                       -> R (BLS) / R_INVALID (edwards25519)
    3 IsCanonical / HasSmallOrder of R (edwards25519 only)    -> R_NOT_CANONICAL, R_SMALL_ORDER
    4 scalar IsCanonical (edwards25519 only)                  -> SIG_NOT_CANONICAL
    5 R.IsInCorrectGroup: cannot fail on BLS12-381, whose UnmarshalBinary checks the subgroup (kilic/g1.go:127-131)
    6 s.UnmarshalBinary: mod.Int rejects s >= r (group/mod/int.go:359-372) -> S (BLS)
    7 public.UnmarshalBinary, then the checks of 3 on it      -> PK (BLS) / PK_INVALID, PK_NOT_CANONICAL, PK_SMALL_ORDER
    8 h = Scalar().SetBytes(SHA-512(R.MarshalTo || public.MarshalTo || msg)): big-endian mod r on BLS12-381 (mod.Int,
      int.go:404-411), little-endian mod l on edwards25519 (scalar.go:187-189); s B != R + h public -> INVALID / NOT_EQUAL
The BLS12-381 statuses are those of B2K_SCHNORR_* (include/b2kyber.h); the edwards25519 ones are the B2K_ED_* codes of
oracle/eddsa.py, returned in Schnorr's order.  The digest here hashes the re-encodings (compress / encode), as the
reference does, not the input bytes.

The reference has no Schnorr vectors on BLS12-381 (its schnorr_test.go runs on edwards25519 only).  The BLS half rests on
oracle/bls12381.py, which the ZCash deserialisation fixtures and the drand KATs pin.  The edwards25519 half is cross-pinned:
every signature sign() makes there also passes oracle/eddsa.verify_with_checks, which RFC 8032 and Wycheproof pin
(the reference's TestEdDSACompatibility).
"""
from __future__ import annotations
import hashlib

from oracle import bls12381 as bls
from oracle import ed25519 as ed
from oracle import eddsa as oe

OK, R_BAD, S_BAD, PK_BAD, INVALID, LENGTH = 0, 1, 2, 3, 4, 5
NAMES = {OK: "OK", R_BAD: "R", S_BAD: "S", PK_BAD: "PK", INVALID: "INVALID", LENGTH: "LENGTH"}
GROUPS = ("bls12381_g1", "bls12381_g2", "ed25519")
POINT_LEN = {"bls12381_g1": 48, "bls12381_g2": 96, "ed25519": 32}
ORDER = {"bls12381_g1": bls.R, "bls12381_g2": bls.R, "ed25519": ed.L}


def _g1_decode(b: bytes):
    pt = bls.g1_decompress(b, subgroup_check=False)
    if not bls.g1_in_subgroup_fast(pt):
        raise ValueError("not in G1")
    return pt


def _g2_decode(b: bytes):
    pt = bls.g2_decompress(b, subgroup_check=False)
    if not bls.g2_in_subgroup_fast(pt):
        raise ValueError("not in G2")
    return pt


# per BLS group: decode (raises ValueError), encode, k P, P + Q, -P, base point
_BLS = {
    "bls12381_g1": (_g1_decode, bls.g1_compress, bls.g1_mul, bls.g1_add, bls.g1_neg, bls.G1),
    "bls12381_g2": (_g2_decode, bls.g2_compress, bls.g2_mul, bls.g2_add, bls.g2_neg, bls.G2),
}


def reduce_be(digest: bytes) -> int:
    """mod.Int.SetBytes on a BLS12-381 suite: the bytes read big-endian, mod r"""
    return int.from_bytes(digest, "big") % bls.R


def challenge(group: str, r_enc: bytes, pk_enc: bytes, msg: bytes) -> int:
    d = hashlib.sha512(r_enc + pk_enc + msg).digest()
    return reduce_be(d) if group != "ed25519" else int.from_bytes(d, "little") % ed.L


def point(group: str, k: int):
    """k B in the group, as the oracle's point object"""
    if group == "ed25519":
        return ed.scalar_mult(k % ed.L)
    return _BLS[group][2](k % bls.R)


def encode(group: str, pt) -> bytes:
    return ed.encode(pt) if group == "ed25519" else _BLS[group][1](pt)


def public_key(group: str, x: int) -> bytes:
    return encode(group, point(group, x))


def sign(group: str, x: int, msg: bytes, k: int) -> bytes:
    """Sign with private scalar x and nonce k (the reference picks k at random)"""
    R = public_key(group, k)
    h = challenge(group, R, public_key(group, x), msg)
    s = (k + h * x) % ORDER[group]
    return R + (s.to_bytes(32, "little") if group == "ed25519" else s.to_bytes(32, "big"))


def _verify_bls(group: str, pub: bytes, msg: bytes, sig: bytes) -> int:
    decode, enc, mul, add, neg, base = _BLS[group]
    pl = POINT_LEN[group]
    if len(sig) != pl + 32:
        return LENGTH
    try:
        R = decode(sig[:pl])
    except ValueError:
        return R_BAD
    s = int.from_bytes(sig[pl:], "big")
    if s >= bls.R:
        return S_BAD
    try:
        if len(pub) != pl:
            raise ValueError("wrong length")
        A = decode(pub)
    except ValueError:
        return PK_BAD
    h = challenge(group, enc(R), enc(A), msg)
    return OK if mul(s, base) == add(R, mul(h, A)) else INVALID


def _verify_ed(pub: bytes, msg: bytes, sig: bytes) -> int:
    if len(sig) != 64:
        return oe.SIG_LENGTH
    R = ed.decode(sig[:32])
    if R is None:
        return oe.R_INVALID
    if not oe.is_canonical_point(sig[:32]):
        return oe.R_NOT_CANONICAL
    if oe.has_small_order(R):
        return oe.R_SMALL_ORDER
    if not oe.is_canonical_scalar(sig[32:]):
        return oe.SIG_NOT_CANONICAL
    s = int.from_bytes(sig[32:], "little")
    A = ed.decode(pub) if len(pub) == 32 else None
    if A is None:
        return oe.PK_INVALID
    if not oe.is_canonical_point(pub):
        return oe.PK_NOT_CANONICAL
    if oe.has_small_order(A):
        return oe.PK_SMALL_ORDER
    h = challenge("ed25519", ed.encode(R), ed.encode(A), msg)
    return oe.OK if ed.encode(ed.scalar_mult(s)) == ed.encode(ed.add(R, ed.scalar_mult(h, A))) else oe.NOT_EQUAL


def verify_with_checks(group: str, pub: bytes, msg: bytes, sig: bytes) -> int:
    return _verify_ed(pub, msg, sig) if group == "ed25519" else _verify_bls(group, pub, msg, sig)


def fails_before_equation(group: str, status: int) -> bool:
    if group == "ed25519":
        return status not in (oe.OK, oe.NOT_EQUAL)
    return status not in (OK, INVALID)
