"""CPU ORACLE (test infrastructure, NOT product code) -- Ed25519 signing and the reference's checked verification.

Restates, from the in-tree reference:
  EdDSA.Sign / NewKeyAndSeed   sign/eddsa/eddsa.go:90-142 (RFC 8032 5.1.6: a = clamp(SHA-512(seed)[:32]), prefix =
                               SHA-512(seed)[32:], r = SHA-512(prefix || M) mod l, S = r + SHA-512(R || A || M) a mod l)
  VerifyWithChecks             sign/eddsa/eddsa.go:149-229 -> verify_with_checks(), line by line:
    scalar.IsCanonical         group/edwards25519/scalar.go:2299-2333 (s < l)
    point.IsCanonical          group/edwards25519/point.go:296-323 (y < p on the raw bytes, bit 255 ignored)
    point.HasSmallOrder        group/edwards25519/point.go:260-294 (re-encoding, bit 255 masked, against the five y of
                               the points of order 1, 2, 4, 8 -- derived here from the curve: small_order_ys())
    h = scalar.SetBytes(SHA-512(R || A || M))   scalar.go:187-189 (little-endian, mod l)
    encode(s B) == encode(R + h A)              eddsa.go:220-227, cofactorless
Return codes are those of b2k_ed25519_verify (include/b2kyber.h); SIG_LENGTH is the host-side length check, which has no
device code.
"""
from __future__ import annotations
import hashlib

from oracle.ed25519 import BASE, D, L, P, SQRT_M1, add, decode, encode, scalar_mult

OK, SIG_NOT_CANONICAL, R_NOT_CANONICAL, R_INVALID, R_SMALL_ORDER = 0, 1, 2, 3, 4
PK_NOT_CANONICAL, PK_INVALID, PK_SMALL_ORDER, NOT_EQUAL = 5, 6, 7, 8
SIG_LENGTH = 9
ERR_NAMES = {SIG_NOT_CANONICAL: "ErrSignatureNotCanonical", R_NOT_CANONICAL: "ErrPointRNotCanonical",
             R_INVALID: "ErrPointRInvalid", R_SMALL_ORDER: "ErrPointRSmallOrder", PK_NOT_CANONICAL: "ErrPKNotCanonical",
             PK_INVALID: "ErrPKInvalid", PK_SMALL_ORDER: "ErrPKSmallOrder", NOT_EQUAL: "ErrSignatureRecNotEqual",
             SIG_LENGTH: "ErrSignatureLength"}


def _sqrt(a: int):
    r = pow(a, (P + 3) // 8, P)
    if r * r % P != a % P:
        r = r * SQRT_M1 % P
    return r if r * r % P == a % P else None


def small_order_ys() -> list:
    """y of every point of order dividing 8: 1 (identity), p - 1 (order 2), 0 (order 4) and the two order-8 y values,
    which solve d y^4 + 2 y^2 - 1 = 0 (doubling (x, y) gives y = 0 exactly when x^2 = -y^2)."""
    ys = [0, 1, P - 1]
    r = _sqrt((1 + D) % P)
    for y2 in ((-1 + r) * pow(D, P - 2, P) % P, (-1 - r) * pow(D, P - 2, P) % P):
        y = _sqrt(y2)
        if y is not None and _sqrt((-y2) % P) is not None:
            ys += sorted((y, P - y))
    return ys


def order8_point():
    """one point of order 8 (x, y)"""
    y = small_order_ys()[3]
    x = _sqrt((y * y - 1) * pow(D * y * y + 1, P - 2, P) % P)
    return (x, y)


def is_canonical_scalar(b: bytes) -> bool:
    return len(b) == 32 and int.from_bytes(b, "little") < L


def is_canonical_point(b: bytes) -> bool:
    return len(b) == 32 and int.from_bytes(b, "little") & ((1 << 255) - 1) < P


def has_small_order(pt) -> bool:
    return int.from_bytes(encode(pt), "little") & ((1 << 255) - 1) in small_order_ys()


def h_scalar(r_bytes: bytes, pk: bytes, msg: bytes) -> int:
    return int.from_bytes(hashlib.sha512(r_bytes + pk + msg).digest(), "little") % L


def keygen(seed: bytes):
    """-> (a, prefix, public key bytes)"""
    d = hashlib.sha512(seed).digest()
    a = bytearray(d[:32])
    a[0] &= 248; a[31] &= 127; a[31] |= 64
    a = int.from_bytes(a, "little")
    return a, d[32:], encode(scalar_mult(a, BASE))


def sign_raw(a: int, prefix: bytes, pk: bytes, msg: bytes) -> bytes:
    """Sign with secret scalar a under the public key bytes pk (which need not be a B; the cofactor tests use a B + T8)"""
    r = int.from_bytes(hashlib.sha512(prefix + msg).digest(), "little") % L
    R = encode(scalar_mult(r, BASE))
    s = (r + h_scalar(R, pk, msg) * a) % L
    return R + s.to_bytes(32, "little")


def sign(seed: bytes, msg: bytes) -> bytes:
    a, prefix, pk = keygen(seed)
    return sign_raw(a, prefix, pk, msg)


def verify_with_checks(pk: bytes, msg: bytes, sig: bytes) -> int:
    if len(sig) != 64:
        return SIG_LENGTH
    if not is_canonical_scalar(sig[32:]):
        return SIG_NOT_CANONICAL
    if not is_canonical_point(sig[:32]):
        return R_NOT_CANONICAL
    R = decode(sig[:32])
    if R is None:
        return R_INVALID
    if has_small_order(R):
        return R_SMALL_ORDER
    s = int.from_bytes(sig[32:], "little")
    if not is_canonical_point(pk):
        return PK_NOT_CANONICAL
    A = decode(pk)
    if A is None:
        return PK_INVALID
    if has_small_order(A):
        return PK_SMALL_ORDER
    h = h_scalar(sig[:32], pk, msg)
    S = scalar_mult(s, BASE)
    RhA = add(R, scalar_mult(h, A))
    return OK if encode(RhA) == encode(S) else NOT_EQUAL
