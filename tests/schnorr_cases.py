"""Shared sign/schnorr cases for the oracle, host-emulation and GPU tests: (name, public key, message, signature) per group.

For BLS12-381 keys on G1 and G2:
  honest signatures over messages of 0, 32 and longer lengths, with R || public || msg around the SHA-512 block boundaries;
  the shapes of sign/schnorr/schnorr_test.go: R replaced, s replaced, wrong key, malleability s + r (-> S);
  encodings of R and of the key with the compression flag clear, x >= p, infinity with the sign flag, off the curve and off
  the subgroup (-> R / PK); keys +-B and small multiples of B; the infinity key, the infinity R and s = 0; s = r - 1;
  digests whose two 256-bit halves both lie above 2 r (the reduction subtracts r twice from each).
For edwards25519, the same shapes where they apply, with s + l, small-order and non-canonical points.
Wrong signature lengths are host checks (length_cases): the device entry points take fixed strides.
Expected statuses come from tests/schnorr_oracle.py, not from this file.
"""
from __future__ import annotations
import functools
import hashlib

from oracle import bls12381 as bls
from oracle import ed25519 as ed
from oracle import eddsa as oe
import schnorr_oracle as so

BLS_GROUPS = ("bls12381_g1", "bls12381_g2")


def _scalar(tag: str, mod: int) -> int:
    return int.from_bytes(hashlib.sha512(tag.encode()).digest(), "big") % mod


def _msg(tag: str, n: int) -> bytes:
    out = b""
    i = 0
    while len(out) < n:
        out += hashlib.sha256(f"{tag}/{i}".encode()).digest()
        i += 1
    return out[:n]


def _s_bytes(group: str, s: int) -> bytes:
    return s.to_bytes(32, "little") if group == "ed25519" else s.to_bytes(32, "big")


def _s_of(group: str, sig: bytes) -> int:
    return int.from_bytes(sig[so.POINT_LEN[group]:], "little" if group == "ed25519" else "big")


def message_lengths(group: str) -> list:
    """0, 1, 32, 1000 and the lengths that put R || public || msg at 111, 112, 127, 128, 239, 240, 255, 256 bytes"""
    pre = 2 * so.POINT_LEN[group]
    out = [0, 1, 32, 1000]
    out += [t - pre for t in (111, 112, 127, 128, 239, 240, 255, 256, 367, 368) if t - pre >= 0]
    return sorted(set(out))


# ---- encodings that do not decode ----------------------------------------------------------------------------------------
def _g1_off_curve() -> bytes:
    x = 1
    while bls.fp_sqrt((x ** 3 + 4) % bls.P) is not None:
        x += 1
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= 0x80
    return bytes(b)


def _g1_off_subgroup() -> bytes:
    x = 1
    while True:
        y = bls.fp_sqrt((x ** 3 + 4) % bls.P)
        if y is not None and not bls.g1_in_subgroup_fast((x, y)):
            return bls.g1_compress((x, y))
        x += 1


def _g2_off_curve() -> bytes:
    x = 1
    while bls.f2_sqrt(bls.f2_add(bls.f2_mul(bls.f2_sqr((x, 1)), (x, 1)), bls.B2)) is not None:
        x += 1
    b = bytearray((1).to_bytes(48, "big") + x.to_bytes(48, "big"))
    b[0] |= 0x80
    return bytes(b)


def _g2_off_subgroup() -> bytes:
    x = 1
    while True:
        y = bls.f2_sqrt(bls.f2_add(bls.f2_mul(bls.f2_sqr((x, 1)), (x, 1)), bls.B2))
        if y is not None and not bls.g2_in_subgroup_fast(((x, 1), y)):
            return bls.g2_compress(((x, 1), y))
        x += 1


def bad_encodings(group: str) -> list:
    """(name, bytes) of encodings that UnmarshalBinary refuses"""
    pl = so.POINT_LEN[group]
    g = bytearray(so.public_key(group, 5))
    no_flag = bytes([g[0] & 0x7F]) + bytes(g[1:])
    big_x = bytearray(bls.P.to_bytes(48, "big") + bytes(pl - 48))
    big_x[0] |= 0x80
    inf_sign = bytes([0xE0]) + bytes(pl - 1)
    inf_nonzero = bytes([0xC0]) + bytes(pl - 2) + b"\x01"
    zero = bytes(pl)
    off_curve = _g1_off_curve() if group == "bls12381_g1" else _g2_off_curve()
    off_sub = _g1_off_subgroup() if group == "bls12381_g1" else _g2_off_subgroup()
    return [("compression flag clear", no_flag), ("x = p", bytes(big_x)), ("infinity with the sign flag", inf_sign),
            ("infinity with x != 0", inf_nonzero), ("all zeros", zero), ("off the curve", off_curve),
            ("off the subgroup", off_sub)]


def _high_digest_msg(group: str, R: bytes, pk: bytes) -> bytes:
    """a 32-byte message whose digest has both 256-bit halves >= 2 r (two subtractions each)"""
    for i in range(1 << 16):
        m = hashlib.sha256(b"high/%d" % i).digest()
        d = hashlib.sha512(R + pk + m).digest()
        if int.from_bytes(d[:32], "big") >= 2 * bls.R and int.from_bytes(d[32:], "big") >= 2 * bls.R:
            return m
    raise AssertionError("no message found")


@functools.lru_cache(maxsize=None)
def bls_cases(group: str) -> tuple:
    """(name, pk, msg, sig) for one BLS12-381 group; every status 0..4 occurs"""
    r = bls.R
    x = _scalar(group + "/x", r)
    pk = so.public_key(group, x)
    out = []
    for n in message_lengths(group):
        m = _msg(f"{group}/len{n}", n)
        out.append((f"honest len {n}", pk, m, so.sign(group, x, m, _scalar(f"{group}/k{n}", r))))
    m = _msg(group + "/shape", 32)
    sig = so.sign(group, x, m, _scalar(group + "/k", r))
    pl = so.POINT_LEN[group]
    s = _s_of(group, sig)
    other = so.public_key(group, 7)
    out += [
        ("R replaced", pk, m, other + sig[pl:]),
        ("s replaced", pk, m, sig[:pl] + _s_bytes(group, (s + 1) % r)),
        ("wrong key", so.public_key(group, x + 1), m, sig),
        ("message changed", pk, m[:-1] + bytes([m[-1] ^ 1]), sig),
        ("s + r", pk, m, sig[:pl] + _s_bytes(group, s + r)),
        ("s = 2^256 - 1", pk, m, sig[:pl] + b"\xff" * 32),
        ("s = r", pk, m, sig[:pl] + _s_bytes(group, r)),
    ]
    for name, enc in bad_encodings(group):
        out.append(("R: " + name, pk, m, enc + sig[pl:]))
        out.append(("key: " + name, enc, m, sig))
        out.append(("R and key: " + name, enc, m, enc + sig[pl:]))                 # R is reported first
    out.append(("R bad and s >= r", pk, m, bad_encodings(group)[0][1] + b"\xff" * 32))
    out.append(("s >= r and key bad", bad_encodings(group)[0][1], m, sig[:pl] + b"\xff" * 32))
    for k in (1, r - 1, 2, r - 2, 3, 4, 8, r - 8):                                   # +-B and small multiples of B
        mk = _msg(f"{group}/small{k}", 32)
        sk = so.sign(group, k, mk, _scalar(f"{group}/ks{k}", r))
        out.append((f"key {k if k < 100 else k - r} B", so.public_key(group, k), mk, sk))
        out.append((f"key {k if k < 100 else k - r} B, s + 1", so.public_key(group, k), mk,
                    sk[:pl] + _s_bytes(group, (_s_of(group, sk) + 1) % r)))
    # nonces equal to the key or its negation: R = +-public, so the walk meets the doubling and the inverse cases
    out.append(("R = public", pk, m, so.sign(group, x, m, x)))
    out.append(("R = -public", pk, m, so.sign(group, x, m, r - x)))
    inf = so.encode(group, None)
    out.append(("key infinity", inf, m, so.sign(group, 0, m, _scalar(group + "/k0", r))))
    out.append(("key infinity, s + 1", inf, m, sig[:pl] + _s_bytes(group, (s + 1) % r)))
    out.append(("R infinity", pk, m, so.sign(group, x, m, 0)))
    out.append(("R, s, key = O, 0, O", inf, m, inf + bytes(32)))
    out.append(("R, s = O, 0 under a key", pk, m, inf + bytes(32)))
    out.append(("s = r - 1, key infinity, R = -B", inf, m, so.public_key(group, r - 1) + _s_bytes(group, r - 1)))
    out.append(("s = r - 1 invalid", pk, m, sig[:pl] + _s_bytes(group, r - 1)))
    R = so.public_key(group, _scalar(group + "/kh", r))
    mh = _high_digest_msg(group, R, pk)
    k = _scalar(group + "/kh", r)
    out.append(("digest halves >= 2r", pk, mh, so.sign(group, x, mh, k)))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def ed_cases() -> tuple:
    """(name, pk, msg, sig) on edwards25519"""
    L, P = ed.L, ed.P
    g = "ed25519"
    x = _scalar("ed/x", L)
    pk = so.public_key(g, x)
    out = []
    for n in message_lengths(g):
        m = _msg(f"ed/len{n}", n)
        out.append((f"honest len {n}", pk, m, so.sign(g, x, m, _scalar(f"ed/k{n}", L))))
    m = _msg("ed/shape", 32)
    sig = so.sign(g, x, m, _scalar("ed/k", L))
    s = _s_of(g, sig)
    t8 = ed.encode(oe.order8_point())
    noncanon = (P + 1).to_bytes(32, "little")             # y = p + 1: decodes to the identity
    not_on_curve = None
    for y in range(2, 100):
        if ed.decode(y.to_bytes(32, "little")) is None:
            not_on_curve = y.to_bytes(32, "little")
            break
    out += [
        ("R replaced", pk, m, so.public_key(g, 7) + sig[32:]),
        ("s replaced", pk, m, sig[:32] + _s_bytes(g, (s + 1) % L)),
        ("wrong key", so.public_key(g, x + 1), m, sig),
        ("s + l", pk, m, sig[:32] + _s_bytes(g, s + L)),
        ("R small order", pk, m, t8 + sig[32:]),
        ("R non-canonical", pk, m, noncanon + sig[32:]),
        ("R not on curve", pk, m, not_on_curve + sig[32:]),
        ("R not on curve, s + l", pk, m, not_on_curve + _s_bytes(g, s + L)),
        ("R small order, s + l", pk, m, t8 + _s_bytes(g, s + L)),
        ("key small order", t8, m, sig),
        ("key non-canonical", noncanon, m, sig),
        ("key not on curve", not_on_curve, m, sig),
        ("key B", so.public_key(g, 1), m, so.sign(g, 1, m, 5)),
        ("key -B", so.public_key(g, L - 1), m, so.sign(g, L - 1, m, 5)),
        ("key 2B", so.public_key(g, 2), m, so.sign(g, 2, m, 9)),
        ("s = l - 1 invalid", pk, m, sig[:32] + _s_bytes(g, L - 1)),
    ]
    return tuple(out)


def cases(group: str) -> tuple:
    return ed_cases() if group == "ed25519" else bls_cases(group)


def length_cases(group: str) -> list:
    """signatures one byte short and one byte long: the reference's length error, answered on the host"""
    pl = so.POINT_LEN[group]
    name, pk, m, sig = cases(group)[0]
    return [("short", pk, m, sig[:-1]), ("long", pk, m, sig + b"\x00"), ("empty", pk, m, b""),
            ("point only", pk, m, sig[:pl])]
