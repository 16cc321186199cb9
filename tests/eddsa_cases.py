"""Ed25519 verification cases shared by the oracle, emulation and GPU tests: the committed fixtures (tests/golden/eddsa_*)
and crafted cases for every rejection path of VerifyWithChecks.  Each case is (name, pk, msg, sig)."""
from __future__ import annotations
import gzip
import hashlib
import json
import os

from oracle import ed25519 as ed
from oracle import eddsa as oe

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return json.load(open(os.path.join(GOLDEN, name)))


def rfc8032():
    return [(bytes.fromhex(c["seed"]), bytes.fromhex(c["pk"]), bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"]))
            for c in _load("eddsa_vectors.json")["rfc8032"]]


def sign_input():
    with gzip.open(os.path.join(GOLDEN, "eddsa_sign_input.json.gz"), "rt") as f:
        cases = json.load(f)["cases"]
    return [(bytes.fromhex(c["seed"]), bytes.fromhex(c["pk"]), bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"])) for c in cases]


def wycheproof():
    """-> [(tcId, pk, msg, sig, valid)]"""
    return [(c["tcId"], bytes.fromhex(c["pk"]), bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"]), c["result"] == "valid")
            for c in _load("eddsa_wycheproof.json")["cases"]]


def weak_keys():
    return [bytes.fromhex(w) for w in _load("eddsa_vectors.json")["weak_keys"]]


def inline():
    """the byte vectors of eddsa_test.go's rejection tests, each applied to RFC 8032 vector 2 (as those tests apply them to a
    fresh valid signature) -> [(name, pk, msg, sig, expected error name)]"""
    _, pk0, msg0, sig0 = rfc8032()[1]
    out = []
    for i, c in enumerate(_load("eddsa_vectors.json")["inline"]["cases"]):
        name = "%s/%d" % (c["test"], i)
        if c["kind"] == "full":
            out.append((name, bytes.fromhex(c["pk"]), bytes.fromhex(c["msg"]), bytes.fromhex(c["sig"]), c["expect"]))
            continue
        v = bytes.fromhex(c["bytes"])
        pk, sig = pk0, sig0
        if c["kind"] == "replace_r":
            sig = v + sig0[32:]
        elif c["kind"] == "replace_pk":
            pk = v
        elif c["kind"] == "add_to_s":
            s = (int.from_bytes(sig0[32:], "little") + int.from_bytes(v, "little")) % (1 << 256)
            sig = sig0[:32] + s.to_bytes(32, "little")
        out.append((name, pk, msg0, sig, c["expect"]))
    return out


def _flip(b: bytes, bit: int) -> bytes:
    x = bytearray(b)
    x[bit >> 3] ^= 1 << (bit & 7)
    return bytes(x)


def _y_bytes(y: int, sign: int) -> bytes:
    return (y | (sign << 255)).to_bytes(32, "little")


def no_sqrt_y() -> int:
    """the smallest y for which no x exists"""
    y = 2
    while ed.decode(_y_bytes(y, 0)) is not None:
        y += 1
    return y


def cofactor_cases(count: int = 16):
    """key A = a B + T8 (T8 of order 8: A is not small order); signatures by a under A's bytes verify, cofactorless,
    exactly when 8 | h.  -> [(name, pk, msg, sig, h % 8)] with at least one h = 0 (mod 8) and several h != 0."""
    a, prefix, _ = oe.keygen(b"\x42" * 32)
    A = ed.encode(ed.add(ed.scalar_mult(a), oe.order8_point()))
    out, zero = [], 0
    i = 0
    while len(out) < count or zero == 0:
        msg = b"cofactor %d" % i
        i += 1
        sig = oe.sign_raw(a, prefix, A, msg)
        h8 = oe.h_scalar(sig[:32], A, msg) % 8
        if h8 == 0:
            zero += 1
            if zero > 2:
                continue
        elif len(out) >= count:
            continue
        out.append(("cofactor/%d" % i, A, msg, sig, h8))
    return out


def crafted():
    """every rejection path, with the key, message and signature of RFC 8032 vector 2 as the valid base case"""
    _, pk, msg, sig = rfc8032()[1]
    R, s = sig[:32], int.from_bytes(sig[32:], "little")
    P, L = ed.P, ed.L
    out = [("valid", pk, msg, sig), ("empty message", *rfc8032()[0][1:])]
    out.append(("s + l", pk, msg, R + ((s + L) % (1 << 256)).to_bytes(32, "little")))
    out.append(("s bit 255", pk, msg, R + (s | 1 << 255).to_bytes(32, "little")))
    out.append(("s = l", pk, msg, R + L.to_bytes(32, "little")))
    out.append(("s = l - 1", pk, msg, R + (L - 1).to_bytes(32, "little")))
    non_canon = [b"\xef" + b"\xff" * 31] + [_y_bytes(y, sg) for y in (P, P + 1, P + 18) for sg in (0, 1)]
    bad_y = no_sqrt_y()
    small = [_y_bytes(int.from_bytes(w, "little"), sg) for w in weak_keys() for sg in (0, 1)]
    for tag, vals in (("non-canonical", non_canon), ("no sqrt", [_y_bytes(bad_y, 0), _y_bytes(bad_y, 1)]), ("small order", small)):
        for j, v in enumerate(vals):
            out.append(("R %s %d" % (tag, j), pk, msg, v + sig[32:]))
            out.append(("pk %s %d" % (tag, j), v, msg, sig))
    for bit in (0, 7, 8 * len(msg) - 1):
        out.append(("msg bit %d" % bit, pk, _flip(msg, bit), sig))
    for bit in (0, 100, 254, 255):
        out.append(("R bit %d" % bit, pk, msg, _flip(R, bit) + sig[32:]))
    for bit in (0, 100, 252, 253):
        out.append(("s bit %d" % bit, pk, msg, R + _flip(sig[32:], bit)))
    out.append(("pk bit 0", _flip(pk, 0), msg, sig))
    out += [c[:4] for c in cofactor_cases()]
    return out


def lengths_cases():
    """messages whose hashed input (64 + m bytes) sits around the SHA-512 padding boundaries, and one of 1 MiB"""
    seed = hashlib.sha256(b"lengths").digest()
    out = []
    for m in (47, 48, 49, 64, 175, 176, 1023, 1 << 20):
        msg = bytes((i * 131 + m) & 0xff for i in range(m))
        out.append(("m=%d" % m, oe.keygen(seed)[2], msg, oe.sign(seed, msg)))
    return out
