"""Boneh-Franklin IBE (CCA) on BLS12-381, restated from the reference (encrypt/ibe/ibe.go:51-309) with Hash = SHA-256.

  H2(gt)         = SHA256("IBE-H2" || GT.MarshalBinary)[:len]                       (gtToHash, ibe.go:291-307)
  H4(sigma)      = SHA256("IBE-H4" || sigma)[:len]                                  (h4, ibe.go:277-289)
  H3(sigma, msg) : buf = SHA256("IBE-H3" || sigma || msg); for i = 1 .. 65534: h = SHA256(LE16(i) || buf), h[0] >>= 1
                   (toMask = 256 - 255, big-endian scalars), the first h < r                    (h3, ibe.go:234-275)

Points travel as compressed kyber wire bytes.  The pairing runs in C (oracle/cpu_ref.c), whose GT bytes are those of
bls12381.pairing_reference, the reference back-ends' convention.  TEST INFRASTRUCTURE (imports oracle.cpu_ref)."""
from __future__ import annotations
import hashlib

from . import bls12381 as o
from . import cpu_ref
from .h2c_bls12381 import DST_G1, hash_to_g1
from .h2c_bls12381_g2 import DST_G2, hash_to_g2

OK, PROOF, POINT = 0, 1, 2          # B2K_IBE_* of include/b2kyber.h
MAX_LEN = 32                        # s.Hash().Size()

_lib = None


def _xor(a: bytes, b: bytes) -> bytes:
    assert len(a) == len(b)
    return bytes(x ^ y for x, y in zip(a, b))


def h2(gt: bytes, n: int) -> bytes:
    return hashlib.sha256(b"IBE-H2" + gt).digest()[:n]


def h4(sigma: bytes, n: int) -> bytes:
    return hashlib.sha256(b"IBE-H4" + sigma).digest()[:n]


def h3_iterations(sigma: bytes, msg: bytes):
    """(r, i): the scalar and the counter that produced it; (None, 65535) when no candidate is below r."""
    buf = hashlib.sha256(b"IBE-H3" + sigma + msg).digest()
    for i in range(1, 65535):
        h = bytearray(hashlib.sha256(i.to_bytes(2, "little") + buf).digest())
        h[0] >>= 1
        v = int.from_bytes(h, "big")
        if v < o.R:
            return v, i
    return None, 65535


def h3(sigma: bytes, msg: bytes):
    return h3_iterations(sigma, msg)[0]


def pair(p1, q2):
    """Suite.Pair(p1, q2) as an Fp12 element (oracle representation)."""
    global _lib
    if _lib is None:
        _lib = cpu_ref.load()
    return o.gt_from_bytes(cpu_ref.pair(_lib, o.g1_to_affine_bytes(p1), o.g2_to_affine_bytes(q2)))


def _decode(group: int, b: bytes):
    """(point, True) or (None, False) -- UnmarshalBinary with the subgroup check."""
    try:
        return (o.g1_decompress(b) if group == 1 else o.g2_decompress(b)), True
    except ValueError:
        return None, False


def _decrypt(u_group: int, priv: bytes, u: bytes, v: bytes, w: bytes):
    """(msg, status) -- DecryptCCAonG1 (u_group 1) / DecryptCCAonG2 (u_group 2); msg is zeroed unless OK."""
    n = len(w)
    assert n <= MAX_LEN and len(v) == n
    key, ok = _decode(3 - u_group, priv)
    if not ok:
        raise ValueError("the private key does not decode")
    U, ok = _decode(u_group, u)
    if not ok:
        return bytes(n), POINT
    g = pair(U, key) if u_group == 1 else pair(key, U)
    sigma = _xor(v, h2(o.gt_to_bytes(g), n))
    msg = _xor(w, h4(sigma, n))
    r = h3(sigma, msg)
    if r is None:
        return bytes(n), PROOF
    rp = o.g1_mul(r) if u_group == 1 else o.g2_mul(r)
    if rp != U:
        return bytes(n), PROOF
    return msg, OK


def _encrypt(u_group: int, master: bytes, ident: bytes, msg: bytes, sigma: bytes, dst: bytes = None):
    """(U, V, W) with U compressed -- EncryptCCAonG1 (u_group 1) / EncryptCCAonG2 (u_group 2) with the caller's sigma."""
    n = len(msg)
    assert n <= MAX_LEN and len(sigma) == n
    M, ok = _decode(u_group, master)
    if not ok:
        raise ValueError("the master key does not decode")
    if u_group == 1:
        gid = pair(M, hash_to_g2(ident, DST_G2 if dst is None else dst))
    else:
        gid = pair(hash_to_g1(ident, DST_G1 if dst is None else dst), M)
    r = h3(sigma, msg)
    if r is None:
        raise ValueError("rejection sampling failure")
    U = o.g1_compress(o.g1_mul(r)) if u_group == 1 else o.g2_compress(o.g2_mul(r))
    V = _xor(sigma, h2(o.gt_to_bytes(o.f12_pow(gid, r)), n))
    W = _xor(msg, h4(sigma, n))
    return U, V, W


def decrypt_cca_g1(priv96: bytes, u48: bytes, v: bytes, w: bytes):
    return _decrypt(1, priv96, u48, v, w)


def decrypt_cca_g2(priv48: bytes, u96: bytes, v: bytes, w: bytes):
    return _decrypt(2, priv48, u96, v, w)


def encrypt_cca_g1(master48: bytes, ident: bytes, msg: bytes, sigma: bytes, dst: bytes = None):
    return _encrypt(1, master48, ident, msg, sigma, dst)


def encrypt_cca_g2(master96: bytes, ident: bytes, msg: bytes, sigma: bytes, dst: bytes = None):
    return _encrypt(2, master96, ident, msg, sigma, dst)


def keypair(u_group: int, s: int, ident: bytes, dst: bytes = None):
    """(master, private) for the master secret s: OnG1 master = s G1, private = s H_G2(id); OnG2 the mirror."""
    if u_group == 1:
        return o.g1_compress(o.g1_mul(s)), o.g2_compress(o.g2_mul(s, hash_to_g2(ident, DST_G2 if dst is None else dst)))
    return o.g2_compress(o.g2_mul(s)), o.g1_compress(o.g1_mul(s, hash_to_g1(ident, DST_G1 if dst is None else dst)))
