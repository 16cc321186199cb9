"""CPU ORACLE (test infrastructure, NOT product code) -- edwards25519 Point.Mul and the reference's seeded RNG.

Restates, from the in-tree reference (group/edwards25519 is a ref10 port; the group law fixes the result):
  point.Mul             group/edwards25519/point.go:235-258  (nil base -> B; raw 256-bit little-endian scalar,
                        no reduction on UnmarshalBinary: scalar.go:226-233, read as geScalarMult's signed
                        nibbles: a top digit above 8 selects nothing -> effective_scalar)
  geScalarMult / Base / Vartime   ge.go:443-502, :373-417, ge_mult_vartime.go:11-73 -> scalar_mult()
  ToBytes / FromBytes   ge.go:99-107, :110-150 (y little-endian, sign(x) in bit 255; non-canonical y accepted)
  Scalar.Pick           scalar.go:180-185 -> random.Int(l) util/random/rand.go:19-46 (mask to bitlen, big-endian,
                        retry while >= l), stored little-endian
  blake2xb.New(nil)     xof/blake2xb/blake.go:19,81-102 (BLAKE2Xb, unkeyed, unknown output length)
Pinned by the reference's own KAT: examples/dh_test.go:17-49 (shared secret 80ea238c...51282847), reproduced
in tests/test_oracle_ed25519.py, and cross-checked against libsodium (PyNaCl) where it is installed.
BASELINE configs[0] ("edwards25519 batch of 1024 Point.Mul ... on CPU") is a parity case built on this module.
"""
from __future__ import annotations
import struct

P = 2 ** 255 - 19
L = 2 ** 252 + 27742317777372353535851937790883648493
D = -121665 * pow(121666, P - 2, P) % P
SQRT_M1 = pow(2, (P - 1) // 4, P)
BY = 4 * pow(5, P - 2, P) % P


def _recover_x(y: int, sign: int):
    u, v = (y * y - 1) % P, (D * y * y + 1) % P
    x = u * pow(v, 3, P) % P * pow(u * pow(v, 7, P) % P, (P - 5) // 8, P) % P     # (u v^3)(u v^7)^((p-5)/8), ge.go:126-134
    vxx = v * x * x % P
    if vxx != u:
        if vxx != (-u) % P:
            return None
        x = x * SQRT_M1 % P
    if (x & 1) != sign:
        x = (-x) % P
    return x


BX = _recover_x(BY, 0)
BASE = (BX, BY)
IDENT = (0, 1)


def add(p1, p2):
    x1, y1 = p1
    x2, y2 = p2
    t = D * x1 * x2 % P * y1 % P * y2 % P
    x3 = (x1 * y2 + x2 * y1) * pow(1 + t, P - 2, P) % P
    y3 = (y1 * y2 + x1 * x2) * pow(1 - t, P - 2, P) % P
    return (x3, y3)


def _ext_add(a, b):
    x1, y1, z1, t1 = a
    x2, y2, z2, t2 = b
    A = (y1 - x1) * (y2 - x2) % P
    B = (y1 + x1) * (y2 + x2) % P
    C = 2 * D * t1 * t2 % P
    Dd = 2 * z1 * z2 % P
    E, F, G, H = B - A, Dd - C, Dd + C, B + A
    return (E * F % P, G * H % P, F * G % P, E * H % P)


def scalar_mult(k: int, pt=BASE):
    """k * pt for ANY non-negative integer k (the reference multiplies by the raw 256-bit integer)."""
    acc = (0, 1, 1, 0)
    q = (pt[0], pt[1], 1, pt[0] * pt[1] % P)
    for bit in bin(k)[2:] if k else "":
        acc = _ext_add(acc, acc)
        if bit == "1":
            acc = _ext_add(acc, q)
    zi = pow(acc[2], P - 2, P)
    return (acc[0] * zi % P, acc[1] * zi % P)


def encode(pt) -> bytes:
    x, y = pt
    return (y | ((x & 1) << 255)).to_bytes(32, "little")


def decode(b: bytes):
    """FromBytes (ge.go:110-150): y may be non-canonical (reduced mod p); None if not on the curve."""
    if len(b) != 32:
        raise ValueError("wrong length")
    v = int.from_bytes(b, "little")
    y, sign = (v & ((1 << 255) - 1)) % P, v >> 255
    x = _recover_x(y, sign)
    if x is None:
        return None
    if x == 0 and sign == 1:
        x = 0
    return (x, y)


_K63 = sum(8 << (4 * i) for i in range(63))


def top_digit(k: int) -> int:
    """e63 of geScalarMult's signed-nibble recoding (ge.go:443-466), in closed form: the carry pass over the 63 lower nibbles
    is the sum low + 0x88..8 (63 nibbles), its carry into the top nibble bit 252 of that sum"""
    return (k >> 252) + (((k & ((1 << 252) - 1)) + _K63) >> 252)


def effective_scalar(k: int) -> int:
    """the integer geScalarMult (and geScalarMultBase) multiplies by, modulo 8 l, the order of the whole group: k itself up to a
    top digit of 8 (every k below 2^255), else k - e63 2^252, because selectCached (ge.go:419-433) selects nothing for it"""
    e63 = top_digit(k)
    return k if e63 <= 8 else (k - (e63 << 252)) % (8 * L)


def point_mul(scalar_le: bytes, point32: bytes | None) -> bytes:
    """point.Mul(s, P).MarshalBinary(): s is the raw little-endian 32-byte scalar, point32 = None means base."""
    k = effective_scalar(int.from_bytes(scalar_le, "little"))
    pt = BASE if point32 is None else decode(point32)
    if pt is None:
        raise ValueError("invalid point")
    return encode(scalar_mult(k, pt))


# ---- BLAKE2b / BLAKE2Xb (the reference's deterministic test RNG) ----------------------------------------------
_IV = [0x6a09e667f3bcc908, 0xbb67ae8584caa73b, 0x3c6ef372fe94f82b, 0xa54ff53a5f1d36f1,
       0x510e527fade682d1, 0x9b05688c2b3e6c1f, 0x1f83d9abfb41bd6b, 0x5be0cd19137e2179]
_SIGMA = [[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15], [14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3],
          [11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4], [7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8],
          [9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13], [2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9],
          [12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11], [13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10],
          [6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5], [10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0]]
_M64 = (1 << 64) - 1


def _rotr(x, n): return ((x >> n) | (x << (64 - n))) & _M64


def _blake2b(data: bytes, param: bytes, outlen: int) -> bytes:
    h = [iv ^ p for iv, p in zip(_IV, struct.unpack("<8Q", param))]
    blocks = [data[i:i + 128] for i in range(0, len(data), 128)] or [b""]
    t = 0
    for bi, blk in enumerate(blocks):
        last = bi == len(blocks) - 1
        t += len(blk)
        m = list(struct.unpack("<16Q", blk.ljust(128, b"\x00")))
        v = h + _IV[:]
        v[12] ^= t & _M64
        v[13] ^= t >> 64
        if last:
            v[14] ^= _M64
        for r in range(12):
            s = _SIGMA[r % 10]
            for i, (a, b, c, d) in enumerate(((0, 4, 8, 12), (1, 5, 9, 13), (2, 6, 10, 14), (3, 7, 11, 15),
                                              (0, 5, 10, 15), (1, 6, 11, 12), (2, 7, 8, 13), (3, 4, 9, 14))):
                v[a] = (v[a] + v[b] + m[s[2 * i]]) & _M64; v[d] = _rotr(v[d] ^ v[a], 32)
                v[c] = (v[c] + v[d]) & _M64; v[b] = _rotr(v[b] ^ v[c], 24)
                v[a] = (v[a] + v[b] + m[s[2 * i + 1]]) & _M64; v[d] = _rotr(v[d] ^ v[a], 16)
                v[c] = (v[c] + v[d]) & _M64; v[b] = _rotr(v[b] ^ v[c], 63)
        h = [h[i] ^ v[i] ^ v[i + 8] for i in range(8)]
    return struct.pack("<8Q", *h)[:outlen]


def _param(digest, fanout, depth, leaf, node_offset, xof_len, node_depth, inner):
    return struct.pack("<BBBBIIIBB14x16x16x", digest, 0, fanout, depth, leaf, node_offset, xof_len, node_depth, inner)


class Blake2Xb:
    """blake2xb.New(seed): unkeyed BLAKE2Xb with unknown output length; read() yields the key stream that
    XORKeyStream applies (on a zero buffer that is the stream itself)."""

    def __init__(self, seed: bytes = b""):
        self.h0 = _blake2b(seed, _param(64, 1, 1, 0, 0, 0xFFFFFFFF, 0, 0), 64)
        self.block, self.buf = 0, b""

    def read(self, n: int) -> bytes:
        while len(self.buf) < n:
            self.buf += _blake2b(self.h0, _param(64, 0, 0, 64, self.block, 0xFFFFFFFF, 0, 64), 64)
            self.block += 1
        out, self.buf = self.buf[:n], self.buf[n:]
        return out


def pick_scalar(rng: Blake2Xb) -> bytes:
    """Scalar.Pick: random.Int(l) then little-endian (scalar.go:180-185, util/random/rand.go:19-46)."""
    while True:
        b = bytearray(rng.read(32))
        b[0] &= 0xFF >> (8 - (L.bit_length() & 7)) if L.bit_length() & 7 else 0xFF
        v = int.from_bytes(b, "big")
        if v < L:
            return v.to_bytes(32, "little")
