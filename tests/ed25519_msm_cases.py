"""Expected values and inputs of the edwards25519 MSM and share/poly tests (CPU oracle tests, host emulation, GPU).

ge_scalar_mult restates the reference's default Point.Mul (group/edwards25519/ge.go:443-502, geScalarMult, varTime off)
literally: 4-bit nibbles of the 32 scalar bytes, the carry pass that makes them signed, the cached table 1..8 A, selectCached
(ge.go:419-433), which selects NOTHING for a digit above 8, and four doublings per nibble.  Below 2^255 it is the plain
product k A; from 2^255 on, a top digit e63 = (k >> 252) + carry above 8 is dropped.  effective_scalar gives the integer the
device multiplies by instead (modulo 8 l, the order of the whole group), so that expected sums of many terms stay one
multiplication of the base point."""
from __future__ import annotations

import random

from oracle import ed25519 as ed

P, L = ed.P, ed.L
IDENTITY = ed.encode(ed.IDENT)          # 01 00 .. 00
ZERO = bytes(32)                        # decodes to a point of order 4 (x^2 = -1), not to the identity
T8 = bytes.fromhex("c7176a703d4dd84fba3c0b760d10670f2a2053fa2c39ccc64ec7fd7792ac037a")   # a point of order 8


def _ext(pt):
    x, y = pt
    return (x, y, 1, x * y % P)


def _neg(q):
    x, y, z, t = q
    return (-x % P, y, z, -t % P)


def _affine(q):
    zi = pow(q[2], P - 2, P)
    return (q[0] * zi % P, q[1] * zi % P)


def nibbles(k_bytes: bytes):
    """e[0..63] of geScalarMult: nibbles, then the carry pass (int8 arithmetic: every value stays within -8..16)"""
    e = []
    for v in k_bytes:
        e += [v & 15, (v >> 4) & 15]
    carry = 0
    for i in range(63):
        e[i] += carry
        carry = (e[i] + 8) >> 4
        e[i] -= carry << 4
    e[63] += carry
    return e


def ge_scalar_mult(k_bytes: bytes, point):
    """geScalarMult(k, A) for a decoded point A (x, y); returns the affine result"""
    e = nibbles(k_bytes)
    a = _ext(point)
    tab = [a]                                               # Ai[0..7] = 1A .. 8A
    for _ in range(7):
        tab.append(ed._ext_add(a, tab[-1]))

    def select(b):
        c = (0, 1, 1, 0)                                    # c.Zero(): the identity
        for i in range(8):
            if abs(b) == i + 1:
                c = tab[i]
        return _neg(c) if b < 0 else c

    t = ed._ext_add((0, 1, 1, 0), select(e[63]))
    for i in range(62, -1, -1):
        for _ in range(4):
            t = ed._ext_add(t, t)
        t = ed._ext_add(t, select(e[i]))
    return _affine(t)


def top_digit(k: int) -> int:
    return nibbles(k.to_bytes(32, "little"))[63]


_K63 = sum(8 << (4 * i) for i in range(63))


def top_digit_fast(k: int) -> int:
    """e63 in closed form: the carry pass is the recoding low + 0x88..8 (63 nibbles), its carry the bit 252 of that sum"""
    return (k >> 252) + (((k & ((1 << 252) - 1)) + _K63) >> 252)


def effective_scalar(k: int) -> int:
    """the integer geScalarMult multiplies by, modulo 8 l: k itself up to a top digit of 8, else k - e63 2^252"""
    if k < 1 << 255:
        return k
    e63 = top_digit_fast(k)
    return k if e63 <= 8 else (k - (e63 << 252)) % (8 * L)


def crafted_high_scalars(rng: random.Random):
    """scalars >= 2^255 on both sides of the rule: e63 = 8 (kept), 9 and 16 (dropped), a[31] = 0x8f with and without a
    carry out of the lower nibbles, and the largest values"""
    low = lambda: rng.getrandbits(240)                                      # bytes 0..29; nibble 59 < 8 keeps carries out of 60
    low = (lambda f: lambda: f() & ~(0x8 << 236))(low)
    return [
        (0x80 << 248) | low(),                    # e63 = 8: kept
        (0x80 << 248) | (0xf0 << 240) | low(),    # 0x80 with a carry from a[30] = 0xf0 (nibble 62 becomes 1): still 8
        (0x8f << 248) | low(),                    # a[31] = 0x8f, no carry into nibble 62: digit -1, e63 = 9
        (0x8f << 248) | (0xf0 << 240) | low(),    # a[31] = 0x8f with a carry into nibble 62: digit 0, e63 = 9
        (0x97 << 248) | low(),                    # e63 = 9 without any carry
        (0xf8 << 248) | low(),                    # e63 = 16 from the nibble 0xf and nibble 62 = 8
        (1 << 256) - 1,                           # e63 = 16
        (0xff << 248) | low(),                    # e63 = 16
    ]


def mixed_point(i: int) -> bytes:
    """(i + 2) B + T8: a point with a torsion part"""
    return ed.encode(ed.add(ed.scalar_mult(i + 2), ed.decode(T8)))


# Every point of the curve is a B + b T8 (a mod l, b mod 8): T8 generates the torsion subgroup.  Inputs are built that way,
# so that the expected MSM is two multiplications whatever n is.
def point(a: int, b: int = 0) -> bytes:
    return ed.encode(ed.add(ed.scalar_mult(a % L), ed.scalar_mult(b % 8, ed.decode(T8))))


ZERO_B = next(b for b in range(8) if point(0, b) == ZERO)     # the all-zero encoding is a pure torsion point


def msm_expected(scalars, ab) -> bytes:
    """encode(sum_i geScalarMult(k_i, a_i B + b_i T8))"""
    eff = [effective_scalar(k) for k in scalars]
    return point(sum(e * a for e, (a, _) in zip(eff, ab)), sum(e * b for e, (_, b) in zip(eff, ab)))


def le(vals) -> bytes:
    return b"".join(v.to_bytes(32, "little") for v in vals)


SETS = ("uniform", "equal", "plus_minus", "zeros", "small", "high", "mixed")


def build_set(name: str, n: int, seed: int = 0):
    """(scalars, ab) of input set `name` with n pairs; the points are a_i B + b_i T8 (points(ab) encodes them)

    uniform     random 256-bit scalars (some at or above 2^255) on prime-order points
    equal       one (k, P) n times: every window's entries fall in one bucket (a cosi-style sum with unit scalars is the same)
    plus_minus  P and -P alternating under one scalar: buckets, slice partials and the total are the identity
    zeros       every third point the identity (01 00..00) or the all-zero encoding (order 4), the rest under scalars < 2^20
    small       scalars < 2^20: the upper windows are empty
    high        scalars >= 2^255 on both sides of the top-digit rule, on points with torsion parts
    mixed       random scalars on points a B + b T8 of every order
    """
    rng = random.Random(f"ed25519/{name}/{n}/{seed}")
    a_pool = [rng.randrange(1, L) for _ in range(64)]
    pick = lambda: a_pool[rng.randrange(len(a_pool))]
    if name == "uniform":
        return [rng.getrandbits(256) for _ in range(n)], [(pick(), 0) for _ in range(n)]
    if name == "equal":
        return [rng.getrandbits(253)] * n, [(a_pool[0], 0)] * n
    if name == "plus_minus":
        k = rng.getrandbits(256)
        return [k] * n, [(a_pool[0], 0) if i % 2 == 0 else (L - a_pool[0], 0) for i in range(n)]
    if name == "zeros":
        ab = [((0, 0) if i % 6 == 0 else (0, ZERO_B)) if i % 3 == 0 else (pick(), 0) for i in range(n)]
        return [rng.getrandbits(256) if i % 3 == 0 else rng.getrandbits(20) for i in range(n)], ab
    if name == "small":
        return [rng.getrandbits(20) for _ in range(n)], [(pick(), 0) for _ in range(n)]
    if name == "high":
        crafted = crafted_high_scalars(rng)
        return [crafted[i % len(crafted)] if i % 2 == 0 else (1 << 255) | rng.getrandbits(255) for i in range(n)], \
               [(pick(), rng.randrange(8)) for _ in range(n)]
    if name == "mixed":
        return [rng.getrandbits(256) for _ in range(n)], [(pick(), rng.randrange(8)) for _ in range(n)]
    raise KeyError(name)


def points(ab) -> bytes:
    cache = {}
    out = []
    for x in ab:
        if x not in cache:
            cache[x] = point(*x)
        out.append(cache[x])
    return b"".join(out)
