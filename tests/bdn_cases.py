"""Cases of the sign/bdn batch (test infrastructure): masks and what each mask's aggregate key must be.

  aggregate_public_keys  AggregatePublicKeys over cached terms (sign/bdn/bdn.go:166-181 with mask.go:34-64): the plain sum of the
                         terms whose bit is set, bit i of byte i/8 least significant bit first (mask.go:88-97), positions >= n
                         ignored; the group law is a parameter, so it serves every curve of the oracle.
  Rosters come from seeded secret keys x_i.  The expected aggregate key of a mask is (sum over enabled i of (c_i + 1) x_i) times
  the base point and a valid aggregate signature is that scalar times H(m): one fixed-base / point multiplication per mask, so
  the device's term additions are checked against a path that never adds terms.
"""
from __future__ import annotations
import random


def bit(mask: bytes, i: int) -> bool:
    return (mask[i >> 3] >> (i & 7)) & 1 == 1


def mask_of(n: int, enabled) -> bytes:
    out = bytearray((n + 7) // 8)
    for i in enabled:
        out[i >> 3] |= 1 << (i & 7)
    return bytes(out)


def aggregate_public_keys(terms, mask: bytes, n: int, add, zero=None):
    """the masked sum of terms[0..n) with the reference's bit order (bits at positions >= n ignored)"""
    acc = zero
    for i in range(n):
        if bit(mask, i):
            acc = add(acc, terms[i])
    return acc


def edge_masks(n: int, rng: random.Random):
    """empty, single-bit (first, last), full, popcount exactly n/2 and n/2 + 1, and ignored bits beyond n"""
    half = rng.sample(range(n), n // 2)
    rest = [i for i in range(n) if i not in set(half)]
    out = [mask_of(n, []), mask_of(n, [0]), mask_of(n, [n - 1]), mask_of(n, range(n)), mask_of(n, half),
           mask_of(n, half + rest[:1])]
    if n % 8:
        junk = bytearray(mask_of(n, rng.sample(range(n), n // 3)))
        junk[-1] |= (0xFF << (n % 8)) & 0xFF                # bits at positions >= n: ignored
        out.append(bytes(junk))
    return out


def random_masks(n: int, m: int, rng: random.Random):
    """m masks at densities spread over 0..1 (so both the direct and the complemented sums are exercised)"""
    out = []
    for k in range(m):
        p = rng.choice([0.02, 0.2, 0.45, 0.5, 0.55, 2 / 3, 0.9, 0.98, rng.random()])
        out.append(mask_of(n, [i for i in range(n) if rng.random() < p]))
    return out


def mask_scalar(factors, xs, mask: bytes, n: int, order: int) -> int:
    """sum over enabled i of (c_i + 1) x_i mod the group order"""
    return sum(factors[i] * xs[i] for i in range(n) if bit(mask, i)) % order


def scalars_be(vals, order: int) -> bytes:
    return b"".join((v % order).to_bytes(32, "big") for v in vals)
