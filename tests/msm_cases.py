"""Input sets and expected values for the MSM tests of every group the Pippenger template is instantiated for.

Shared by tests/test_gpu_msm_curves.py (the device pipeline) and tests/test_host_emulation.py (the same kernel bodies
compiled for the CPU), so the input construction and the oracle side are the same code in both.

Points are P_i = a_i G.  The expected MSM is then ((sum s_i a_i) mod r) G: one oracle multiplication per case, which keeps
the G2 cases cheap in Python.  Infinity is the all-zero operand in every group."""
from __future__ import annotations

import random
from dataclasses import dataclass
from typing import Callable

from oracle import bls12381 as _bls
from oracle import bn254 as _bn254
from oracle import bn254_pairing as _bn254_g2
from oracle import bn256 as _bn256


@dataclass(frozen=True)
class Group:
    name: str
    r: int                          # group order (scalars must be below it)
    p: int                          # base field prime
    scalar_bits: int                # bit length the device plans its windows for (SCALAR_BITS of the curve config)
    in_bytes: int                   # operand (affine) bytes
    out_bytes: int                  # MSM output bytes
    coord_bytes: int                # bytes of one big-endian base-field element in the operand encoding
    canonical: bool                 # the operand check refuses a coordinate >= p (wire_canonical)
    mul: Callable                   # k -> k G (oracle point; None = infinity)
    encode: Callable                # oracle point -> MSM output bytes
    operand: Callable               # oracle point -> operand bytes

    @property
    def gen(self) -> bytes:
        return self.operand(self.mul(1))

    def expected(self, a, s) -> bytes:
        """encode(sum s_i (a_i G)) = encode(((sum s_i a_i) mod r) G)"""
        acc = 0
        for x, y in zip(a, s):
            acc += x * y
        return self.encode(self.mul(acc % self.r))


GROUPS = {
    "bls12381_g1": Group("bls12381_g1", _bls.R, _bls.P, 255, 96, 48, 48, True, _bls.g1_mul, _bls.g1_compress, _bls.g1_to_affine_bytes),
    "bls12381_g2": Group("bls12381_g2", _bls.R, _bls.P, 255, 192, 96, 48, True, _bls.g2_mul, _bls.g2_compress, _bls.g2_to_affine_bytes),
    "bn254_g1": Group("bn254_g1", _bn254.ORDER, _bn254.P, 254, 64, 64, 32, True, _bn254.g1_mul, _bn254.g1_marshal, _bn254.g1_marshal),
    "bn254_g2": Group("bn254_g2", _bn254.ORDER, _bn254.P, 254, 128, 128, 32, True, _bn254_g2.g2_mul, _bn254_g2.g2_marshal,
                      _bn254_g2.g2_marshal),
    "bn256_g1": Group("bn256_g1", _bn256.ORDER, _bn256.P, 256, 64, 64, 32, False, _bn256.g1_mul, _bn256.g1_marshal, _bn256.g1_marshal),
    "bn256_g2": Group("bn256_g2", _bn256.ORDER, _bn256.P, 256, 128, 128, 32, False, _bn256.g2_mul, _bn256.g2_marshal, _bn256.g2_marshal),
}

# BLS12-381 affine output (b2k_bls12381_{g1,g2}_msm_affine): the operand encoding of the sum
AFFINE_ENCODE = {"bls12381_g1": _bls.g1_to_affine_bytes, "bls12381_g2": _bls.g2_to_affine_bytes}


def scalars_to_bytes(vals) -> bytes:
    return b"".join(v.to_bytes(32, "big") for v in vals)


def signed_digits(k: int, c: int, scalar_bits: int):
    """The device's window digits of k (msm.cuh: msm_recode / msm_digit): k + sum_w 2^(c-1) 2^(c w), each c-bit field
    minus 2^(c-1), over W = (scalar_bits + c) // c windows; every digit lies in [-2^(c-1), 2^(c-1) - 1]."""
    W = (scalar_bits + c) // c
    h = 1 << (c - 1)
    sp = k + sum(h << (c * w) for w in range(W))
    return [((sp >> (c * w)) & ((1 << c) - 1)) - h for w in range(W)]


def largest_bucket(scalars, c: int, scalar_bits: int) -> int:
    """entries of the most populated bucket (window, |digit|) for these scalars"""
    counts = {}
    for k in scalars:
        for w, d in enumerate(signed_digits(k, c, scalar_bits)):
            if d:
                counts[(w, abs(d))] = counts.get((w, abs(d)), 0) + 1
    return max(counts.values(), default=0)


# window widths whose largest bucket the edge set fills (the forced c of the plan lists, and a few more)
EDGE_WINDOWS = (4, 5, 7, 8, 12, 13, 16)


def digit_pattern_scalars(r: int, c: int, scalar_bits: int):
    """scalars whose signed digits are -2^(c-1) (the largest bucket, index 2^(c-1) - 1) and 2^(c-1) - 1, under a top digit
    2^(c-1) - 1 at several heights; only those below r are kept"""
    W = (scalar_bits + c) // c
    h = 1 << (c - 1)
    out = []
    for top in (1, W // 2, W - 3, W - 2):
        for digits in ([-h if w % 2 == 0 else h - 1 for w in range(top)], [-h] * top):
            digits = digits + [h - 1]
            k = sum(d << (c * w) for w, d in enumerate(digits))
            if 0 < k < r:
                assert signed_digits(k, c, scalar_bits)[:top + 1] == digits
                out.append(k)
    return out


def edge_scalars(g: Group):
    r = g.r
    base = [0, 1, r - 1, r - 2, (r - 1) // 2]
    for c in EDGE_WINDOWS:
        base += digit_pattern_scalars(r, c, g.scalar_bits)
    return base


SETS = ("uniform", "equal", "plus_minus", "zeros", "small", "one_and_minus_one", "bdn128", "edges")


def build_set(g: Group, name: str, n: int, A, seed: int = 0):
    """(a, s) of input set `name` with n pairs; multipliers come from A (distinct, nonzero, below r).

    uniform            a_i from A, s_i uniform below r
    equal              one (s, P) n times: every window's entries fall in one bucket
    plus_minus         P and -P alternating under one scalar (n even): buckets, slice partials and the total are infinity
    zeros              every third operand at infinity, all under one full-size scalar, the others under scalars < 2^20:
                       the upper windows' buckets hold nothing but infinities
    small              s_i < 2^20: the upper windows are empty and the Horner chain starts from infinity
    one_and_minus_one  s_i in {1, r - 1}
    bdn128             128-bit BDN factors (sign/bdn hashPointToR) + 1
    edges              0, 1, r-1, r-2, (r-1)/2 and digit patterns that fill the largest bucket of several windows
    """
    r = g.r
    rng = random.Random(f"{g.name}/{name}/{n}/{seed}")
    pick = [A[i % len(A)] for i in range(n)]
    if name == "uniform":
        return pick, [rng.randrange(r) for _ in range(n)]
    if name == "equal":
        return [A[0]] * n, [rng.randrange(1 << 200, r)] * n
    if name == "plus_minus":
        assert n % 2 == 0
        k = rng.randrange(1, r)
        return [A[0] if i % 2 == 0 else r - A[0] for i in range(n)], [k] * n
    if name == "zeros":
        big = rng.randrange(1 << 250, r)
        a = [0 if i % 3 == 0 else pick[i] for i in range(n)]
        return a, [big if i % 3 == 0 else rng.randrange(1 << 20) for i in range(n)]
    if name == "small":
        return pick, [rng.randrange(1 << 20) for _ in range(n)]
    if name == "one_and_minus_one":
        return pick, [rng.choice((1, r - 1)) for _ in range(n)]
    if name == "bdn128":
        return pick, [rng.randrange(1 << 128) + 1 for _ in range(n)]
    if name == "edges":
        e = edge_scalars(g)
        return pick, [e[i % len(e)] for i in range(n)]
    raise KeyError(name)


def multipliers(g: Group, count: int, seed: str = "A"):
    """count distinct nonzero multipliers below r (the plus_minus set also uses r - A[0])"""
    rng = random.Random(f"{g.name}/mult/{seed}")
    out, seen = [], set()
    while len(out) < count:
        v = rng.randrange(1, g.r)
        if v not in seen and g.r - v not in seen:
            seen.add(v)
            out.append(v)
    return out


# (window c, reduction chunk m, slice length L) of the host emulation (L = 0: one thread per bucket): the forced windows, chunks
# and slice lengths of the device plans in tests/test_gpu_msm_curves.py, at sizes the CPU runs in seconds
EMUL_PLANS = ((4, 2, 3), (5, 16, 1), (7, 1, 64), (7, 64, 3), (8, 4, 0), (12, 2048, 1))
