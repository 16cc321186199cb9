"""GPU: the GT entry points (b2k_*_gt_mul, gt_inv, gt_exp, final_exp / finalize) on crafted Fp12 elements, through the public API,
against the oracles' f12_* functions.  These entry points accept ANY element with coefficients below p, not only pairing values:
elements with one nonzero coefficient, coefficients equal to p - 1, embedded Fp / Fp2 / Fp6 elements, random non-unitary elements and
zero, in batches of 1, 63, 64, 65 and 4097 (one element past the 4096 cap of the warp-cooperative exponentiation).  Unlike the field
harness (test_gpu_field_arith.py), this runs the arithmetic inside the kernels that ship, in their own inlining context."""
import functools
import random

import pytest

from oracle import bls12381 as o
from oracle import bn254, bn256, bn254_pairing as b4, bn256_pairing as b6

pytestmark = pytest.mark.gpu

SIZES = [1, 63, 64, 65, 4097]
COOP_DEFAULT = 10240                       # b2k_ctx.h: the library's default cap of the warp-cooperative kernels
Z6 = ((0, 0), (0, 0), (0, 0))
ZERO = (Z6, Z6)


class Curve:
    def __init__(self, name, p, order, ns, to_bytes, final):
        self.name, self.p, self.order, self.ns, self.to_bytes, self.final = name, p, order, ns, to_bytes, final


CURVES = {
    "bls12381": Curve("bls12381", o.P, o.R, o, o.gt_to_bytes, o.final_exponentiation_cubed),
    "bn254": Curve("bn254", bn254.P, bn254.ORDER, b4, b4.gt_to_bytes, b4.final_exponentiation),
    "bn256": Curve("bn256", bn256.P, bn256.ORDER, b6, b6.gt_to_bytes, b6.final_exponentiation),
}


def from_flat(v):
    f2 = [(v[2 * i], v[2 * i + 1]) for i in range(6)]
    return ((f2[0], f2[1], f2[2]), (f2[3], f2[4], f2[5]))


@functools.lru_cache(maxsize=None)
def pool(name):
    """the crafted elements: one nonzero coefficient (1, p - 1 or random) in each of the 12 slots, all coefficients p - 1, embedded
    Fp / Fp2 / Fp6 elements, random non-unitary elements, edge-valued mixes, and zero last"""
    c = CURVES[name]
    p = c.p
    rng = random.Random(f"gt-edges/{name}")
    out = []
    for k in range(12):
        for val in (1, p - 1, rng.randrange(1, p)):
            out.append(from_flat([0] * k + [val] + [0] * (11 - k)))
    out.append(from_flat([p - 1] * 12))
    out.append(from_flat([p - 1, 1] * 6))
    for width in (1, 2, 6):
        for _ in range(3):
            out.append(from_flat([rng.randrange(p) for _ in range(width)] + [0] * (12 - width)))
    edge = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2]
    for _ in range(8):
        out.append(from_flat([rng.choice(edge) for _ in range(12)]))
    for _ in range(16):
        out.append(from_flat([rng.randrange(p) for _ in range(12)]))
    out.append(ZERO)
    return out


def batch(name, n, shift=0):
    """n elements drawn from the pool in a stride that mixes the kinds inside every warp; a batch of one is the zero element"""
    P = pool(name)
    if n == 1:
        return [P[-1]]
    return [P[(7 * i + shift) % len(P)] for i in range(n)]


def enc(c, elems):
    return b"".join(c.to_bytes(e) for e in elems)


@functools.lru_cache(maxsize=None)
def f12_mul(name, a, b):
    return CURVES[name].ns.f12_mul(a, b)


@functools.lru_cache(maxsize=None)
def f12_inv(name, a):
    return ZERO if a == ZERO else CURVES[name].ns.f12_inv(a)


@functools.lru_cache(maxsize=None)
def f12_pow(name, a, k):
    ns = CURVES[name].ns
    return ns.F12_ONE if k == 0 else ns.f12_pow(a, k)   # k = 0: one, also for the zero element (the kernels start from one)


@functools.lru_cache(maxsize=None)
def final(name, a):
    return CURVES[name].final(a)


def first_difference(got, want, size, elems, what):
    for i in range(len(got) // size):
        if got[i * size:(i + 1) * size] != want[i * size:(i + 1) * size]:
            return f"{what}: element {i} differs, input {elems[i]}"
    return None


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("curve", ["bls12381", "bn254"])
def test_gt_mul_and_inv_on_crafted_elements(engine, curve, n):
    c = CURVES[curve]
    size = engine.GT_BYTES[curve]
    A, B = batch(curve, n), batch(curve, n, shift=5)
    got = engine.gt_mul(curve, enc(c, A), enc(c, B))
    want = enc(c, [f12_mul(curve, a, b) for a, b in zip(A, B)])
    assert got == want, first_difference(got, want, size, list(zip(A, B)), f"{curve} gt_mul n={n}")
    got = engine.gt_inv(curve, enc(c, A))
    want = enc(c, [f12_inv(curve, a) for a in A])
    assert got == want, first_difference(got, want, size, A, f"{curve} gt_inv n={n}")


def test_gt_inv_of_zero_is_zero(engine):
    """fp12_inv maps 0 to 0 (the inversion of 0 is 0 all the way down the tower); the header documents it"""
    for curve in ("bls12381", "bn254"):
        z = bytes(engine.GT_BYTES[curve])
        assert engine.gt_inv(curve, z * 3) == z * 3


@pytest.mark.parametrize("coop", ["default", "off"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("curve", ["bls12381", "bn254"])
def test_gt_exp_on_crafted_elements(engine, curve, n, coop):
    c = CURVES[curve]
    size = engine.GT_BYTES[curve]
    rng = random.Random(f"gt-exp/{curve}")
    ks = [0, 1, 2, c.order - 1] + [rng.randrange(c.order) for _ in range(4)]
    A = batch(curve, n)
    K = [ks[(i // 3) % len(ks)] for i in range(n)]
    if coop == "off":
        engine.set_pairing_coop(0)
    try:
        got = engine.gt_exp(curve, b"".join(k.to_bytes(32, "big") for k in K), enc(c, A))
    finally:
        engine.set_pairing_coop(COOP_DEFAULT)
    want = enc(c, [f12_pow(curve, a, k) for a, k in zip(A, K)])
    assert got == want, first_difference(got, want, size, list(zip(A, K)), f"{curve} gt_exp n={n} coop={coop}")


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("curve", ["bls12381", "bn254", "bn256"])
def test_final_exp_on_crafted_elements(engine, curve, n):
    """BLS12-381: the exponent 3 (p^12 - 1)/r of pairing_reference; bn254 / bn256: the oracles' exact (p^12 - 1)/n"""
    c = CURVES[curve]
    size = engine.GT_BYTES[curve]
    A = batch(curve, n)
    got = engine.final_exp(curve, enc(c, A))
    want = enc(c, [final(curve, a) for a in A])
    assert got == want, first_difference(got, want, size, A, f"{curve} final_exp n={n}")
