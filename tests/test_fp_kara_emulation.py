"""CPU tests: the Karatsuba products (fp.cuh: fp_mul_sum2_inl, the Y3 of the XYZZ additions; tools/probe/fp_kara.cuh: fp_mul_k_inl)
compiled for the host (tests/host_emul/emul_fp_kara.cpp) and checked against Python integers; the XYZZ additions of ec.cuh that use the
sum of two products are checked against the same formulas written with the CIOS product alone and against the oracle's group law."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import bls12381 as o
from oracle import bn254, bn256

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")

FIELDS = [("fp381", 12, o.P), ("fp254", 8, bn254.P), ("fp256", 10, bn256.P)]   # N = 12 and 8: Karatsuba; N = 10: schoolbook


@pytest.fixture(scope="module")
def emul():
    src = os.path.join(EMU, "emul_fp_kara.cpp")
    so = os.path.join(EMU, "libemul_fp_kara.so")
    newest = max([os.path.getmtime(src)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cuh")])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", src, "-o", so],
                       check=True)
    return ctypes.CDLL(so)


def limbs(x, n):
    return (ctypes.c_uint32 * n)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)])


def value(arr):
    return sum(int(v) << (32 * i) for i, v in enumerate(arr))


def wide_operands(n, rng):
    """N-limb operands (any value below 2^(32N), not only field elements) covering the signs of a0 - a1 and b0 - b1"""
    h, top = n // 2, (1 << (32 * n)) - 1
    lo, hi = rng.getrandbits(32 * (n // 2)), rng.getrandbits(32 * (n - n // 2))
    equal_halves = lo | (lo << (32 * h)) if n % 2 == 0 else rng.getrandbits(32 * n)
    vals = [0, 1, top, top - 1, equal_halves, lo, hi << (32 * h), lo | (hi << (32 * h)), (1 << (32 * h)) - 1, 1 << (32 * h)]
    vals += [rng.getrandbits(32 * n) for _ in range(8)]
    return vals


@pytest.mark.parametrize("name,n,p", FIELDS)
def test_karatsuba_wide_product_is_exact_for_any_operands(emul, name, n, p):
    rng = random.Random(n)
    mul = getattr(emul, f"emul_{name}_wide_mul_kara")
    sum2 = getattr(emul, f"emul_{name}_wide_mul_kara_sum2") if n % 4 == 0 else None
    vals = wide_operands(n, rng)
    for a in vals:
        for b in vals:
            t = (ctypes.c_uint32 * (2 * n))()
            mul(limbs(a, n), limbs(b, n), t)
            assert value(t) == a * b, (hex(a), hex(b))
            if sum2 is None:
                continue
            c = rng.choice(vals)                                   # a b + c d < 2^(64N)
            d = min(rng.choice(vals), ((1 << (64 * n)) - 1 - a * b) // c if c else (1 << (32 * n)) - 1)
            sum2(limbs(a, n), limbs(b, n), limbs(c, n), limbs(d, n), t)
            assert value(t) == a * b + c * d, (hex(a), hex(b), hex(c), hex(d))


@pytest.mark.parametrize("name,n,p", FIELDS)
def test_mul_k_and_sum_of_two_products(emul, name, n, p):
    rng = random.Random(100 + n)
    rinv = pow(1 << (32 * n), -1, p)
    vals = [0, 1, p - 1, p - 2, (p - 1) // 2] + [rng.randrange(p) for _ in range(10)]
    mul_k, sum2 = (getattr(emul, f"emul_{name}_{f}") for f in ("mul_k", "mul_sum2"))
    r = (ctypes.c_uint32 * n)()
    for a in vals:
        for b in vals:
            mul_k(limbs(a, n), limbs(b, n), r)
            assert value(r) == a * b * rinv % p, (hex(a), hex(b))
            c, d = rng.choice(vals), rng.choice(vals)
            sum2(limbs(a, n), limbs(b, n), limbs(c, n), limbs(d, n), r)
            assert value(r) == (a * b + c * d) * rinv % p, (hex(a), hex(b), hex(c), hex(d))
    for c in (p - 1, p - 2):                                      # the largest sums of two products of field elements
        sum2(limbs(p - 1, n), limbs(p - 1, n), limbs(c, n), limbs(p - 1, n), r)
        assert value(r) == ((p - 1) ** 2 + c * (p - 1)) * rinv % p


# ---- XYZZ additions (Y3 through the sum of two products), BLS12-381 G1 ------------------------------------------------------
P, N = o.P, 12
RM = 1 << (32 * N)
RMINV = pow(RM, -1, P)


def mont(x):
    return x * RM % P


def xyzz(pt, lam):
    """the affine point pt as XYZZ with ZZ = lam^2, ZZZ = lam^3 (None: infinity, ZZ = ZZZ = 0), Montgomery limbs"""
    coords = (mont(1), mont(1), 0, 0) if pt is None else (mont(pt[0] * lam * lam), mont(pt[1] * lam ** 3), mont(lam * lam), mont(lam ** 3))
    return (ctypes.c_uint32 * (4 * N))(*[w for c in coords for w in limbs(c, N)])


def affine_of(arr):
    X, Y, ZZ, ZZZ = (value(arr[i * N:(i + 1) * N]) * RMINV % P for i in range(4))
    return None if ZZ == 0 else (X * pow(ZZ, -1, P) % P, Y * pow(ZZZ, -1, P) % P)


def aff_limbs(pt):
    x, y = (0, 0) if pt is None else (mont(pt[0]), mont(pt[1]))
    return (ctypes.c_uint32 * (2 * N))(*(list(limbs(x, N)) + list(limbs(y, N))))


def cases():
    """P + Q, P + P, P + (-P), operands at infinity, with random Z scalings"""
    rng = random.Random(7)
    A, B = o.g1_mul(rng.randrange(1, o.R)), o.g1_mul(rng.randrange(1, o.R))
    lam = [rng.randrange(1, P) for _ in range(4)]
    return [(A, B, lam[0], lam[1]), (A, A, lam[0], lam[2]), (A, o.g1_neg(A), lam[1], lam[3]), (None, B, 1, lam[1]),
            (A, None, lam[2], 1), (None, None, 1, 1), (B, A, 1, 1)]


def test_xyzz_madd_matches_cios_formula_and_oracle(emul):
    for p1, q, lp, _ in cases():
        for negate in (0, 1):
            want = o.g1_add(p1, o.g1_neg(q) if negate and q is not None else q)
            got = []
            for old in (0, 1):
                r = (ctypes.c_uint32 * (4 * N))()
                emul.emul_xyzz381_madd(xyzz(p1, lp), aff_limbs(q), negate, old, r)
                got.append(affine_of(r))
            assert got[0] == got[1] == want, (p1, q, negate)


def test_xyzz_add_matches_cios_formula_and_oracle(emul):
    for p1, q, lp, lq in cases():
        got = []
        for old in (0, 1):
            r = (ctypes.c_uint32 * (4 * N))()
            emul.emul_xyzz381_add(xyzz(p1, lp), xyzz(q, lq), old, r)
            got.append(affine_of(r))
        assert got[0] == got[1] == o.g1_add(p1, q), (p1, q)
