"""Case lists and Python-integer expectations for the field harness (tests/device/field_harness.cu).

Every operand is a RAW Montgomery limb vector: the integer a below p that the device holds for the field element a R^-1
(R = 2^(32 N)).  So a product is checked as a b R^-1 mod p, an inverse as a^-1 R^2, a power x^e as (a R^-1)^e R, and a tower
operation by converting each coefficient out of Montgomery form, applying the oracle's f2_/f6_/f12_ function and converting back.
The same lists drive the host-emulated twin (test_field_arith_emulation.py) and the three device builds
(test_gpu_field_arith.py)."""
from __future__ import annotations

import ctypes
import functools
import random
from dataclasses import dataclass

import numpy as np

from oracle import bls12381 as o
from oracle import bn254, bn256, bn254_pairing, bn256_pairing
from oracle import ed25519

# ---- the harness's operation codes (field_harness.cu: FpOp, TwOp) -------------------------------------------------------------
FP_OPS = ["add", "sub", "neg", "dbl", "addsub_plus", "addsub_minus", "mul", "sqr", "mul_i", "mul_sum2", "to_mont", "from_mont",
          "inv", "inv_fermat", "inv_vartime", "pow_sqrt", "pow_legendre", "pow_p58", "gt_half", "lt_mod", "store_be", "load_be"]
TW_OPS = ["f2_mul", "f2_sqr", "f2_inv", "f2_mul_lazy", "f2_mul_xi", "f6_mul", "f6_sqr", "f6_inv", "f6_mul_by_01", "f6_mul_by_1",
          "f12_mul", "f12_sqr", "f12_inv", "f12_conj", "f12_cyclotomic_sqr", "f12_frob1", "f12_frob2", "f12_frob3",
          "fp_sqrt", "fp2_sqrt"]
BINARY_FP = {"add", "sub", "addsub_plus", "addsub_minus", "mul", "mul_i", "mul_sum2"}
BINARY_TW = {"f2_mul", "f2_mul_lazy", "f6_mul", "f6_mul_by_01", "f6_mul_by_1", "f12_mul"}
ALIASES = {0: "r = op(x, y)", 1: "op(x, x, y)", 2: "op(y, x, y)", 3: "op(x, x, x)"}


@dataclass(frozen=True)
class Field:
    name: str
    n: int
    p: int
    bits: int
    exps: tuple          # the pow_* operations the configuration carries (constants.cuh)


FIELDS = [
    Field("bls381_fp", 12, o.P, 381, ("sqrt", "legendre")),
    Field("bls381_fr", 8, o.R, 255, ("legendre",)),
    Field("bn254_fp", 8, bn254.P, 254, ("sqrt", "legendre")),
    Field("bn254_fr", 8, bn254.ORDER, 254, ("legendre",)),
    Field("bn256_fp", 10, bn256.P, 256, ("sqrt", "legendre")),
    Field("ed25519_fp", 8, ed25519.P, 255, ("legendre", "p58")),
    Field("ed25519_fr", 8, ed25519.L, 253, ("legendre",)),
]
FIELD = {f.name: f for f in FIELDS}


def exponent(f: Field, which: str) -> int:
    return {"sqrt": (f.p + 1) // 4, "legendre": (f.p - 1) // 2, "p58": (f.p - 5) // 8}[which]


# ---- limb packing -----------------------------------------------------------------------------------------------------------
def pack(vals, n) -> np.ndarray:
    return np.frombuffer(b"".join(v.to_bytes(4 * n, "little") for v in vals), dtype="<u4").copy()


def unpack(words: np.ndarray, n):
    b = words.astype("<u4").tobytes()
    return [int.from_bytes(b[4 * n * i:4 * n * (i + 1)], "little") for i in range(len(words) // n)]


def call(lib, kind: str, target: str, op: int, alias: int, inp: np.ndarray, rows: int, out_words: int) -> np.ndarray:
    out = np.zeros(rows * out_words, dtype="<u4")
    fn = getattr(lib, f"fh_{kind}_{target}")
    fn.restype = ctypes.c_int
    u32p = ctypes.POINTER(ctypes.c_uint32)
    err = fn(ctypes.c_int(op), ctypes.c_int(alias), ctypes.c_int(rows), inp.ctypes.data_as(u32p), out.ctypes.data_as(u32p))
    assert err == 0, f"fh_{kind}_{target}: CUDA error {err}"
    return out


# ---- operands -----------------------------------------------------------------------------------------------------------------
def edges(f: Field):
    """0, 1, 2, p-1, p-2, (p+-1)/2, R mod p, R^2 mod p; 2^(32k) and 2^(32k)-1 below p, 2^(BITS-1), p - 2^(32k); values whose two
    halves are equal or differ by one; alternating all-ones / zero limbs"""
    p, n = f.p, f.n
    R = 1 << (32 * n)
    v = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R % p, R * R % p, 1 << (f.bits - 1)]
    for k in range(1, n):
        v += [(1 << (32 * k)), (1 << (32 * k)) - 1, p - (1 << (32 * k)), p - (1 << (32 * (k - 1)))]
    h = n // 2
    top = p >> (32 * h)
    for lo in (1, 0xffffffff, top - 1, top - 2, (1 << (32 * h)) - 1):
        for hi in (lo, lo + 1, lo - 1):
            v.append(lo + (hi << (32 * h)))
    for start in (0, 1):
        x = sum(0xffffffff << (32 * j) for j in range(start, n, 2))
        v.append(x if x < p else x & ((1 << (32 * (n - 1))) - 1))
    out, seen = [], set()
    for x in v:
        if 0 <= x < p and x not in seen:
            seen.add(x)
            out.append(x)
    return out


def randoms(f: Field, rng: random.Random, k: int):
    """uniform values and values built from limbs that sit at the carry edges (0, 1, 2^31, all-ones), reduced below p"""
    out = []
    for i in range(k):
        if i % 2:
            out.append(rng.randrange(f.p))
        else:
            x = sum(rng.choice((0, 1, 0x80000000, 0xffffffff, 0xfffffffe, rng.getrandbits(32))) << (32 * j) for j in range(f.n))
            out.append(x % f.p)
    return out


def inv_extras(f: Field):
    """powers of two and their negatives, (p + 1) / 2^k, small integers and their negatives"""
    p = f.p
    v = [1 << k for k in range(f.bits - 1)] + [p - (1 << k) for k in range(f.bits - 1)]
    v += [(p + 1) >> k for k in range(1, 64)] + list(range(1, 65)) + [p - k for k in range(1, 65)]
    return sorted(set(x for x in v if 0 < x < p))


# ---- Fp expectations --------------------------------------------------------------------------------------------------------
def fp_expect(f: Field, op: str, a: int, b: int, c: int, d: int) -> int:
    p, n = f.p, f.n
    R = 1 << (32 * n)
    ri = pow(R, -1, p)
    if op == "add":
        return (a + b) % p
    if op in ("sub", "addsub_minus"):
        return (a - b) % p
    if op == "addsub_plus":
        return (a + b) % p
    if op == "neg":
        return -a % p
    if op == "dbl":
        return 2 * a % p
    if op in ("mul", "mul_i"):
        return a * b * ri % p
    if op == "sqr":
        return a * a * ri % p
    if op == "mul_sum2":
        return (a * b + c * d) * ri % p
    if op == "to_mont":
        return a * R % p
    if op == "from_mont":
        return a * ri % p
    if op in ("inv", "inv_fermat", "inv_vartime"):
        return 0 if a == 0 else pow(a, -1, p) * R * R % p
    if op.startswith("pow_"):
        which = op[4:]
        if which not in f.exps:
            return 0
        return pow(a * ri % p, exponent(f, which), p) * R % p
    if op == "gt_half":
        return int(a > (p - 1) // 2)
    if op == "lt_mod":
        return int(a < p)
    if op == "store_be":
        return int.from_bytes(a.to_bytes(4 * n, "big"), "little")
    if op == "load_be":
        return int.from_bytes(a.to_bytes(4 * n, "little"), "big")
    raise ValueError(op)


@dataclass
class Batch:
    kind: str            # "fp" or "tw"
    target: str          # field or tower name
    op: str
    alias: int
    operands: list       # per case: (a, b, c, d) integers (fp) or (A, B) tuples of 12 integers (tw)
    inp: np.ndarray
    want: np.ndarray
    out_words: int
    mask: np.ndarray = None   # words that are compared (tw: a failed square root leaves its result undefined)

    @property
    def opcode(self):
        return (FP_OPS if self.kind == "fp" else TW_OPS).index(self.op)

    def describe(self, i):
        ops = self.operands[i]
        fmt = (lambda x: hex(x)) if self.kind == "fp" else (lambda t: "[" + ", ".join(hex(x) for x in t) + "]")
        return f"{self.target} {self.op} {ALIASES[self.alias]} case {i}: operands {', '.join(fmt(x) for x in ops)}"


def _fp_batch(f: Field, op: str, alias: int, quads) -> Batch:
    n = f.n
    if alias == 3:
        quads = [(a, a, a, a) for a, _, _, _ in quads]
    inp = pack([x for q in quads for x in q], n)
    want = pack([fp_expect(f, op, *q) for q in quads], n)
    return Batch("fp", f.name, op, alias, list(quads), inp, want, n)


UNARY_EXPENSIVE = {"inv", "inv_fermat", "inv_vartime", "pow_sqrt", "pow_legendre", "pow_p58"}


@functools.lru_cache(maxsize=None)
def fp_batches(name: str, n_random: int = 2000):
    """every operation of one field: the edge x edge grid plus n_random random cases, the aliased forms, the extreme sums of two
    products, and one launch of at least 64K inversions with converging and long-running lanes shuffled into the same warps"""
    f = FIELD[name]
    rng = random.Random(f"field-cases/{name}")
    E = edges(f)
    grid = [(a, b) for a in E for b in E]
    out = []
    for op in FP_OPS:
        if op.startswith("pow_") and op[4:] not in f.exps:
            continue
        rnd = randoms(f, rng, 4 * n_random)
        quads = []
        if op in BINARY_FP:
            quads += [(a, b, rng.choice(E), rng.choice(E)) for a, b in grid]
            quads += [(rnd[4 * i], rnd[4 * i + 1], rnd[4 * i + 2], rnd[4 * i + 3]) for i in range(n_random)]
            if op == "mul_sum2":                          # the largest sums of two products of field elements, and their mixes
                ext = [f.p - 1, f.p - 2, (f.p + 1) // 2, (f.p - 1) // 2, 0, 1]
                quads += [(a, b, c, d) for a in ext for b in ext for c in ext for d in ext]
        else:
            src = E + (inv_extras(f) if op.startswith("inv") else []) + rnd[:n_random]
            if op == "lt_mod":                           # the only operation that takes values at or above p
                src += [f.p, f.p + 1, f.p + (1 << 32), (1 << (32 * f.n)) - 1, (1 << (32 * f.n - 1))]
                src = [x for x in src if x < (1 << (32 * f.n))]
            quads = [(a, 0, 0, 0) for a in src]
        out.append(_fp_batch(f, op, 0, quads))
        aliases = (1, 2, 3) if op in BINARY_FP else (1,)
        for al in aliases:
            sub = quads if op not in UNARY_EXPENSIVE else [(a, 0, 0, 0) for a in E]
            sub = sub[:len(grid) + 256]
            out.append(_fp_batch(f, op, al, sub))
    # 64K inversions in one launch: 0, small and power-of-two operands (few rounds) next to uniform ones (all rounds)
    src = [0] * 64 + E + inv_extras(f)
    src += [rng.randrange(f.p) for _ in range(65536 - len(src))]
    rng.shuffle(src)
    out.append(_fp_batch(f, "inv", 0, [(a, 0, 0, 0) for a in src]))
    return out


# ---- towers ---------------------------------------------------------------------------------------------------------------------
class Tower:
    def __init__(self, name, n, p, ns, is_bls):
        self.name, self.n, self.p, self.ns, self.is_bls = name, n, p, ns, is_bls
        self.R = 1 << (32 * n)
        self.ri = pow(self.R, -1, p)

    # flat 12-coefficient vectors (tower order) <-> the oracle's nested tuples, out of / into Montgomery form
    def to_f12(self, flat):
        v = [x * self.ri % self.p for x in flat]
        f2 = [(v[2 * i], v[2 * i + 1]) for i in range(6)]
        return ((f2[0], f2[1], f2[2]), (f2[3], f2[4], f2[5]))

    def from_f12(self, a):
        return [x * self.R % self.p for c6 in a for c2 in c6 for x in c2]

    def mul_v(self, a):
        return self.ns.f6_mul_v(a) if self.is_bls else self.ns.f6_mul_tau(a)

    def frob_pow(self, a, k):
        return self.ns.f12_pow(a, self.p ** k)


TOWERS = {
    "bls381": Tower("bls381", 12, o.P, o, True),
    "bn254": Tower("bn254", 8, bn254.P, bn254_pairing, False),
    "bn256": Tower("bn256", 10, bn256.P, bn256_pairing, False),
}

_Z2 = (0, 0)
_Z6 = (_Z2, _Z2, _Z2)


def tw_expect(tw: Tower, op: str, A, B):
    """the expected 12 result coefficients (Montgomery) and flag for the harness's result layout; None for a failed root"""
    ns, a, b = tw.ns, tw.to_f12(A), tw.to_f12(B)
    level = {"f2": 2, "f6": 6, "f1": 12}[op[:2]] if op[:2] in ("f2", "f6", "f1") else None
    flag = 0
    if op == "f2_mul" or op == "f2_mul_lazy":
        r = ns.f2_mul(a[0][0], b[0][0])
    elif op == "f2_sqr":
        r = ns.f2_sqr(a[0][0])
    elif op == "f2_inv":
        r = _Z2 if a[0][0] == _Z2 else ns.f2_inv(a[0][0])
    elif op == "f2_mul_xi":
        r = ns.f2_mul_xi(a[0][0])
    elif op == "f6_mul":
        r = ns.f6_mul(a[0], b[0])
    elif op == "f6_sqr":
        r = ns.f6_mul(a[0], a[0])
    elif op == "f6_inv":
        r = _Z6 if a[0] == _Z6 else ns.f6_inv(a[0])
    elif op == "f6_mul_by_01":
        r = ns.f6_mul(a[0], (b[0][0], b[0][1], _Z2))
    elif op == "f6_mul_by_1":
        r = ns.f6_mul(a[0], (_Z2, b[0][0], _Z2))
    elif op == "f12_mul":
        r = ns.f12_mul(a, b)
    elif op in ("f12_sqr", "f12_cyclotomic_sqr"):
        r = ns.f12_mul(a, a)
    elif op == "f12_inv":
        r = (_Z6, _Z6) if a == (_Z6, _Z6) else ns.f12_inv(a)
    elif op == "f12_conj":
        r = ns.f12_conj(a)
    elif op.startswith("f12_frob"):
        r = ns.f12_frobenius(a, int(op[-1]))
    elif op == "fp_sqrt":
        s = o.fp_sqrt(a[0][0][0])
        return (None if s is None else [s * tw.R % tw.p]), int(s is not None), 1
    elif op == "fp2_sqrt":
        s = o.f2_sqrt(a[0][0])
        return (None if s is None else [x * tw.R % tw.p for x in s]), int(s is not None), 2
    else:
        raise ValueError(op)
    if level == 2:
        flat = [x * tw.R % tw.p for x in r]
    elif level == 6:
        flat = [x * tw.R % tw.p for c2 in r for x in c2]
    else:
        flat = tw.from_f12(r)
    return flat, flag, level


def tw_edge_elements(tw: Tower, rng: random.Random, count: int):
    """Fp12 elements (12 Montgomery coefficients) with one nonzero coefficient, every coefficient p - 1, embedded Fp / Fp2 / Fp6
    elements, edge-valued coefficients in random slots, and zero"""
    f = Field(tw.name, tw.n, tw.p, tw.p.bit_length(), ())
    E = edges(f)
    out = [[0] * 12, [tw.p - 1] * 12, [tw.R % tw.p] + [0] * 11]
    for k in range(12):
        out.append([0] * k + [rng.choice(E[1:])] + [0] * (11 - k))
    for width in (1, 2, 6):
        for _ in range(4):
            out.append([rng.choice(E) for _ in range(width)] + [0] * (12 - width))
    while len(out) < count:
        out.append([rng.choice(E) for _ in range(12)])
    return out


def tw_random_elements(tw: Tower, rng: random.Random, count: int):
    return [[rng.randrange(tw.p) for _ in range(12)] for _ in range(count)]


def cyclotomic(tw: Tower, flat):
    """f^((p^6 - 1)(p^2 + 1)): an element of the cyclotomic subgroup (Montgomery coefficients)"""
    ns, a = tw.ns, tw.to_f12(flat)
    if a == (_Z6, _Z6):
        return tw.from_f12(ns.F12_ONE)
    t = ns.f12_mul(ns.f12_conj(a), ns.f12_inv(a))
    return tw.from_f12(ns.f12_mul(ns.f12_frobenius(t, 2), t))


def _tw_batch(tw: Tower, op: str, alias: int, pairs) -> Batch:
    n = tw.n
    if alias == 3:
        pairs = [(A, A) for A, _ in pairs]
    words = 12 * n + 1
    inp = pack([x for A, B in pairs for x in list(A) + list(B)], n)
    want = np.zeros(len(pairs) * words, dtype="<u4")
    mask = np.ones(len(pairs) * words, dtype=bool)
    for i, (A, B) in enumerate(pairs):
        flat, flag, width = tw_expect(tw, op, A, B)
        base = [0] * 12 if alias == 0 else list(A if alias in (1, 3) else B)
        row = want[i * words:(i + 1) * words]
        if flat is None:                          # failed square root: only the flag is defined
            mask[i * words:i * words + 12 * n] = False
        else:
            base[:len(flat)] = flat
            row[:12 * n] = pack(base, n)
        row[12 * n] = flag
    return Batch("tw", tw.name, op, alias, list(pairs), inp, want, words, mask)


TW_COUNTS = {"f2": 2000, "f6": 500, "f12": 300}


@functools.lru_cache(maxsize=None)
def tw_batches(name: str, scale: float = 1.0):
    """every tower operation: edge-valued elements against each other, random elements, the aliased forms; the cyclotomic squaring
    on cyclotomic elements only; the BLS12-381 square roots on squares, non-squares and zero"""
    tw = TOWERS[name]
    rng = random.Random(f"tower-cases/{name}")
    edge = tw_edge_elements(tw, rng, 48)
    out = []
    for op in TW_OPS:
        if op in ("fp_sqrt", "fp2_sqrt") and not tw.is_bls:
            continue
        k = int(TW_COUNTS["f12" if op.startswith("f12") else op[:2] if op[:2] in ("f2", "f6") else "f2"] * scale)
        if op.startswith("f12_frob"):
            k = min(k, 100)
        rnd = tw_random_elements(tw, rng, 2 * k)
        if op in BINARY_TW:
            pairs = [(A, B) for A in edge[:24] for B in edge[:24]] + [(rnd[2 * i], rnd[2 * i + 1]) for i in range(k)]
        elif op == "f12_cyclotomic_sqr":
            pairs = [(cyclotomic(tw, A), [0] * 12) for A in edge + rnd[:k]]
        elif op in ("fp_sqrt", "fp2_sqrt"):
            w = 1 if op == "fp_sqrt" else 2
            src = [A[:w] + [0] * (12 - w) for A in edge + rnd[:k]]
            sq = []                               # squares: every second element squared (as Montgomery values)
            for A in src[::2]:
                v = [x * tw.ri % tw.p for x in A[:w]]
                s = [v[0] * v[0] % tw.p] if w == 1 else list(o.f2_sqr((v[0], v[1])))
                sq.append([x * tw.R % tw.p for x in s] + [0] * (12 - w))
            pairs = [(A, [0] * 12) for A in src + sq]
        else:
            pairs = [(A, [0] * 12) for A in edge + rnd[:k]]
        out.append(_tw_batch(tw, op, 0, pairs))
        for al in ((1, 2, 3) if op in BINARY_TW else (1,)):
            out.append(_tw_batch(tw, op, al, pairs[:200]))
    return out


def frobenius_by_power(name: str, count: int = 3):
    """(input, power, x^(p^power)) with the power computed by square-and-multiply on Python integers"""
    tw = TOWERS[name]
    rng = random.Random(f"frobenius/{name}")
    out = []
    for A in tw_random_elements(tw, rng, count):
        for k in (1, 2, 3):
            out.append((A, k, tw.from_f12(tw.frob_pow(tw.to_f12(A), k))))
    return out


def mismatches(batch: Batch, got: np.ndarray, limit: int = 5):
    """descriptions of the first cases whose words differ from the expectation"""
    w = batch.out_words
    diff = got != batch.want
    if batch.mask is not None:
        diff &= batch.mask
    rows = np.nonzero(diff.reshape(-1, w).any(axis=1))[0]
    msgs = []
    for i in rows[:limit]:
        msgs.append(f"{batch.describe(int(i))}: got {[hex(x) for x in got[i * w:(i + 1) * w]]}, "
                    f"want {[hex(x) for x in batch.want[i * w:(i + 1) * w]]}")
    return len(rows), msgs
