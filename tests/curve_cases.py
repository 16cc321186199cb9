"""Case lists and expectations for the curve harness (tests/device/curve_harness.cu).

Coordinates travel as RAW Montgomery limbs (c R mod p for every Fp coefficient, c0 before c1 in Fp2), so a test chooses the
projective scale of every operand.  Projective results are compared as group elements after the Python side divides out Z
(Jacobian), ZZ / ZZZ (XYZZ) or Z (extended Edwards); a result that must be infinity must carry the library's own encoding (Z = 0,
ZZ = ZZZ = 0, affine (0, 0)), and the representation invariants ZZ^3 = ZZZ^2 and X Y = Z T are checked where they apply.
Expectations come from oracle/: the group laws of bls12381, bn254 / bn254_pairing and bn256, the maps of h2c_bls12381{,_g2}, and
ed25519.  The same lists drive the host-emulated twin (test_curve_arith_emulation.py) and the three device builds
(test_gpu_curve_arith.py)."""
from __future__ import annotations

import ctypes
import functools
import random
from dataclasses import dataclass, field

import numpy as np

from oracle import bls12381 as o
from oracle import bn254, bn256, bn254_pairing, bn256_pairing
from oracle import ed25519 as ed
from oracle import h2c_bls12381 as h2c1
from oracle import h2c_bls12381_g2 as h2c2

# ---- the harness's operation codes (curve_harness.cu: WOp, EdOp) ----------------------------------------------------------------
W_OPS = ["jac_dbl", "jac_add", "jac_madd", "jac_neg", "jac_to_affine", "jac_to_affine_bg",
         "xyzz_dbl", "xyzz_add", "xyzz_add_reduce", "xyzz_madd", "xyzz_to_affine", "xyzz_to_affine_vt", "xyzz_mul_small",
         "aff_on_curve", "jac_eq_affine", "scalar_mul", "scalar_mul_w4",
         "jac_mul_xabs", "jac_mul_xabs_jac", "in_subgroup", "decompress", "map_sswu", "iso_map", "sgn0",
         "glv_split", "scalar_mul_glv", "fp_from_64_bytes",
         "jac_psi", "clear_cofactor"]
ED_OPS = ["ed_add", "ed_dbl", "ed_dbl_xyz", "ed_add_cached", "ed_madd", "ed_decode", "ed_decode_aff", "ed_encode", "ed_encode_z1",
          "ed_bytes_canonical", "ed_has_small_order", "ed_eq", "ed_scalar_mul", "ed_mul_var"]
XMD_OPS = ["expand_message_xmd_128", "expand_message_xmd_256"]
DEVICE_ONLY = {"jac_to_affine_bg", "xyzz_to_affine_vt"}       # bodies in kernels.cuh, which only nvcc compiles
ALIASES = {0: "r = op(p, q)", 1: "op(p, p, q)", 2: "op(q, p, q)", 3: "op(p, p, p)"}


# ---- fields -------------------------------------------------------------------------------------------------------------------
class Fld:
    """Fp (deg 1, ints) or Fp2 = Fp[u]/(u^2 + 1) (deg 2, (c0, c1) tuples), with the device's limb count n"""

    def __init__(self, p, n, deg):
        self.p, self.n, self.deg = p, n, deg
        self.R = 1 << (32 * n)
        self.ri = pow(self.R, -1, p)
        self.words = n * deg

    def coeffs(self, a):
        return [a] if self.deg == 1 else list(a)

    def elem(self, cs):
        return cs[0] if self.deg == 1 else (cs[0], cs[1])

    @property
    def zero(self):
        return self.elem([0] * self.deg)

    @property
    def one(self):
        return self.elem([1] + [0] * (self.deg - 1))

    def add(self, a, b):
        return self.elem([(x + y) % self.p for x, y in zip(self.coeffs(a), self.coeffs(b))])

    def neg(self, a):
        return self.elem([-x % self.p for x in self.coeffs(a)])

    def mul(self, a, b):
        p = self.p
        if self.deg == 1:
            return a * b % p
        return ((a[0] * b[0] - a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)

    def inv(self, a):
        p = self.p
        if self.deg == 1:
            return pow(a, -1, p)
        t = pow(a[0] * a[0] + a[1] * a[1], -1, p)
        return (a[0] * t % p, -a[1] * t % p)

    def pw(self, a, e):
        r = self.one
        for bit in bin(e)[2:]:
            r = self.mul(r, r)
            if bit == "1":
                r = self.mul(r, a)
        return r

    def sqrt(self, a):
        """a square root (p = 3 mod 4 for every field here), None for a non-square"""
        p = self.p
        if self.deg == 1:
            s = pow(a, (p + 1) // 4, p)
            return s if s * s % p == a % p else None
        if a == (0, 0):
            return a
        a1 = self.pw(a, (p - 3) // 4)
        alpha = self.mul(a1, self.mul(a1, a))
        x0 = self.mul(a1, a)
        if alpha == (p - 1, 0):
            s = self.mul((0, 1), x0)
        else:
            s = self.mul(self.pw(self.add(alpha, self.one), (p - 1) // 2), x0)
        return s if self.mul(s, s) == a else None

    def rand(self, rng):
        return self.elem([rng.randrange(self.p) for _ in range(self.deg)])

    def enc(self, a) -> bytes:
        return b"".join((c * self.R % self.p).to_bytes(4 * self.n, "little") for c in self.coeffs(a))

    def dec(self, words: np.ndarray):
        b = words.astype("<u4").tobytes()
        k = 4 * self.n
        return self.elem([int.from_bytes(b[k * i:k * (i + 1)], "little") * self.ri % self.p for i in range(self.deg)])


# ---- Weierstrass groups -------------------------------------------------------------------------------------------------------
@dataclass
class Group:
    name: str
    F: Fld
    b: object
    r: int                  # prime subgroup order
    gen: tuple
    add_fn: object          # the oracle's affine addition (None = infinity)
    bls: int = 0            # 1: BLS12-381 G1, 2: BLS12-381 G2

    def add(self, a, b):
        return self.add_fn(a, b)

    def neg(self, a):
        return None if a is None else (a[0], self.F.neg(a[1]))

    def mul(self, k, pt):
        """k pt for any integer k and any point of the curve (no reduction of k)"""
        if k < 0:
            return self.mul(-k, self.neg(pt))
        acc = None
        for bit in bin(k)[2:] if k else "":
            acc = self.add(acc, acc)
            if bit == "1":
                acc = self.add(acc, pt)
        return acc

    def on_curve(self, pt):
        F = self.F
        x, y = pt
        return F.mul(y, y) == F.add(F.mul(F.mul(x, x), x), self.b)

    def lift(self, x):
        y = self.F.sqrt(self.F.add(self.F.mul(self.F.mul(x, x), x), self.b))
        return None if y is None else (x, y)

    @property
    def E(self):
        return self.F.words


def _bn_g2_add(ns):
    return ns.g2_add


FP381, FP381_2 = Fld(o.P, 12, 1), Fld(o.P, 12, 2)
FP254, FP254_2 = Fld(bn254.P, 8, 1), Fld(bn254.P, 8, 2)
FP256, FP256_2 = Fld(bn256.P, 10, 1), Fld(bn256.P, 10, 2)

GROUPS = {
    "bls381_g1": Group("bls381_g1", FP381, o.B1, o.R, o.G1, o.g1_add, 1),
    "bls381_g2": Group("bls381_g2", FP381_2, o.B2, o.R, o.G2, o.g2_add, 2),
    "bn254_g1": Group("bn254_g1", FP254, bn254.B, bn254.ORDER, bn254.G1, bn254.g1_add),
    "bn254_g2": Group("bn254_g2", FP254_2, bn254_pairing.TWIST_B, bn254.ORDER, bn254_pairing.G2, bn254_pairing.g2_add),
    "bn256_g1": Group("bn256_g1", FP256, bn256.B, bn256.ORDER, bn256.G1, bn256.g1_add),
    "bn256_g2": Group("bn256_g2", FP256_2, bn256.TWIST_B, bn256.ORDER, bn256.G2, bn256.g2_add),
}

# the scalar edges: small values, r - 1, r - 2, the GLV boundaries of glv_split_bls381, and the signed-radix-16 carry patterns
X2 = o.X_ABS ** 2


def scalar_edges(r: int, full_width: bool):
    v = list(range(18)) + [r - 1, r - 2]
    v += [X2, X2 - 1, X2 + 1, X2 // 2, X2 // 2 + 1, (r - 1) // 2, (r + 1) // 2, r - X2, 3 * X2 + X2 // 2, (1 << 128) - 1,
          1 << 128, (1 << 128) + 1]
    if full_width:
        v += [(1 << 256) - 1, int("8" * 64, 16), int("7" * 64, 16), 1 << 255, int("8" * 63, 16), int("f" * 63, 16)]
    return v


GLV_EDGES = [X2, X2 - 1, X2 + 1, X2 // 2, X2 // 2 + 1, (o.R - 1) // 2, (o.R + 1) // 2, o.R - X2, 3 * X2 + X2 // 2,
             (1 << 128) - 1, (1 << 128) + 1]


def glv_split(k: int):
    """glv_split_bls381 restated: k (or r - k) = q x^2 +- rem, |rem| <= x^2 / 2; returns (k1, k2, neg1, neg2)"""
    neg = o.R - k < k
    kk = o.R - k if neg else k
    q, rem = divmod(kk, X2)
    negr = 2 * rem > X2
    if negr:
        rem, q = X2 - rem, q + 1
    return rem, q, int(neg != negr), int(neg)


# ---- case rows and checks -----------------------------------------------------------------------------------------------------
@dataclass
class Case:
    operands: tuple           # what the failure message prints
    row: bytes                # the input words
    want: object              # the expectation, interpreted by the batch's kind
    kind: str                 # "jac", "xyzz", "aff", "flag", "words", "ed", "ed_xyz", "ed_bytes", "ed_aff"


@dataclass
class Batch:
    family: str               # "w_<group>", "ed", "xmd"
    op: str
    alias: int
    cases: list = field(default_factory=list)

    @property
    def opcode(self):
        return (W_OPS if self.family.startswith("w_") else ED_OPS if self.family == "ed" else XMD_OPS).index(self.op)

    def inp(self):
        return np.frombuffer(b"".join(c.row for c in self.cases), dtype="<u4").copy()


def w_sizes(g: Group):
    return 8 * g.E + 9, 4 * g.E + 1


def jac_enc(g: Group, pt, lam, inf_xy=None):
    F = g.F
    if pt is None:
        x, y = inf_xy if inf_xy else (F.one, F.one)
        return [x, y, F.zero, F.zero]
    l2 = F.mul(lam, lam)
    return [F.mul(pt[0], l2), F.mul(pt[1], F.mul(l2, lam)), lam, F.zero]


def xyzz_enc(g: Group, pt, lam, inf_xy=None):
    F = g.F
    if pt is None:
        x, y = inf_xy if inf_xy else (F.one, F.one)
        return [x, y, F.zero, F.zero]
    l2 = F.mul(lam, lam)
    l3 = F.mul(l2, lam)
    return [F.mul(pt[0], l2), F.mul(pt[1], l3), l2, l3]


def aff_enc(g: Group, pt):
    F = g.F
    return [F.zero, F.zero, F.zero, F.zero] if pt is None else [pt[0], pt[1], F.zero, F.zero]


def w_row(g: Group, A, B=None, k=0, w=0, raw_a: bytes = None):
    F = g.F
    B = B or [F.zero] * 4
    a = raw_a.ljust(16 * g.E, b"\0") if raw_a is not None else b"".join(F.enc(c) for c in A)
    return a + b"".join(F.enc(c) for c in B) + (k % (1 << 256)).to_bytes(32, "little") + w.to_bytes(4, "little")


def w_check(g: Group, batch: Batch, got: np.ndarray, layout: str, limit: int = 5):
    """the failure messages of the cases whose output differs from the expectation"""
    F, E = g.F, g.E
    _, ow = w_sizes(g)
    msgs = []
    count = 0
    for i, c in enumerate(batch.cases):
        row = got[i * ow:(i + 1) * ow]
        co = [F.dec(row[j * E:(j + 1) * E]) for j in range(4)]
        flag = int(row[4 * E])
        err = None
        if c.kind == "flag":
            if flag != int(c.want):
                err = f"flag {flag}, want {int(c.want)}"
        elif c.kind == "words":
            if [int(x) for x in row[:len(c.want)]] != list(c.want):
                err = f"words {[hex(int(x)) for x in row[:len(c.want)]]}, want {[hex(x) for x in c.want]}"
        else:
            want, want_flag = c.want if isinstance(c.want, tuple) and len(c.want) == 2 and isinstance(c.want[1], bool) else (c.want, None)
            if want_flag is not None and flag != int(want_flag):
                err = f"flag {flag}, want {int(want_flag)}"
            elif want_flag is False:
                pass
            elif c.kind == "field":
                if co[0] != want:
                    err = f"{co[0]}, want {want}"
            else:
                pt, bad = decode_w(F, c.kind, co)
                if bad:
                    err = bad
                elif pt != want:
                    err = f"point {fmt(pt)}, want {fmt(want)}"
        if err:
            count += 1
            if len(msgs) < limit:
                msgs.append(f"[{layout}] {g.name} {batch.op} {ALIASES[batch.alias]} case {i}: operands {c.operands}: {err}")
    return count, msgs


def decode_w(F: Fld, kind: str, co):
    """the affine point of a result (None = infinity) and a message when the representation is broken"""
    if kind == "jac":
        X, Y, Z = co[:3]
        if Z == F.zero:
            return None, None
        zi = F.inv(Z)
        z2 = F.mul(zi, zi)
        return (F.mul(X, z2), F.mul(Y, F.mul(z2, zi))), None
    if kind == "xyzz":
        X, Y, ZZ, ZZZ = co
        if ZZ == F.zero or ZZZ == F.zero:
            if ZZ != ZZZ:
                return None, f"half an infinity: ZZ {ZZ}, ZZZ {ZZZ}"
            return None, None
        if F.mul(F.mul(ZZ, ZZ), ZZ) != F.mul(ZZZ, ZZZ):
            return None, "ZZ^3 != ZZZ^2"
        return (F.mul(X, F.inv(ZZ)), F.mul(Y, F.inv(ZZZ))), None
    if kind == "aff":
        if co[0] == F.zero and co[1] == F.zero:
            return None, None
        return (co[0], co[1]), None
    raise ValueError(kind)


def fmt(pt):
    if pt is None:
        return "inf"
    return "(" + ", ".join(hex(c) if isinstance(c, int) else "(" + ", ".join(hex(x) for x in c) + ")" for c in pt) + ")"


def call(lib, family: str, op: int, alias: int, inp: np.ndarray, rows: int, out_words: int) -> np.ndarray:
    out = np.zeros(rows * out_words, dtype="<u4")
    fn = getattr(lib, f"ch_{family}")
    fn.restype = ctypes.c_int
    u32p = ctypes.POINTER(ctypes.c_uint32)
    err = fn(ctypes.c_int(op), ctypes.c_int(alias), ctypes.c_int(rows), inp.ctypes.data_as(u32p), out.ctypes.data_as(u32p))
    assert err == 0, f"ch_{family}: CUDA error {err}"
    return out


# ---- operand pools ------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def pools(name: str):
    """subgroup points, on-curve points outside the subgroup (where the curve has any), points with x = 0, and scales"""
    g = GROUPS[name]
    rng = random.Random(f"curve-cases/{name}")
    sub, q = [], g.gen
    for i in range(6):
        sub.append(q)
        q = g.add(g.add(q, q), g.gen if i % 2 else sub[0])
    lifted = []
    while len(lifted) < 4:
        pt = g.lift(g.F.rand(rng))
        if pt is not None:
            lifted.append(pt)
    prime_order = not g.bls and g.F.deg == 1     # bn254 / bn256 G1: every point of the curve is a subgroup point
    other = [] if prime_order else lifted
    if prime_order:
        sub += lifted
    x0 = []
    y = g.F.sqrt(g.b)
    if y is not None:
        x0 = [(g.F.zero, y), (g.F.zero, g.F.neg(y))]
    lams = [g.F.one, g.F.neg(g.F.one)] + [g.F.rand(rng) for _ in range(3)]
    return sub, other, x0, lams, rng


def weird_inf(g: Group, rng):
    return (g.F.rand(rng), g.F.rand(rng))


def w_batches_for(name: str):
    g = GROUPS[name]
    sub, other, x0, lams, _ = pools(name)
    rng = random.Random(f"curve-batches/{name}")
    pts = sub + other + x0
    fam = f"w_{name}"
    out = []

    def lam():
        return rng.choice(lams[2:]) if rng.random() < 0.8 else rng.choice(lams)

    # binary operations: random pairs, P + P and P + (-P) at different scales, infinity in either and both slots
    pairs = []
    for i, P in enumerate(pts):
        Q = pts[(i + 1) % len(pts)]
        pairs += [(P, Q), (P, P), (P, g.neg(P)), (P, None), (None, P), (g.neg(P), P)]
    pairs += [(None, None)]
    for enc, opname, kind in ((jac_enc, "jac_add", "jac"), (xyzz_enc, "xyzz_add", "xyzz"), (xyzz_enc, "xyzz_add_reduce", "xyzz")):
        for alias in (0, 1, 2, 3):
            b = Batch(fam, opname, alias)
            for P, Q in pairs:
                for same_scale in (False, True):
                    l1 = lam()
                    l2 = l1 if same_scale else lam()
                    wi = weird_inf(g, rng) if rng.random() < 0.5 else None
                    A = enc(g, P, l1, wi)
                    B = enc(g, Q, l2, weird_inf(g, rng) if wi else None)
                    want = g.add(P, P) if alias == 3 else g.add(P, Q)
                    b.cases.append(Case((fmt(P), fmt(Q), "same scale" if same_scale else "rescaled"), w_row(g, A, B), want, kind))
            out.append(b)
    # mixed additions: an affine q (infinity = (0, 0)) into a projective p, in place or not; xyzz_madd also subtracts
    for opname, enc, kind, negs in (("jac_madd", jac_enc, "jac", (0,)), ("xyzz_madd", xyzz_enc, "xyzz", (0, 1))):
        for alias in (0, 1):
            b = Batch(fam, opname, alias)
            for P, Q in pairs:
                for w in negs:
                    Qs = g.neg(Q) if w else Q
                    for Pp, Qq in ((P, Q), (P, g.neg(P) if w else P), (P, P if w else g.neg(P))):
                        l1 = lam()
                        wi = weird_inf(g, rng) if rng.random() < 0.5 else None
                        want = g.add(Pp, g.neg(Qq) if w else Qq)
                        b.cases.append(Case((fmt(Pp), fmt(Qq), f"negate {w}"), w_row(g, enc(g, Pp, l1, wi), aff_enc(g, Qq), 0, w), want, kind))
            out.append(b)
    # unary operations on every pool point at several scales and on infinities
    singles = [(P, lam()) for P in pts for _ in range(3)] + [(None, lams[0])] * 2
    unary = [("jac_dbl", jac_enc, "jac", lambda P: g.add(P, P)), ("jac_neg", jac_enc, "jac", g.neg),
             ("xyzz_dbl", xyzz_enc, "xyzz", lambda P: g.add(P, P)),
             ("jac_to_affine", jac_enc, "aff", lambda P: P), ("jac_to_affine_bg", jac_enc, "aff", lambda P: P),
             ("xyzz_to_affine", xyzz_enc, "aff", lambda P: P), ("xyzz_to_affine_vt", xyzz_enc, "aff", lambda P: P)]
    for opname, enc, kind, fn in unary:
        for alias in ((0, 1) if opname in ("jac_dbl", "jac_neg", "xyzz_dbl") else (0,)):
            b = Batch(fam, opname, alias)
            for P, l in singles:
                wi = weird_inf(g, rng) if P is None and rng.random() < 0.5 else None
                b.cases.append(Case((fmt(P), "scaled"), w_row(g, enc(g, P, l, wi)), fn(P), kind))
            out.append(b)
    # small multiples of an XYZZ point (bucket-reduction offsets)
    for alias in (0, 1):
        b = Batch(fam, "xyzz_mul_small", alias)
        for P in pts[:3] + x0 + [None]:
            for k in [0, 1, 2, 3, 4, 7, 8, 15, 16, 17, 255, 1 << 31, (1 << 32) - 1, rng.getrandbits(32)]:
                b.cases.append(Case((fmt(P), k), w_row(g, xyzz_enc(g, P, lam()), None, k), g.mul(k, P), "xyzz"))
        out.append(b)
    # the curve equation and the affine comparison
    b = Batch(fam, "aff_on_curve", 0)
    for P in pts + [None]:
        b.cases.append(Case((fmt(P),), w_row(g, aff_enc(g, P)), True, "flag"))
        if P is not None:
            bad = (P[0], g.F.add(P[1], g.F.one))
            b.cases.append(Case((fmt(bad),), w_row(g, aff_enc(g, bad)), False, "flag"))
    b.cases.append(Case(("(0, 1)",), w_row(g, aff_enc(g, (g.F.zero, g.F.one))), g.on_curve((g.F.zero, g.F.one)), "flag"))
    out.append(b)
    b = Batch(fam, "jac_eq_affine", 0)
    for i, P in enumerate(pts + [None]):
        Q = pts[(i + 1) % len(pts)]
        for A, B, want in ((P, P, True), (P, g.neg(P), P is None or P[1] == g.F.zero), (P, Q, P == Q), (None, P, P is None)):
            b.cases.append(Case((fmt(A), fmt(B)), w_row(g, jac_enc(g, A, lam()), aff_enc(g, B)), want, "flag"))
    out.append(b)
    # scalar multiplication: every scalar edge on a subgroup point, points outside the subgroup, x = 0 points and infinity
    ks = scalar_edges(g.r, True) + [rng.randrange(g.r) for _ in range(8)] + [rng.getrandbits(256) for _ in range(4)]
    spts = [sub[1]] + other[:1] + x0[:1]
    for opname in ("scalar_mul", "scalar_mul_w4"):
        b = Batch(fam, opname, 0)
        for P in spts:
            for k in ks:
                b.cases.append(Case((fmt(P), hex(k)), w_row(g, aff_enc(g, P), None, k), _mul(name, k, P), "jac"))
        for k in ks[:20]:
            b.cases.append(Case(("inf", hex(k)), w_row(g, aff_enc(g, None), None, k), None, "jac"))
        out.append(b)
    if g.bls:
        out += bls_batches(g, sub, other, x0, lams, rng)
    return out


@functools.lru_cache(maxsize=None)
def _mul_cached(name, k, P):
    return GROUPS[name].mul(k, P)


def _mul(name, k, P):
    return _mul_cached(name, k, P)


def bls_batches(g: Group, sub, other, x0, lams, rng):
    fam = f"w_{g.name}"
    F = g.F
    out = []

    def lam():
        return rng.choice(lams[2:])

    pts = sub[:3] + other[:2] + x0
    b = Batch(fam, "jac_mul_xabs", 0)
    for P in pts + [None]:
        b.cases.append(Case((fmt(P),), w_row(g, aff_enc(g, P)), _mul(g.name, o.X_ABS, P), "jac"))
    out.append(b)
    for alias in (0, 1):
        b = Batch(fam, "jac_mul_xabs_jac", alias)
        for P in pts + [None]:
            b.cases.append(Case((fmt(P), "scaled"), w_row(g, jac_enc(g, P, lam())), _mul(g.name, o.X_ABS, P), "jac"))
        out.append(b)
    b = Batch(fam, "in_subgroup", 0)
    for P in sub[:4] + [None]:
        b.cases.append(Case((fmt(P),), w_row(g, aff_enc(g, P)), True, "flag"))
    for P in other + x0:
        b.cases.append(Case((fmt(P),), w_row(g, aff_enc(g, P)), False, "flag"))
    out.append(b)
    # decompression: both signs, infinity, the subgroup check on and off, and the rejections
    comp = o.g1_compress if g.bls == 1 else o.g2_compress
    decomp = o.g1_decompress if g.bls == 1 else o.g2_decompress
    nb = 48 if g.bls == 1 else 96
    encs = []
    for P in sub[:3] + other[:2] + x0 + [None]:
        encs.append(comp(P))
        if P is not None:
            encs.append(comp(g.neg(P)))
    inf = comp(None)
    encs += [bytes([0xE0]) + inf[1:], bytes([0xC0]) + bytes(nb - 2) + b"\x01", bytes([0x40]) + inf[1:], encs[0][:1] + bytes([0x7f]) + encs[0][2:]]
    pbytes = o.P.to_bytes(48, "big")
    encs += [bytes([0x80 | pbytes[0]]) + pbytes[1:] + bytes(nb - 48), bytes([encs[0][0] & 0x7f]) + encs[0][1:]]
    if g.bls == 2:
        encs.append(bytes([0x80]) + bytes(47) + pbytes)                  # x.c0 = p
    while sum(1 for e in encs if _dec(decomp, e, False) == "reject") < 10:  # x with no point
        x = rng.randrange(o.P)
        e = bytearray(x.to_bytes(48, "big") + (rng.randrange(o.P).to_bytes(48, "big") if g.bls == 2 else b""))
        e[0] |= 0x80
        encs.append(bytes(e))
    for check in (0, 1):
        b = Batch(fam, "decompress", 0)
        for e in encs:
            d = _dec(decomp, e, bool(check))
            want = (None, False) if d == "reject" else (d, True)
            b.cases.append(Case((e.hex(), f"check {check}"), w_row(g, None, None, 0, check, raw_a=e), want, "aff"))
        out.append(b)
    # SSWU map, isogeny and sgn0
    map_fn = h2c1.map_to_curve_sswu if g.bls == 1 else h2c2.map_to_curve_sswu
    iso_fn = h2c1.iso_map if g.bls == 1 else h2c2.iso_map
    sgn_fn = (lambda a: a & 1) if g.bls == 1 else h2c2.sgn0
    p = o.P
    if g.bls == 1:
        us = [0, 1, p - 1, 2, p - 2, (p - 1) // 2, (p + 1) // 2]
    else:
        us = [(0, 0), (1, 0), (p - 1, 0), (0, 1), (0, p - 1), (0, 2), (2, 0), (1, 1), (p - 1, p - 1)]
        us += [(0, rng.randrange(p)) for _ in range(4)] + [(rng.randrange(p), 0) for _ in range(4)]
    sq, nsq = 0, 0
    while sq < 6 or nsq < 6:                    # u for which gx1 is a square, and for which it is not
        u = F.rand(rng)
        x1 = map_x1(g, u)
        is_sq = F.sqrt(F.add(F.add(F.mul(F.mul(x1, x1), x1), F.mul(_iso_a(g), x1)), _iso_b(g))) is not None
        if (is_sq and sq < 6) or (not is_sq and nsq < 6):
            us.append(u)
            sq, nsq = sq + is_sq, nsq + (not is_sq)
    b = Batch(fam, "map_sswu", 0)
    mapped = []
    for u in us:
        m = map_fn(u)
        mapped.append(m)
        b.cases.append(Case((str(u),), w_row(g, [u, F.zero, F.zero, F.zero]), m, "aff"))
    out.append(b)
    b = Batch(fam, "iso_map", 0)
    isos = mapped[:]
    if g.bls == 2:
        isos += [(h2c2.X0, F.one), (h2c2.X0, F.rand(rng))]               # the kernel of the 3-isogeny
    for m in isos:
        b.cases.append(Case((fmt(m),), w_row(g, [m[0], m[1], F.zero, F.zero]), iso_fn(m), "jac"))
    out.append(b)
    b = Batch(fam, "sgn0", 0)
    for u in us + [F.zero, F.one, F.neg(F.one)]:
        b.cases.append(Case((str(u),), w_row(g, [u, F.zero, F.zero, F.zero]), sgn_fn(u), "flag"))
    out.append(b)
    if g.bls == 1:
        out += bls_g1_batches(g, sub, other, x0, rng)
    else:
        out += bls_g2_batches(g, sub, other, lams, rng)
    return out


def _iso_a(g):
    return h2c1.ISO_A if g.bls == 1 else h2c2.A2


def _iso_b(g):
    return h2c1.ISO_B if g.bls == 1 else h2c2.B2


def map_x1(g: Group, u):
    """the first SSWU candidate x1 (RFC 9380 6.6.2), to sort u by whether g(x1) is a square"""
    F = g.F
    z = F.elem([h2c1.Z]) if g.bls == 1 else h2c2.Z2
    a, b = _iso_a(g), _iso_b(g)
    zu2 = F.mul(z, F.mul(u, u))
    tv1 = F.add(F.mul(zu2, zu2), zu2)
    if tv1 == F.zero:
        return F.mul(b, F.inv(F.mul(z, a)))
    return F.mul(F.mul(F.neg(b), F.inv(a)), F.add(F.one, F.inv(tv1)))


def _dec(fn, e, check):
    try:
        return fn(e, check)
    except ValueError:
        return "reject"


def bls_g1_batches(g: Group, sub, other, x0, rng):
    fam = "w_bls381_g1"
    out = []
    ks = GLV_EDGES + list(range(18)) + [o.R - 1, o.R - 2, o.R - X2 + 1, o.R - X2 // 2, o.R - X2 // 2 - 1]
    ks += [rng.randrange(o.R) for _ in range(64)]
    ks += [q * X2 + X2 // 2 + d for q in (1, (1 << 127) - 1, rng.getrandbits(126)) for d in (-1, 0, 1)]
    b = Batch(fam, "glv_split", 0)
    for k in ks:
        k1, k2, n1, n2 = glv_split(k)
        words = [(v >> (32 * j)) & 0xffffffff for v in (k1, k2) for j in range(8)] + [n1, n2]
        b.cases.append(Case((hex(k),), w_row(g, [0] * 4, None, k), words, "words"))
    out.append(b)
    b = Batch(fam, "scalar_mul_glv", 0)
    for P in sub[:2] + [None]:
        for k in ks[:40] + GLV_EDGES:
            b.cases.append(Case((fmt(P), hex(k)), w_row(g, aff_enc(g, P), None, k), _mul(g.name, k, P), "jac"))
    out.append(b)
    b = Batch(fam, "fp_from_64_bytes", 0)
    srcs = [bytes(64), b"\xff" * 64, o.P.to_bytes(64, "big"), (o.P - 1).to_bytes(64, "big"), (o.P << 128).to_bytes(64, "big"), ((1 << 512) - o.P).to_bytes(64, "big")]
    srcs += [rng.randbytes(64) for _ in range(32)]
    for s in srcs:
        # the harness reads the 64 bytes in order from the words of the A operand
        b.cases.append(Case((s.hex(),), w_row(g, None, None, 0, 0, raw_a=s), int.from_bytes(s, "big") % o.P, "field"))
    out.append(b)
    return out


def bls_g2_batches(g: Group, sub, other, lams, rng):
    fam = "w_bls381_g2"
    out = []
    pts = sub[:3] + other
    for alias in (0, 1):
        b = Batch(fam, "jac_psi", alias)
        for P in pts + [None]:
            b.cases.append(Case((fmt(P),), w_row(g, jac_enc(g, P, rng.choice(lams[2:]))), None if P is None else o.g2_psi(P), "jac"))
        out.append(b)
        b = Batch(fam, "clear_cofactor", alias)
        for P in pts + [None]:
            b.cases.append(Case((fmt(P),), w_row(g, jac_enc(g, P, rng.choice(lams[2:]))), h2c2.clear_cofactor(P), "jac"))
        out.append(b)
    return out


@functools.lru_cache(maxsize=None)
def w_batches(name: str):
    return w_batches_for(name)


# ---- expand_message_xmd ---------------------------------------------------------------------------------------------------------
XMD_DSTS = [1, 21, 22, 43, 55, 56, 200, 255]


def xmd_msg_lengths(dst_len: int):
    """message lengths where the padded b0 input (Z_pad || msg || l_i_b || 0 || DST || len) sits at a SHA-256 block edge"""
    out = {0, 1, 255}
    for m in range(256):
        if (64 + m + 3 + dst_len + 1) % 64 in (54, 55, 56, 63, 0, 1):
            out.add(m)
    return sorted(out)


@functools.lru_cache(maxsize=None)
def xmd_batches():
    rng = random.Random("curve-cases/xmd")
    out = []
    for op, length in (("expand_message_xmd_128", 128), ("expand_message_xmd_256", 256)):
        b = Batch("xmd", op, 0)
        for dl in XMD_DSTS:
            dst = bytes(rng.randrange(32, 127) for _ in range(dl))
            for ml in xmd_msg_lengths(dl):
                msg = rng.randbytes(ml)
                row = ml.to_bytes(4, "little") + dl.to_bytes(4, "little") + msg.ljust(256, b"\0") + dst.ljust(256, b"\0")
                want = h2c1.expand_message_xmd(msg, dst, length)
                b.cases.append(Case((f"msg {ml} B", f"dst {dl} B"), row, want, "xmd"))
        out.append(b)
    return out


def xmd_check(batch: Batch, got: np.ndarray, layout: str, limit: int = 5):
    msgs, count = [], 0
    for i, c in enumerate(batch.cases):
        g = got[i * 64:(i + 1) * 64].astype("<u4").tobytes()[:len(c.want)]
        if g != c.want:
            count += 1
            if len(msgs) < limit:
                msgs.append(f"[{layout}] {batch.op} case {i}: {c.operands}: got {g.hex()}, want {c.want.hex()}")
    return count, msgs


# ---- edwards25519 -------------------------------------------------------------------------------------------------------------
EFLD = Fld(ed.P, 8, 1)
ED_IN, ED_OUT = 81, 41


def ed_neg(P):
    return (-P[0] % ed.P, P[1])


def ed_mul(k, P):
    acc, q = (0, 1), P
    while k:
        if k & 1:
            acc = ed.add(acc, q)
        q = ed.add(q, q)
        k >>= 1
    return acc


def ed_ext(P, lam=1):
    x, y = P
    return [x * lam % ed.P, y * lam % ed.P, lam % ed.P, x * y % ed.P * lam % ed.P]


def ed_row(A=None, B=None, by=b"", k=0, w=0):
    A = A or [0, 1, 1, 0]
    B = B or [0, 1, 1, 0]
    return (b"".join(EFLD.enc(c) for c in A) + b"".join(EFLD.enc(c) for c in B) + by.ljust(32, b"\0")
            + (k % (1 << 256)).to_bytes(32, "little") + w.to_bytes(4, "little"))


@functools.lru_cache(maxsize=None)
def ed_torsion():
    """the 8 points of the 8-torsion, T8[j] = j T for a point T of order 8"""
    rng = random.Random("curve-cases/ed-torsion")
    while True:
        P = ed.decode(rng.randbytes(32))
        if P is None:
            continue
        T = ed_mul(ed.L, P)
        if ed_mul(4, T) != (0, 1):
            return [ed_mul(j, T) for j in range(8)]


def ed_recoded_mul(k: int, P):
    """geScalarMult's signed radix-16 schedule (ed_mul_var): the top digit is used only when it is at most 8"""
    e, carry = [], 0
    for i in range(63):
        v = ((k >> (4 * i)) & 15) + carry
        carry = (v + 8) >> 4
        e.append(v - (carry << 4))
    e.append((k >> 252) + carry)
    total = sum(d << (4 * i) for i, d in enumerate(e) if i < 63 or d <= 8)
    return ed_mul(total, P) if total >= 0 else ed_mul(-total, ed_neg(P))


def ed_bytes_cases(rng):
    """encodings: random points, the 8-torsion with both sign bits, the identity with the sign bit, the 19 y >= p with both sign
    bits, and y with no x"""
    T8 = ed_torsion()
    out = []
    for j in range(1, 6):
        out.append(ed.encode(ed_mul(j * 7919, ed.BASE)))
    for T in T8:
        e = ed.encode(T)
        out += [e, bytes(e[:31]) + bytes([e[31] ^ 0x80])]
    out.append((1 | (1 << 255)).to_bytes(32, "little"))
    for j in range(19):
        y = ed.P + j
        out += [y.to_bytes(32, "little"), (y | (1 << 255)).to_bytes(32, "little")]
    nox = 0
    while nox < 6:
        bb = rng.randbytes(32)
        if ed.decode(bb) is None:
            out.append(bb)
            nox += 1
    return out


@functools.lru_cache(maxsize=None)
def ed_batches():
    rng = random.Random("curve-cases/ed")
    T8 = ed_torsion()
    base = [ed_mul(k, ed.BASE) for k in (1, 2, 3, 7, 1 << 100, ed.L - 1)]
    mixed = [ed.add(base[1], T8[1]), ed.add(base[2], T8[4]), ed.add(base[3], T8[6])]
    pts = base + T8 + mixed

    def lam():
        return rng.randrange(1, ed.P)

    out = []
    pairs = []
    for i, P in enumerate(pts):
        Q = pts[(i + 3) % len(pts)]
        pairs += [(P, Q), (P, P), (P, ed_neg(P)), (P, (0, 1))]
    for alias in (0, 1, 2, 3):
        b = Batch("ed", "ed_add", alias)
        for P, Q in pairs:
            want = ed.add(P, P) if alias == 3 else ed.add(P, Q)
            b.cases.append(Case((fmt(P), fmt(Q)), ed_row(ed_ext(P, lam()), ed_ext(Q, lam())), want, "ed"))
        out.append(b)
    for opname, kind in (("ed_dbl", "ed"), ("ed_dbl_xyz", "ed_xyz")):
        for alias in (0, 1):
            b = Batch("ed", opname, alias)
            for P in pts:
                for l in (1, lam()):
                    b.cases.append(Case((fmt(P), l), ed_row(ed_ext(P, l)), ed.add(P, P), kind))
            out.append(b)
    for alias in (0, 1):
        b = Batch("ed", "ed_add_cached", alias)
        for P, Q in pairs:
            for w in range(4):
                lq = lam() if w & 1 else 1                 # without 2 Z the operand must have Z = 1
                want = ed.add(P, ed_neg(Q) if w & 2 else Q)
                b.cases.append(Case((fmt(P), fmt(Q), f"z2 {w & 1}", f"neg {w >> 1}"), ed_row(ed_ext(P, lam()), ed_ext(Q, lq), w=w),
                                    want, "ed"))
        out.append(b)
    b = Batch("ed", "ed_madd", 1)
    for P, Q in pairs:
        for w in (0, 1):
            b.cases.append(Case((fmt(P), fmt(Q), f"neg {w}"), ed_row(ed_ext(P, lam()), ed_ext(Q), w=w),
                                ed.add(P, ed_neg(Q) if w else Q), "ed"))
    out.append(b)
    encs = ed_bytes_cases(rng)
    for opname in ("ed_decode", "ed_decode_aff"):
        b = Batch("ed", opname, 0)
        for e in encs:
            d = ed.decode(e)
            want = ((0, 1) if opname == "ed_decode_aff" else None, False) if d is None else (d, True)
            b.cases.append(Case((e.hex(),), ed_row(by=e), want, "ed_aff" if opname == "ed_decode_aff" else "ed_z1"))
        out.append(b)
    b = Batch("ed", "ed_bytes_canonical", 0)
    for e in encs:
        b.cases.append(Case((e.hex(),), ed_row(by=e), (int.from_bytes(e, "little") & ((1 << 255) - 1)) < ed.P, "flag"))
    out.append(b)
    b = Batch("ed", "ed_has_small_order", 0)
    for e in encs:
        d = ed.decode(e)
        if d is not None:
            b.cases.append(Case((e.hex(),), ed_row(ed_ext(d)), ed_mul(8, d) == (0, 1), "flag"))
    out.append(b)
    for opname in ("ed_encode", "ed_encode_z1"):
        b = Batch("ed", opname, 0)
        for P in pts:
            b.cases.append(Case((fmt(P),), ed_row(ed_ext(P, lam() if opname == "ed_encode" else 1)), ed.encode(P), "ed_bytes"))
        out.append(b)
    b = Batch("ed", "ed_eq", 0)
    for i, P in enumerate(pts):
        Q = pts[(i + 1) % len(pts)]
        for A, B in ((P, P), (P, ed_neg(P)), (P, Q)):
            b.cases.append(Case((fmt(A), fmt(B)), ed_row(ed_ext(A, lam()), ed_ext(B, lam())), A == B, "flag"))
    out.append(b)
    L = ed.L
    ks = list(range(18)) + [L, 8 * L, L - 1, L + 1, (1 << 256) - 1, int("8" * 64, 16), int("7" * 64, 16), int("f" * 64, 16),
                            1 << 255, int("8" * 63, 16), (1 << 252) - 1] + [rng.getrandbits(256) for _ in range(6)]
    for opname in ("ed_scalar_mul", "ed_mul_var"):
        b = Batch("ed", opname, 0)
        for P in (base[0], T8[1], mixed[0]):
            for k in ks:
                want = ed_mul(k, P) if opname == "ed_scalar_mul" else ed_recoded_mul(k, P)
                b.cases.append(Case((fmt(P), hex(k)), ed_row(ed_ext(P, lam()), k=k), want, "ed"))
        out.append(b)
    return out


def ed_check(batch: Batch, got: np.ndarray, layout: str, limit: int = 5):
    msgs, count = [], 0
    p = ed.P
    for i, c in enumerate(batch.cases):
        row = got[i * ED_OUT:(i + 1) * ED_OUT]
        X, Y, Z, T = (EFLD.dec(row[8 * j:8 * (j + 1)]) for j in range(4))
        by = row[32:40].astype("<u4").tobytes()
        flag = int(row[40])
        err = None
        if c.kind == "flag":
            if flag != int(c.want):
                err = f"flag {flag}, want {int(c.want)}"
        elif c.kind == "ed_bytes":
            if by != c.want:
                err = f"bytes {by.hex()}, want {c.want.hex()}"
        elif c.kind in ("ed_z1", "ed_aff"):
            want, ok = c.want
            if flag != int(ok):
                err = f"flag {flag}, want {int(ok)}"
            elif want is not None and (X, Y) != want:
                err = f"point {fmt((X, Y))}, want {fmt(want)}"
            elif c.kind == "ed_z1" and ok and (Z != 1 or T != X * Y % p):
                err = f"Z {Z}, T {T}: want Z = 1, T = x y"
        else:
            if Z == 0:
                err = "Z = 0"
            else:
                zi = pow(Z, -1, p)
                pt = (X * zi % p, Y * zi % p)
                if pt != c.want:
                    err = f"point {fmt(pt)}, want {fmt(c.want)}"
                elif c.kind == "ed" and X * Y % p != Z * T % p:
                    err = "X Y != Z T"
        if err:
            count += 1
            if len(msgs) < limit:
                msgs.append(f"[{layout}] {batch.op} {ALIASES[batch.alias]} case {i}: operands {c.operands}: {err}")
    return count, msgs


# ---- running a family -----------------------------------------------------------------------------------------------------------
def families():
    return [f"w_{n}" for n in GROUPS] + ["xmd", "ed"]


def batches(family: str):
    if family.startswith("w_"):
        return w_batches(family[2:])
    return xmd_batches() if family == "xmd" else ed_batches()


def run_family(lib, family: str, layout: str, device: bool):
    """every batch of one family through one build; returns the failure messages"""
    failures = []
    for b in batches(family):
        if b.op in DEVICE_ONLY and not device:
            continue
        if family.startswith("w_"):
            g = GROUPS[family[2:]]
            iw, ow = w_sizes(g)
            got = call(lib, family, b.opcode, b.alias, b.inp(), len(b.cases), ow)
            count, msgs = w_check(g, b, got, layout)
        elif family == "xmd":
            got = call(lib, "xmd", b.opcode, 0, b.inp(), len(b.cases), 64)
            count, msgs = xmd_check(b, got, layout)
        else:
            got = call(lib, "ed", b.opcode, b.alias, b.inp(), len(b.cases), ED_OUT)
            count, msgs = ed_check(b, got, layout)
        if count:
            failures.append(f"{count} of {len(b.cases)} wrong:\n  " + "\n  ".join(msgs))
    return failures


def case_counts(device: bool):
    """{(family, operation): cases} over every alias mode"""
    out = {}
    for fam in families():
        for b in batches(fam):
            if b.op in DEVICE_ONLY and not device:
                continue
            out[(fam, b.op)] = out.get((fam, b.op), 0) + len(b.cases)
    return out
