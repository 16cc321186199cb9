"""Reference restatement and inputs of the Neff shuffle tests on edwards25519 (CPU oracle tests, host emulation, GPU).

Restates, from the in-tree reference:
  proof.HashProve / HashVerify   proof/hash.go:12-175: pubrand = blake2xb.New(protocolName); every PubRand first Reseeds (128
                                 stream bytes -> New(them): key = the first 64, message = the last 64, xof/blake2xb/blake.go:55-75)
                                 and Writes the RAW message bytes put / read since the last PubRand; scalars are then Picked
                                 (ScalarUnmarshalFrom on a cipher.Stream, group/internal/marshalling/marshal.go:53-63)
                                 -> HashProver, HashVerifier
  PairShuffle.Prove / Verify     shuffle/pair.go:129-312                                     -> pair_prove, pair_verify
  SimpleShuffle.Prove / Verify   shuffle/simple.go:91-254 (thver :178-183)                   -> simple_prove, simple_verify
  Shuffle                        pair.go:318-361                                             -> shuffle
  SequencesShuffle               shuffle/sequences.go:36-124                                 -> sequences_shuffle
  GetSequenceVerifiable          sequences.go:155-190                                        -> get_sequence_verifiable
The prover's private randomness comes from a deterministic stream (pvss_cases.RandomStream), not the suite's.  Point
multiplications go through a callback `mul(scalars, points) -> points` (raw integers, Point.Mul semantics, points as 32-byte
encodings, None = the base point) so bulk inputs can use the engine's b2k_ed25519_mul_batch; the default is the Python
geScalarMult (ed25519_msm_cases.ge_scalar_mult).  The prover takes its point arithmetic from an ops object: BytesOps (encodings,
through `mul`) or, for large honest inputs, DlogOps (discrete logs, one batched encoding per message).  The large absorbs hash with hashlib.blake2b and the BLAKE2X parameters
(FastXof); test_oracle_shuffle.py checks that against the explicit form (pvss_cases.Xof).
"""
from __future__ import annotations

import hashlib
import random

from oracle import ed25519 as ed
import ed25519_msm_cases as mc
import pvss_cases as pc

L = ed.L
OK, SIMPLE, PAIR, POINT = 0, 1, 2, 3
G = pc.G


class PointError(Exception):
    """a point of the proof or of the inputs does not decode: the reference's Get / the caller fails first"""


class ProofError(Exception):
    def __init__(self, status: int):
        super().__init__({SIMPLE: "incorrect SimpleShuffleProof", PAIR: "invalid PairShuffleProof"}[status])
        self.status = status


# ---- the XOF ----------------------------------------------------------------------------------------------------------------
class FastXof(pc.Xof):
    """blake2xb.New(seed) + Write(extra) with the root on hashlib: BLAKE2b-512 keyed with seed[:64] over seed[64:] || extra,
    fanout 1, depth 1, XOF length 2^32 - 1.  The output blocks (depth 0, which hashlib does not take) stay pvss_cases.Xof's."""

    def __init__(self, seed: bytes = b"", extra: bytes = b""):
        self.root = hashlib.blake2b(seed[64:] + extra, digest_size=64, key=seed[:64], fanout=1, depth=1,
                                    node_offset=0xFFFFFFFF << 32).digest()
        self.block, self.buf = 0, b""


class _Transcript:
    xof_class = FastXof

    def __init__(self, proto: bytes):
        self.x = self.xof_class(proto)

    def _stir(self, msg: bytes):
        """consumeMsg: Reseed, then Write(msg)"""
        key = self.x.read(128)
        self.x = self.xof_class(key, msg)

    def _picks(self, n: int):
        return [pc.pick_int(self.x) for _ in range(n)]


class HashProver(_Transcript):
    def __init__(self, proto: bytes):
        super().__init__(proto)
        self.msg, self.proof = b"", b""

    def put(self, data: bytes):
        self.msg += data

    def pub_rand(self, n: int):
        if self.msg:
            self._stir(self.msg)
            self.proof += self.msg
            self.msg = b""
        return self._picks(n)

    def final(self) -> bytes:
        return self.proof + self.msg


class HashVerifier(_Transcript):
    def __init__(self, proto: bytes, proof: bytes):
        super().__init__(proto)
        self.proof, self.read, self.mark = proof, 0, 0

    def _take(self, n: int):
        if self.read + 32 * n > len(self.proof):
            raise PointError("short proof")
        out = [self.proof[self.read + 32 * i:self.read + 32 * i + 32] for i in range(n)]
        self.read += 32 * n
        return out

    def get_points(self, n: int):
        out = self._take(n)
        for p in out:
            if ed.decode(p) is None:
                raise PointError("invalid Ed25519 curve point")
        return out

    def get_scalars(self, n: int):
        return [int.from_bytes(s, "little") for s in self._take(n)]       # raw, UnmarshalBinary does not reduce

    def pub_rand(self, n: int):
        if self.read > self.mark:
            self._stir(self.proof[self.mark:self.read])
            self.mark = self.read
        return self._picks(n)


# ---- point arithmetic through a multiplication callback ------------------------------------------------------------------------
def py_mul(scalars, points):
    """[Point.Mul(k, P)] with geScalarMult's semantics for raw k; P None = the base point (geScalarMultBase drops a top digit
    above 8 the same way)"""
    return [ed.encode(mc.ge_scalar_mult((k % (1 << 256)).to_bytes(32, "little"), ed.decode(p if p is not None else G)))
            for k, p in zip(scalars, points)]


def add(a: bytes, b: bytes) -> bytes:
    return ed.encode(ed.add(ed.decode(a), ed.decode(b)))


def neg(a: bytes) -> bytes:
    x, y = ed.decode(a)
    return ed.encode(((-x) % ed.P, y))


def sub(a: bytes, b: bytes) -> bytes:
    return add(a, neg(b))


def equal(a: bytes, b: bytes) -> bool:
    return pc.canon(a) == pc.canon(b)


def total(pts) -> bytes:
    acc = ed.IDENT
    for p in pts:
        acc = ed.add(acc, ed.decode(p))
    return ed.encode(acc)


def proof_len(k: int) -> int:
    return 32 * (12 * k + 3)


def le(v: int) -> bytes:
    return (v % (1 << 256)).to_bytes(32, "little")


class BytesOps:
    """the prover's point arithmetic on 32-byte encodings, multiplications through `mul`"""
    base = None

    def __init__(self, mul=None):
        self.mul = mul or py_mul

    add = staticmethod(add)
    total = staticmethod(total)

    def enc(self, pts):
        return list(pts)


class DlogOps:
    """the prover's points as their discrete logs to the base point (honest inputs without torsion only): adds are scalar adds,
    and the encodings of a message come from one call of `mul_base(scalars) -> encodings` (e.g. b2k_ed25519_mul_batch)"""
    base = 1

    def __init__(self, mul_base):
        self.mul_base = mul_base

    def mul(self, scalars, pts):
        return [a * (1 if p is None else p) % L for a, p in zip(scalars, pts)]

    def add(self, a, b):
        return (a + b) % L

    def total(self, pts):
        return sum(pts) % L

    def enc(self, pts):
        return self.mul_base(list(pts))


def _ops(ops):
    return ops if ops is not None else BytesOps()


# ---- SimpleShuffle ------------------------------------------------------------------------------------------------------------
def simple_prove(ctx: HashProver, g, gamma: int, x, y, rs: pc.RandomStream, ops=None):
    ops = _ops(ops)
    k = len(x)
    assert k > 1 and len(y) == k
    X = ops.mul(x, [g] * k)
    Y = ops.mul(y, [g] * k)
    ctx.put(b"".join(ops.enc(X + Y)))                                    # ssa0
    t, = ctx.pub_rand(1)
    gamma_t = gamma * t % L
    xhat = [(xi - t) % L for xi in x]
    yhat = [(yi - gamma_t) % L for yi in y]
    thlen = 2 * k - 1
    theta = [rs.scalar() for _ in range(thlen)]
    e = [(-theta[0] * yhat[0]) % L]
    e += [(theta[i - 1] * xhat[i] - theta[i] * yhat[i]) % L for i in range(1, k)]
    e += [(theta[i - 1] * gamma - theta[i]) % L for i in range(k, thlen)]
    e += [theta[thlen - 1] * gamma % L]
    Theta = ops.mul(e, [g] * (thlen + 1))
    ctx.put(b"".join(ops.enc(Theta)))                                    # ssa2
    c, = ctx.pub_rand(1)
    alpha = [0] * thlen
    runprod = c
    for i in range(k):
        runprod = runprod * xhat[i] % L * pow(yhat[i], -1, L) % L
        alpha[i] = (theta[i] + runprod) % L
    gammainv = pow(gamma, -1, L)
    rungamma = c
    for i in range(1, k):
        rungamma = rungamma * gammainv % L
        alpha[thlen - i] = (theta[thlen - i] + rungamma) % L
    ctx.put(b"".join(le(a) for a in alpha))                              # ssa4


def thver_terms(k, Xhat, Yhat, Theta, G_, Gamma, alpha, c):
    """the 2k thver operands (A, B, T, a, b) of SimpleShuffle.Verify, in order"""
    out = [(Xhat[0], Yhat[0], Theta[0], c, alpha[0])]
    out += [(Xhat[i], Yhat[i], Theta[i], alpha[i - 1], alpha[i]) for i in range(1, k)]
    out += [(Gamma, G_, Theta[i], alpha[i - 1], alpha[i]) for i in range(k, 2 * k - 1)]
    out += [(Gamma, G_, Theta[2 * k - 1], alpha[2 * k - 2], c)]
    return out


def thver(A, B, T, a: int, b: int, mul=py_mul) -> bool:
    """P = a A (a raw), Q = Neg(b) B (b negated and reduced mod l), P + Q == T"""
    P, Q = mul([a, (-b) % L], [A, B])
    return equal(add(P, Q), T)


def simple_verify(ctx: HashVerifier, k: int, g, Gamma, mul=py_mul):
    X = ctx.get_points(k)
    Y = ctx.get_points(k)
    t, = ctx.pub_rand(1)
    Theta = ctx.get_points(2 * k)
    c, = ctx.pub_rand(1)
    alpha = ctx.get_scalars(2 * k - 1)
    negt = (-t) % L
    U, W = mul([negt, negt], [g, Gamma])
    Xhat = [add(xi, U) for xi in X]
    Yhat = [add(yi, W) for yi in Y]
    terms = thver_terms(k, Xhat, Yhat, Theta, g if g is not None else G, Gamma, alpha, c)
    res = mul([s for tm in terms for s in (tm[3], (-tm[4]) % L)], [p for tm in terms for p in (tm[0], tm[1])])
    good = all(equal(add(res[2 * i], res[2 * i + 1]), tm[2]) for i, tm in enumerate(terms))
    if not good:
        raise ProofError(SIMPLE)
    return {"X": X, "Y": Y, "t": t, "c": c, "Theta": Theta, "alpha": alpha}


# ---- PairShuffle --------------------------------------------------------------------------------------------------------------
def pair_prove(ctx: HashProver, pi, g, h, beta, X, Y, rs: pc.RandomStream, ops=None):
    ops = _ops(ops)
    g = ops.base if g is None else g
    h = ops.base if h is None else h
    k = len(pi)
    piinv = [0] * k
    for i in range(k):
        piinv[pi[i]] = i
    u = [rs.scalar() for _ in range(k)]
    w = [rs.scalar() for _ in range(k)]
    a = [rs.scalar() for _ in range(k)]
    tau0, _nu, gamma = rs.scalar(), rs.scalar(), rs.scalar()
    Gamma, = ops.mul([gamma], [g])
    A = ops.mul(a, [g] * k)
    C = ops.mul([gamma * a[pi[i]] % L for i in range(k)], [g] * k)
    U = ops.mul(u, [g] * k)
    W = ops.mul([gamma * w[i] % L for i in range(k)], [g] * k)
    wbetasum = (tau0 + sum(w[i] * beta[pi[i]] for i in range(k))) % L
    wu = [(w[piinv[i]] - u[i]) % L for i in range(k)]
    Lambda1 = ops.total(ops.mul(wu + [wbetasum], list(X) + [g]))
    Lambda2 = ops.total(ops.mul(wu + [wbetasum], list(Y) + [h]))
    ctx.put(b"".join(ops.enc([Gamma] + A + C + U + W + [Lambda1, Lambda2])))                        # ega1
    zrho = ctx.pub_rand(k)
    b = [(zrho[i] - u[i]) % L for i in range(k)]
    d = [gamma * b[pi[i]] % L for i in range(k)]
    D = ops.mul(d, [g] * k)
    ctx.put(b"".join(ops.enc(D)))                                                                    # ega3
    zlambda, = ctx.pub_rand(1)
    r = [(a[i] + zlambda * b[i]) % L for i in range(k)]
    s = [gamma * r[pi[i]] % L for i in range(k)]
    ztau = (-tau0 + sum(b[i] * beta[i] for i in range(k))) % L
    zsigma = [(w[i] + b[pi[i]]) % L for i in range(k)]
    ctx.put(b"".join(le(z) for z in zsigma) + le(ztau))                                              # ega5
    simple_prove(ctx, g, gamma, r, s, rs, ops)


def pair_verify(ctx: HashVerifier, k: int, g, h, X, Y, Xbar, Ybar, mul=py_mul):
    p1 = ctx.get_points(4 * k + 3)
    Gamma, Wv = p1[0], p1[3 * k + 1:4 * k + 1]
    Lambda1, Lambda2 = p1[4 * k + 1], p1[4 * k + 2]
    zrho = ctx.pub_rand(k)
    D = ctx.get_points(k)
    ctx.pub_rand(1)                                                       # Zlambda: unused, consumes stream
    zsigma = ctx.get_scalars(k)
    ztau, = ctx.get_scalars(1)
    simple_verify(ctx, k, g, Gamma, mul)
    terms = mul(zsigma + zrho + zsigma + zrho + zsigma + [ztau, ztau],
                list(Xbar) + list(X) + list(Ybar) + list(Y) + [Gamma] * k + [g, h])
    phi1 = total(sub(terms[i], terms[k + i]) for i in range(k))           # Sub negates the point
    phi2 = total(sub(terms[2 * k + i], terms[3 * k + i]) for i in range(k))
    for i in range(k):
        if not equal(terms[4 * k + i], add(Wv[i], D[i])):                 # (33)
            raise ProofError(PAIR)
    tg, th = terms[5 * k], terms[5 * k + 1]
    if not equal(add(Lambda1, tg), phi1) or not equal(add(Lambda2, th), phi2):   # (34), (35)
        raise ProofError(PAIR)


def hash_verify(proto: bytes, g, h, X, Y, Xbar, Ybar, proof: bytes, mul=py_mul) -> int:
    """proof.HashVerify(suite, proto, shuffle.Verifier(suite, g, h, X, Y, Xbar, Ybar), proof) as a status; g / h None = the
    base point"""
    k = len(X)
    assert k >= 2 and len(Y) == len(Xbar) == len(Ybar) == k
    if not pc.decodes(*(p for p in (g, h) if p is not None), *X, *Y, *Xbar, *Ybar):
        return POINT
    try:
        pair_verify(HashVerifier(proto, proof), k, g, h, X, Y, Xbar, Ybar, mul)
    except PointError:
        return POINT
    except ProofError as e:
        return e.status
    return OK


# ---- Shuffle and the sequence variant --------------------------------------------------------------------------------------
def permutation(k: int, rng: random.Random):
    pi = list(range(k))
    for i in range(k - 1, 0, -1):
        j = rng.randrange(i + 1)
        pi[i], pi[j] = pi[j], pi[i]
    return pi


def shuffle(g, h, X, Y, proto: bytes, seed: str, ops=None):
    """Shuffle + HashProve: (Xbar, Ybar, proof) in the representation of ops; the permutation and the blinding factors come
    from seed"""
    ops = _ops(ops)
    k = len(X)
    rng = random.Random(seed)
    rs = pc.RandomStream(seed)
    pi = permutation(k, rng)
    beta = [rs.scalar() for _ in range(k)]
    bg = ops.mul([beta[pi[i]] for i in range(k)], [ops.base if g is None else g] * k)
    bh = ops.mul([beta[pi[i]] for i in range(k)], [ops.base if h is None else h] * k)
    Xbar = [ops.add(bg[i], X[pi[i]]) for i in range(k)]
    Ybar = [ops.add(bh[i], Y[pi[i]]) for i in range(k)]
    ctx = HashProver(proto)
    pair_prove(ctx, pi, g, h, beta, X, Y, rs, ops)
    return Xbar, Ybar, ctx.final()


def get_sequence_verifiable(X, Y, Xbar, Ybar, e, mul=py_mul):
    """xUp[i] = sum_j e[j] X[j][i] (Mul then Add), likewise yUp, xDown, yDown; e raw integers"""
    nq, k = len(X), len(X[0])
    out = []
    for M in (X, Y, Xbar, Ybar):
        prods = mul([e[j] for i in range(k) for j in range(nq)], [M[j][i] for i in range(k) for j in range(nq)])
        out.append([total(prods[i * nq:(i + 1) * nq]) for i in range(k)])
    return tuple(out)


def sequences_shuffle(g, h, X, Y, e, proto: bytes, seed: str, mul=py_mul):
    """SequencesShuffle + getProver(e) + HashProve: (Xbar, Ybar, proof) over the NQ x k sequences; the proof is a PairShuffle
    proof over GetSequenceVerifiable's (xUp, yUp) -> (xDown, yDown)"""
    nq, k = len(X), len(X[0])
    rng = random.Random(seed)
    rs = pc.RandomStream(seed)
    pi = permutation(k, rng)
    beta = [[rs.scalar() for _ in range(k)] for _ in range(nq)]
    Xbar, Ybar = [], []
    for j in range(nq):
        bg = mul([beta[j][pi[i]] for i in range(k)], [g] * k)
        bh = mul([beta[j][pi[i]] for i in range(k)], [h] * k)
        Xbar.append([add(bg[i], X[j][pi[i]]) for i in range(k)])
        Ybar.append([add(bh[i], Y[j][pi[i]]) for i in range(k)])
    beta2 = [sum(e[j] * beta[j][i] for j in range(nq)) % L for i in range(k)]
    xup, yup, _, _ = get_sequence_verifiable(X, Y, Xbar, Ybar, e, mul)
    ctx = HashProver(proto)
    pair_prove(ctx, pi, g, h, beta2, xup, yup, rs, BytesOps(mul))
    return Xbar, Ybar, ctx.final()


# ---- inputs ---------------------------------------------------------------------------------------------------------------------
def elgamal_pairs(k: int, rng: random.Random, h=None, ops=None, torsion: bool = False):
    """k ElGamal pairs (X, Y) = (r G, r H + M) of random messages M = m G in the representation of ops; torsion adds an
    order-8 component to M (encodings only)"""
    ops = _ops(ops)
    r = [rng.randrange(1, L) for _ in range(k)]
    msg = [rng.randrange(1, L) for _ in range(k)]
    b = ops.base
    prods = ops.mul(r + r + msg, [b] * k + [b if h is None else h] * k + [b] * k)
    X, rh, M = prods[:k], prods[k:2 * k], prods[2 * k:]
    if torsion:
        M = [add(mi, mc.point(0, rng.randrange(1, 8))) for mi in M]
    return X, [ops.add(a, c) for a, c in zip(rh, M)]


def items(proof: bytes):
    return [proof[i:i + 32] for i in range(0, len(proof), 32)]


def with_item(proof: bytes, j: int, b: bytes) -> bytes:
    return proof[:32 * j] + b + proof[32 * j + 32:]


# item indices of the proof (see include/b2kyber.h)
def item(k: int, name: str, i: int = 0) -> int:
    base = {"Gamma": 0, "A": 1, "C": k + 1, "U": 2 * k + 1, "W": 3 * k + 1, "Lambda1": 4 * k + 1, "Lambda2": 4 * k + 2,
            "D": 4 * k + 3, "Zsigma": 5 * k + 3, "Ztau": 6 * k + 3, "X": 6 * k + 4, "Y": 7 * k + 4, "Theta": 8 * k + 4,
            "Zalpha": 10 * k + 4}[name]
    return base + i


def noncanonical(b: bytes):
    """a non-canonical encoding of the same point (y + p), or None when y + p does not fit (y >= 19)"""
    y = int.from_bytes(b, "little") & ((1 << 255) - 1)
    if y + ed.P >= 1 << 255:
        return None
    return ((y + ed.P) | (int.from_bytes(b, "little") & (1 << 255))).to_bytes(32, "little")
