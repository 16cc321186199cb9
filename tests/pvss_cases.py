"""Reference restatement and inputs of the DLEQ / PVSS tests on edwards25519 (CPU oracle tests, host emulation, GPU).

Restates, from the in-tree reference:
  blake2xb.New(seed)        xof/blake2xb/blake.go:19-41: blake2b.NewXOF(OutputLengthUnknown, seed[:64]) -- the first 64 bytes are
                            the BLAKE2b KEY -- then Write(seed[64:]); output block i is an unkeyed BLAKE2b-512 of the root hash
                            with the BLAKE2X node parameters (golang.org/x/crypto/blake2b/blake2x.go)        -> Xof
  Scalar.Pick               scalar.go:180-185 -> random.Int(l), util/random/rand.go:19-46                    -> pick
  dleq.NewDLEQProof/Verify  proof/dleq/dleq.go:41-86, :161-172 (Verify through Point.Mul = geScalarMult)    -> new_dleq_proof, dleq_verify
  pvss                      share/pvss/pvss.go: EncShares :51-92, computeCommitments :94-114, computeGlobalChallenge
                            :116-149, VerifyEncShare(Batch) :154-194, DecShare :199-217, VerifyDecShare(Batch) :248-299,
                            RecoverSecret :303-323
oracle.ed25519.Blake2Xb treats its seed as the message, which agrees with blake2xb.New only for the empty seed (the dh KAT's);
Xof here is the keyed construction, and test_oracle_pvss.py checks the two agree on the empty seed.
"""
from __future__ import annotations

import hashlib
import random

from oracle import ed25519 as ed
from oracle.ed25519 import _blake2b, _param
import ed25519_msm_cases as mc

L, P = ed.L, ed.P
OK, CHALLENGE, INVALID, POINT = 0, 1, 2, 3


# ---- keyed BLAKE2Xb and Pick ------------------------------------------------------------------------------------------------
def blake2b_keyed(key: bytes, msg: bytes, param: bytes) -> bytes:
    """BLAKE2b-512 with the parameter block `param` (its key-length byte set here): a key is a zero-padded first block"""
    param = param[:1] + bytes([len(key)]) + param[2:]
    return _blake2b((key.ljust(128, b"\x00") if key else b"") + msg, param, 64)


class Xof:
    """blake2xb.New(seed) followed by Write(extra): the stream that XORKeyStream / Read yield"""

    def __init__(self, seed: bytes = b"", extra: bytes = b""):
        key, msg = seed[:64], seed[64:] + extra
        self.root = blake2b_keyed(key, msg, _param(64, 1, 1, 0, 0, 0xFFFFFFFF, 0, 0))
        self.block, self.buf = 0, b""

    def block_bytes(self, i: int) -> bytes:
        return _blake2b(self.root, _param(64, 0, 0, 64, i, 0xFFFFFFFF, 0, 64), 64)

    def read(self, n: int) -> bytes:
        while len(self.buf) < n:
            self.buf += self.block_bytes(self.block)
            self.block += 1
        out, self.buf = self.buf[:n], self.buf[n:]
        return out


def pick_int(x: Xof) -> int:
    """random.Int(l): 32 bytes, the top 3 bits of the first cleared, big-endian, drawn again while >= l"""
    while True:
        b = bytearray(x.read(32))
        b[0] &= 0x1F
        v = int.from_bytes(b, "big")
        if v < L:
            return v


def pick(x: Xof) -> bytes:
    """Scalar.Pick: the little-endian 32 bytes of random.Int(l)"""
    return pick_int(x).to_bytes(32, "little")


def pick_draws(seed: bytes) -> int:
    """how many 32-byte draws Pick(blake2xb.New(seed)) takes"""
    x, k = Xof(seed), 0
    while True:
        k += 1
        b = bytearray(x.read(32))
        b[0] &= 0x1F
        if int.from_bytes(b, "big") < L:
            return k


class RandomStream:
    """a deterministic stand-in for suite.RandomStream(): an Xof over a label"""

    def __init__(self, label: str):
        self.x = Xof(hashlib.sha256(label.encode()).digest())

    def scalar(self) -> int:
        return pick_int(self.x)


# ---- points -----------------------------------------------------------------------------------------------------------------
def canon(b: bytes) -> bytes:
    """MarshalTo of the decoded point: its canonical encoding"""
    pt = ed.decode(b)
    assert pt is not None
    return ed.encode(pt)


def mul(k: int, pt_bytes: bytes) -> bytes:
    """Point.Mul(k, P) for the raw integer k (geScalarMult's top-digit rule included)"""
    return ed.encode(mc.ge_scalar_mult(k.to_bytes(32, "little"), ed.decode(pt_bytes)))


def add(a: bytes, b: bytes) -> bytes:
    return ed.encode(ed.add(ed.decode(a), ed.decode(b)))


def base_mul(k: int) -> bytes:
    return ed.encode(ed.scalar_mult(k % L))


G = ed.encode(ed.BASE)
IDENTITY = mc.IDENTITY
T8 = mc.T8


def challenge(*points: bytes) -> bytes:
    """Pick(XOF(SHA-256 over MarshalTo of the points)) as 32 little-endian bytes"""
    return pick(Xof(hashlib.sha256(b"".join(canon(p) for p in points)).digest()))


# ---- dleq ---------------------------------------------------------------------------------------------------------------------
def new_dleq_proof(g: bytes, h: bytes, x: int, v: int):
    """NewDLEQProof with the commitment v given: (proof C || R || VG || VH, xG, xH)"""
    xg, xh, vg, vh = mul(x, g), mul(x, h), mul(v, g), mul(v, h)
    c = challenge(xg, xh, vg, vh)
    r = (v - x * int.from_bytes(c, "little")) % L
    return c + r.to_bytes(32, "little") + vg + vh, xg, xh


def dleq_holds(g, h, xg, xh, proof) -> bool:
    """VG == R G + C xG and VH == R H + C xH, with the scalars read raw"""
    c, r = int.from_bytes(proof[:32], "little"), int.from_bytes(proof[32:64], "little")
    a = add(mul(r, g), mul(c, xg))
    b = add(mul(r, h), mul(c, xh))
    return canon(proof[64:96]) == a and canon(proof[96:]) == b


def decodes(*pts) -> bool:
    return all(ed.decode(p) is not None for p in pts)


def dleq_verify(g, h, xg, xh, proof) -> int:
    if not decodes(g, h, xg, xh, proof[64:96], proof[96:]):
        return POINT
    return OK if dleq_holds(g, h, xg, xh, proof) else INVALID


# ---- pvss ---------------------------------------------------------------------------------------------------------------------
def eval_commits(commits, x: int) -> bytes:
    """sum_j x^j commits[j] (Horner, as computeCommitments and PubPoly.Eval)"""
    acc = ed.IDENT
    for c in reversed(commits):
        acc = ed.add(ed.scalar_mult(x, acc), ed.decode(c))
    return ed.encode(acc)


def enc_shares(h: bytes, xs, secret: int, t: int, rs: RandomStream):
    """EncShares: (commits, [(index, V, proof)], priv shares); the polynomial and commitments v from rs"""
    coeffs = [secret % L] + [rs.scalar() for _ in range(t - 1)]
    commits = [mul(a, h) for a in coeffs]
    out, priv = [], []
    for i, x in enumerate(xs):
        s = sum(a * pow(i + 1, j, L) for j, a in enumerate(coeffs)) % L
        priv.append(s)
        out.append([i, None, None, None, s])
    # NewDLEQProofBatch(HS, X, values): one challenge over xG[], xH[], vG[], vH[]
    v = [rs.scalar() for _ in xs]
    xg = [mul(s, h) for s in priv]
    xh = [mul(s, x) for s, x in zip(priv, xs)]
    vg = [mul(vi, h) for vi in v]
    vh = [mul(vi, x) for vi, x in zip(v, xs)]
    c = pick(Xof(hashlib.sha256(b"".join(canon(p) for p in xg + xh + vg + vh)).digest()))
    ci = int.from_bytes(c, "little")
    shares = []
    for i in range(len(xs)):
        r = (v[i] - priv[i] * ci) % L
        shares.append((i, xh[i], c + r.to_bytes(32, "little") + vg[i] + vh[i]))
    return commits, shares, priv


def global_challenge(commits, vs, proofs) -> bytes:
    """computeGlobalChallenge over n = len(vs) shares"""
    n = len(vs)
    coms = [eval_commits(commits, i + 1) for i in range(n)]
    data = b"".join(coms) + b"".join(canon(v) for v in vs) + b"".join(canon(p[64:96]) for p in proofs) + \
        b"".join(canon(p[96:]) for p in proofs)
    return pick(Xof(hashlib.sha256(data).digest()))


def verify_enc_share_batch(h, commits, xs, shs, vs, proofs):
    """VerifyEncShareBatch as one status per share (POINT for inputs the reference could not have built)"""
    n = len(xs)
    if not decodes(h, *commits, *vs, *[p[64:96] for p in proofs], *[p[96:] for p in proofs]):
        return [POINT] * n
    gc = global_challenge(commits, vs, proofs)
    out = []
    for x, sh, v, p in zip(xs, shs, vs, proofs):
        if not decodes(x, sh):
            out.append(POINT)
        elif p[:32] != gc:
            out.append(CHALLENGE)
        else:
            out.append(OK if dleq_holds(h, x, sh, v, p) else INVALID)
    return out


def dec_share(x_priv: int, enc_v: bytes, v: int):
    """DecShare without the encrypted-share check: (decV, proof) with commitment v; decV = x^-1 encV"""
    dec_v = mul(pow(x_priv, -1, L), enc_v)
    proof, _, _ = new_dleq_proof(G, dec_v, x_priv, v)
    return dec_v, proof


def verify_dec_share(g, x, enc_v, dec_v, proof) -> int:
    if not decodes(g, x, enc_v, dec_v, proof[64:96], proof[96:]):
        return POINT
    if proof[:32] != challenge(x, enc_v, proof[64:96], proof[96:]):
        return CHALLENGE
    return OK if dleq_holds(g, dec_v, x, enc_v, proof) else INVALID


def lagrange_recover(pairs, t: int) -> bytes:
    """RecoverCommit: the first t of the (index, point) pairs sorted by index, interpolated at 0"""
    pairs = sorted(pairs)[:t]
    acc = ed.IDENT
    for i, (xi, pt) in enumerate(pairs):
        num, den = 1, 1
        for j, (xj, _) in enumerate(pairs):
            if i != j:
                num = num * (xj + 1) % L
                den = den * ((xj + 1) - (xi + 1)) % L
        acc = ed.add(acc, ed.decode(mul(num * pow(den, -1, L) % L, pt)))
    return ed.encode(acc)


def recover_secret(g, xs, enc_vs, dec_shares, t: int):
    """RecoverSecret: None below t valid shares, else RecoverCommit of the valid ones; dec_shares = [(index, decV, proof)]"""
    good = [(i, dv) for (i, dv, p), x, ev in zip(dec_shares, xs, enc_vs) if verify_dec_share(g, x, ev, dv, p) == OK]
    if len(good) < t:
        return None
    return lagrange_recover(good, t)


# ---- input helpers ------------------------------------------------------------------------------------------------------------
def noncanonical_identity() -> bytes:
    """01 00..00 with y + p: y = 2^255 - 18 decodes to the identity; its canonical encoding is 01 00..00"""
    return ((1 << 255) - 18).to_bytes(32, "little")


def undecodable() -> bytes:
    """a y with no x on the curve"""
    y = 2
    while ed.decode(y.to_bytes(32, "little")) is not None:
        y += 1
    return y.to_bytes(32, "little")


def random_point(rng: random.Random, torsion: bool = False) -> bytes:
    return mc.point(rng.randrange(1, L), rng.randrange(8) if torsion else 0)
