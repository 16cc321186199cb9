"""Reference restatement and inputs of the ring signature tests on edwards25519 (CPU oracle tests, host emulation, GPU).

Restates, from the in-tree reference, literally:
  anon.Sign / anon.Verify   sign/anon/sig.go:110-184, :192-248                                    -> sign, verify
  signH1pre / signH1        sig.go:24-46: blake2xb.New(message), Write(scope), Write(tag); Clone, Write(PG [, PH]), Pick -> h1
  Point.Pick = Embed(nil)   group/edwards25519/point.go:132-182: 32-byte chunks of the stream, skip what FromBytes rejects,
                            multiply by the cofactor with geScalarMult, retry on the identity                  -> point_pick
  Point.Mul                 geScalarMult / geScalarMultBase on the RAW scalar (ed25519_msm_cases.ge_scalar_mult; the base
                            schedule drops a top digit above 8 exactly as the variable one does)             -> mul
The XOF and Scalar.Pick are pvss_cases.Xof and pick (blake2xb.New keys BLAKE2b with seed[:64] and writes seed[64:]).
"""
from __future__ import annotations

import random

from oracle import ed25519 as ed
import ed25519_msm_cases as mc
import pvss_cases as pc

L = ed.L
OK, INVALID, POINT = 0, 1, 2
ERR_SIGNATURE, ERR_POINT = "invalid signature", "invalid Ed25519 curve point"


def mul(k: int, p: bytes | None) -> bytes:
    """Point.Mul(k, P) for the raw 32-byte integer k; P None is the base point (geScalarMultBase)"""
    return ed.encode(mc.ge_scalar_mult(k.to_bytes(32, "little"), ed.BASE if p is None else ed.decode(p)))


def add(a: bytes, b: bytes) -> bytes:
    return pc.add(a, b)


def point_pick(x: pc.Xof) -> bytes:
    """Point.Pick(stream): canonical encoding of the point"""
    while True:
        pt = ed.decode(x.read(32))
        if pt is None:
            continue
        q = mc.ge_scalar_mult((8).to_bytes(32, "little"), pt)
        if q == ed.IDENT:
            continue
        return ed.encode(q)


def link_base(scope: bytes) -> bytes:
    return point_pick(pc.Xof(scope))


def h1(msg: bytes, scope: bytes | None, tag: bytes | None, pg: bytes, ph: bytes | None) -> int:
    """signH1(signH1pre(message, scope, tag), PG, PH) as an integer"""
    extra = (scope + tag if scope is not None else b"") + pg + (ph if scope is not None else b"")
    return pc.pick_int(pc.Xof(msg, extra))


def sign(msg: bytes, ring, scope: bytes | None, mine: int, priv: int, rand: pc.Xof, mul=mul) -> bytes:
    """anon.Sign with RandomStream = rand (consumed as the reference consumes it); mul(k, P) may be replaced by another
    Point.Mul (the signer's scalars are canonical)"""
    n, linkable = len(ring), scope is not None
    H = tag = None
    if linkable:
        H = link_base(scope)
        tag = mul(priv, H)
    u = pc.pick_int(rand)
    ub, ul = mul(u, None), (mul(u, H) if linkable else None)
    s, c = [0] * n, [0] * n
    c[(mine + 1) % n] = h1(msg, scope, tag, ub, ul)
    i = (mine + 1) % n
    while i != mine:
        s[i] = pc.pick_int(rand)
        pg = add(mul(s[i], None), mul(c[i], ring[i]))
        ph = add(mul(s[i], H), mul(c[i], tag)) if linkable else None
        c[(i + 1) % n] = h1(msg, scope, tag, pg, ph)
        i = (i + 1) % n
    s[mine] = (u - priv * c[mine]) % L
    return mc.le([c[0]] + s) + (tag if linkable else b"")


def verify(msg: bytes, ring, scope: bytes | None, sig: bytes):
    """anon.Verify on a signature of exactly 32 (n + 1 + linkable) bytes -> (status, tag): tag = canonical Tag when linkable
    and OK, b"" when unlinkable and OK, None on failure"""
    n, linkable = len(ring), scope is not None
    assert len(sig) == 32 * (n + 1 + linkable)
    c0 = int.from_bytes(sig[:32], "little")
    S = [int.from_bytes(sig[32 * (i + 1):32 * (i + 2)], "little") for i in range(n)]
    H = tag = None
    if linkable:
        t = ed.decode(sig[32 * (n + 1):])
        if t is None:
            return POINT, None
        tag = ed.encode(t)
        H = link_base(scope)
    c = c0
    for i in range(n):
        pg = add(mul(S[i], None), mul(c, ring[i]))
        ph = add(mul(S[i], H), mul(c, tag)) if linkable else None
        c = h1(msg, scope, tag, pg, ph)
    if c != c0:
        return INVALID, None
    return OK, (tag if linkable else b"")


def replay_example(e):
    """(message, ring, scope, signatures) of one Example of sign/anon/sig_test.go (an entry of tests/golden/anon_examples.json),
    re-signed with this restatement in the Example's order of draws"""
    name = e["name"]
    rand = pc.Xof(b"")                                  # blake2xb.New(nil)
    msg, scope = e["message"].encode(), (e["scope"].encode() if e["scope"] is not None else None)
    if name == "ExampleSign_one":
        x = pc.pick_int(rand)
        ring = [mul(x, None)]
        return msg, ring, scope, [sign(msg, ring, scope, 0, x, rand)]
    ring = [point_pick(rand) for _ in range(e["n"])]
    xs = [pc.pick_int(rand) for _ in e["mine"]]
    for mine, x in zip(e["mine"], xs):
        ring[mine] = mul(x, None)
    if name == "ExampleSign_anonSet":
        return msg, ring, scope, [sign(msg, ring, scope, e["mine"][0], xs[0], rand)]
    order = [(e["mine"][0], xs[0])] * 2 + [(e["mine"][1], xs[1])] * 2
    return msg, ring, scope, [sign(msg, ring, scope, mine, x, rand) for mine, x in order]


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def keypair(rng: random.Random):
    x = rng.randrange(1, L)
    return x, mul(x, None)


def ring_with_signer(rng: random.Random, n: int, mine: int, x: int, torsion: bool = False):
    """(ring, clean): n random keys a B + b T8 (b = 0 unless torsion) with the signer's x B at position mine, and the same
    ring without the torsion parts"""
    ab = [(rng.randrange(1, L), rng.randrange(1, 8) if torsion else 0) for _ in range(n)]
    ring, clean = [mc.point(a, b) for a, b in ab], [mc.point(a, 0) for a, _ in ab]
    ring[mine] = clean[mine] = mul(x, None)
    return ring, clean


def signed_batch(label: str, n: int, m: int, scope: bytes | None, msg_lens=(12,)):
    """(ring, msgs, sigs, signers) of m signatures by random members of one random ring of n keys"""
    rng = random.Random(label)
    keys = [keypair(rng) for _ in range(n)]
    ring = [k[1] for k in keys]
    rand = pc.Xof(label.encode())
    msgs, sigs, who = [], [], []
    for j in range(m):
        mine = rng.randrange(n)
        msg = bytes(rng.getrandbits(8) for _ in range(msg_lens[j % len(msg_lens)]))
        msgs.append(msg)
        sigs.append(sign(msg, ring, scope, mine, keys[mine][0], rand))
        who.append(mine)
    return ring, msgs, sigs, who


def flip(b: bytes, byte: int, bit: int = 0) -> bytes:
    out = bytearray(b)
    out[byte] ^= 1 << bit
    return bytes(out)


def with_scalar(sig: bytes, slot: int, v: int) -> bytes:
    """the signature with its 32-byte item `slot` (0 = C0, 1 + i = S_i) replaced by the raw integer v"""
    return sig[:32 * slot] + v.to_bytes(32, "little") + sig[32 * slot + 32:]


def high_variants(s: int):
    """s + k l (k = 1..15, below 2^256) with their top digits: some keep the value (e63 <= 8), some drop it"""
    return [(s + k * L, mc.top_digit(s + k * L)) for k in range(1, 16) if s + k * L < 1 << 256]
