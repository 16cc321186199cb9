"""GPU: Neff shuffle verification on edwards25519 (b2k_ed25519_shuffle_verify, b2k_ed25519_shuffle_sequence_verifiable) against
the restatement in tests/shuffle_cases.py.

Honest proofs are built by the restated prover with the engine's b2k_ed25519_mul_batch for its multiplications (the prover's
scalars are canonical); the expected status of every small case is the restated verifier's, in pure Python."""
import random

import pytest

import pvss_cases as pc
import shuffle_cases as sc

pytestmark = pytest.mark.gpu
L = sc.L
OK, SIMPLE, PAIR, POINT = sc.OK, sc.SIMPLE, sc.PAIR, sc.POINT


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def engine_mul(eng):
    def mul(scalars, points):
        if not scalars:
            return []
        pts = b"".join(p if p is not None else sc.G for p in points)
        out = eng.ed25519_mul_batch(b"".join(sc.le(k) for k in scalars), pts)
        return [out[i:i + 32] for i in range(0, len(out), 32)]
    return mul


def make(eng, k: int, seed: int, g=None, h="random", proto=b"PairShuffle", torsion=False):
    """an honest shuffle of k pairs; g / h None = the base point"""
    rng = random.Random(seed)
    if h == "random":
        h = pc.random_point(rng)
    ops = sc.BytesOps(engine_mul(eng))
    X, Y = sc.elgamal_pairs(k, rng, h, ops, torsion)
    Xb, Yb, prf = sc.shuffle(g, h, X, Y, proto, "gpu shuffle %d" % seed, ops)
    return dict(g=g, h=h, X=X, Y=Y, Xbar=Xb, Ybar=Yb, proof=prf, proto=proto)


def run(eng, cases, k, proto=b"PairShuffle", gh_given=None):
    """the device status of every case (one call); g / h passed when any case has one"""
    given = gh_given if gh_given is not None else any(c["g"] is not None for c in cases)
    cat = lambda key: b"".join(b"".join(c[key]) for c in cases)
    g = b"".join(c["g"] or sc.G for c in cases) if given else None
    h = b"".join(c["h"] or sc.G for c in cases) if any(c["h"] is not None for c in cases) else None
    return list(eng.ed25519_shuffle_verify(k, cat("X"), cat("Y"), cat("Xbar"), cat("Ybar"), b"".join(c["proof"] for c in cases),
                                           proto, g, h))


def oracle(c, proto=b"PairShuffle"):
    return sc.hash_verify(proto, c["g"], c["h"], c["X"], c["Y"], c["Xbar"], c["Ybar"], c["proof"])


def test_honest_base_point_and_given_g(eng):
    k = 3
    c0 = make(eng, k, 1)
    c1 = make(eng, k, 2, g=pc.random_point(random.Random(22)))
    c2 = make(eng, k, 5, h=None)
    assert run(eng, [c0], k) == [OK] == [oracle(c0)]
    assert run(eng, [c2], k) == [OK] == [oracle(c2)]
    assert run(eng, [c0, c1, c2], k) == [OK, OK, OK] == [oracle(c0), oracle(c1), oracle(c2)]
    assert run(eng, [c0], k, proto=b"other") == [oracle(c0, b"other")] == [SIMPLE]


def corruptions(c, k):
    """(name, case) pairs: an undecodable point in each message and input vector, and changed proof values"""
    bad = pc.undecodable()
    out = []
    for name in ("Gamma", "A", "C", "U", "W", "Lambda1", "Lambda2", "D", "X", "Y", "Theta"):
        out.append(("bad " + name, dict(c, proof=sc.with_item(c["proof"], sc.item(k, name, k - 1 if name in "ACUWDXY" else 0), bad))))
    for key in ("X", "Y", "Xbar", "Ybar"):
        out.append(("bad input " + key, dict(c, **{key: c[key][:1] + [bad] + c[key][2:]})))
    out.append(("bad h", dict(c, h=bad)))
    out.append(("swapped Xbar", dict(c, Xbar=[c["Xbar"][1], c["Xbar"][0]] + c["Xbar"][2:])))
    out.append(("torsion on Xbar", dict(c, Xbar=c["Xbar"][:-1] + [sc.add(c["Xbar"][-1], pc.T8)])))
    bump = lambda b, d=1: sc.le(int.from_bytes(b, "little") + d)
    its = sc.items(c["proof"])
    for name, i in (("Zalpha", 0), ("Zalpha", 2 * k - 2), ("Zsigma", 0), ("Zsigma", k - 1), ("Ztau", 0)):
        j = sc.item(k, name, i)
        out.append(("changed %s[%d]" % (name, i), dict(c, proof=sc.with_item(c["proof"], j, bump(its[j])))))
        out.append(("%s[%d] + l" % (name, i), dict(c, proof=sc.with_item(c["proof"], j, bump(its[j], L)))))
    for name, i in (("Theta", 0), ("Theta", 2 * k - 1), ("Lambda1", 0), ("Lambda2", 0), ("D", 0), ("W", 1)):
        j = sc.item(k, name, i)
        out.append(("changed %s[%d]" % (name, i), dict(c, proof=sc.with_item(c["proof"], j, sc.add(its[j], sc.G)))))
        out.append(("torsion on %s[%d]" % (name, i), dict(c, proof=sc.with_item(c["proof"], j, sc.add(its[j], pc.T8)))))
    # e63-rule scalars: Zsigma_0 + 2^255 ... (top nibble >= 9 selects nothing in the reference)
    for name in ("Zsigma", "Ztau", "Zalpha"):
        j = sc.item(k, name, 0)
        v = int.from_bytes(its[j], "little")
        for hi in (0x9, 0xF):
            out.append(("%s e63=%x" % (name, hi), dict(c, proof=sc.with_item(c["proof"], j, sc.le((v & ((1 << 252) - 1)) | (hi << 252))))))
    # a proof point replaced by a non-canonical encoding of the same point (the identity, y = 1 + p), against the canonical one
    for name in ("D", "Theta", "Lambda1"):
        j = sc.item(k, name, 0)
        out.append(("identity %s" % name, dict(c, proof=sc.with_item(c["proof"], j, pc.IDENTITY))))
        out.append(("noncanonical identity %s" % name, dict(c, proof=sc.with_item(c["proof"], j, pc.noncanonical_identity()))))
    return out


def test_every_corruption_matches_the_oracle(eng):
    k = 3
    c = make(eng, k, 3)
    cases = corruptions(c, k)
    got = run(eng, [cs for _, cs in cases], k)
    want = [oracle(cs) for _, cs in cases]
    assert got == want, [(n, g, w) for (n, _), g, w in zip(cases, got, want) if g != w]
    assert set(got) == {OK, SIMPLE, PAIR, POINT}
    named = dict(zip([n for n, _ in cases], got))
    assert named["bad Gamma"] == named["bad input Ybar"] == named["bad Theta"] == POINT
    assert named["changed Zalpha[0]"] == SIMPLE and named["swapped Xbar"] == PAIR
    assert named["Zalpha[0] + l"] == OK         # Zalpha is not hashed, and its bases have prime order


def test_torsion_inputs_and_noncanonical_inputs(eng):
    k = 4
    c = make(eng, k, 4, torsion=True)
    t = dict(c, X=[sc.add(c["X"][0], pc.T8)] + c["X"][1:])
    n = dict(c, Ybar=c["Ybar"][:-1] + [sc.add(c["Ybar"][-1], pc.T8)])
    cases = [c, t, n]
    assert run(eng, cases, k) == [oracle(x) for x in cases]


def test_batch_of_64_mixed(eng):
    k = 2
    rng = random.Random(64)
    base = [make(eng, k, 100 + i) for i in range(4)]
    cases = []
    for i in range(64):
        c = base[i % 4]
        kind = rng.randrange(6)
        if kind == 1:
            c = dict(c, proof=sc.with_item(c["proof"], sc.item(k, "Theta", rng.randrange(2 * k)), sc.G))
        elif kind == 2:
            c = dict(c, Xbar=c["Xbar"][::-1])
        elif kind == 3:
            c = dict(c, proof=sc.with_item(c["proof"], rng.randrange(4 * k + 3), pc.undecodable()))
        elif kind == 4:
            j = sc.item(k, "Zsigma", rng.randrange(k))
            c = dict(c, proof=sc.with_item(c["proof"], j, sc.le(int.from_bytes(sc.items(c["proof"])[j], "little") + L)))
        cases.append(c)
    got = run(eng, cases, k)
    assert got == [oracle(c) for c in cases]
    assert set(got) == {OK, SIMPLE, PAIR, POINT}


def test_protocol_names(eng):
    k = 2
    for proto in (b"", b"SequencesShuffle", bytes(range(64)), bytes(range(65)), bytes(200)):
        c = make(eng, k, 7, proto=proto)
        assert run(eng, [c], k, proto=proto) == [OK]
        assert run(eng, [c], k, proto=proto + b"x") == [oracle(c, proto + b"x")]


@pytest.mark.parametrize("nq,k", [(6, 5), (3, 3)])
def test_sequence_round_trip(eng, nq, k):
    rng = random.Random(nq * 10 + k)
    mul = engine_mul(eng)
    h = pc.random_point(rng)
    X, Y = [], []
    for _ in range(nq):
        a, b = sc.elgamal_pairs(k, rng, h, sc.BytesOps(mul))
        X.append(a)
        Y.append(b)
    e = [rng.randrange(L) for _ in range(nq)]
    Xb, Yb, prf = sc.sequences_shuffle(None, h, X, Y, e, b"SequencesShuffle", "seq %d" % nq, mul)
    flat = lambda M: b"".join(b"".join(r) for r in M)
    got = eng.ed25519_shuffle_sequence_verifiable(nq, flat(X), flat(Y), flat(Xb), flat(Yb), b"".join(sc.le(v) for v in e))
    want = sc.get_sequence_verifiable(X, Y, Xb, Yb, e)
    assert got == tuple(b"".join(w) for w in want)
    xup, yup, xdown, ydown = [[o[i:i + 32] for i in range(0, len(o), 32)] for o in got]
    c = dict(g=None, h=h, X=xup, Y=yup, Xbar=xdown, Ybar=ydown, proof=prf)
    assert run(eng, [c], k, b"SequencesShuffle") == [OK] == [oracle(c, b"SequencesShuffle")]
    # the reference's negative test: X[0][0] replaced
    X2 = [[pc.random_point(rng)] + X[0][1:]] + X[1:]
    got2 = eng.ed25519_shuffle_sequence_verifiable(nq, flat(X2), flat(Y), flat(Xb), flat(Yb), b"".join(sc.le(v) for v in e))
    xup2 = [got2[0][i:i + 32] for i in range(0, 32 * k, 32)]
    c2 = dict(c, X=xup2)
    assert run(eng, [c2], k, b"SequencesShuffle") == [oracle(c2, b"SequencesShuffle")] == [PAIR]


def test_sequence_raw_scalars_and_bad_point(eng):
    from kyber_b200.capi import B2KError
    rng = random.Random(9)
    nq, k = 3, 2
    X = [[pc.random_point(rng, torsion=True) for _ in range(k)] for _ in range(nq)]
    e = [(0x9 << 252) | rng.getrandbits(250), (1 << 256) - 1, L + 5]
    flat = lambda M: b"".join(b"".join(r) for r in M)
    got = eng.ed25519_shuffle_sequence_verifiable(nq, flat(X), flat(X), flat(X), flat(X), b"".join(sc.le(v) for v in e))
    want = sc.get_sequence_verifiable(X, X, X, X, e)
    assert got == tuple(b"".join(w) for w in want)
    X[1][1] = pc.undecodable()
    with pytest.raises(B2KError):
        eng.ed25519_shuffle_sequence_verifiable(nq, flat(X), flat(X), flat(X), flat(X), b"".join(sc.le(v) for v in e))


def test_argument_errors(eng):
    from kyber_b200.capi import B2KError
    c = make(eng, 2, 11)
    with pytest.raises(B2KError):               # k < 2
        eng.ed25519_shuffle_verify(1, c["X"][0], c["Y"][0], c["Xbar"][0], c["Ybar"][0], bytes(32 * 15))
    assert run(eng, [c], 2) == [OK]             # the context still works


def dlog_ops(eng):
    """the prover on discrete logs, encoded by b2k_ed25519_mul_batch on the base point"""
    return sc.DlogOps(lambda ks: engine_mul(eng)(ks, [None] * len(ks)))


def honest_dlog(eng, k: int, seed: str):
    """an honest shuffle of k pairs built on discrete logs (no torsion): the case dict with encodings"""
    ops = dlog_ops(eng)
    rng = random.Random(seed)
    hd = rng.randrange(1, L)
    X, Y = sc.elgamal_pairs(k, rng, hd, ops)
    Xb, Yb, prf = sc.shuffle(None, hd, X, Y, b"PairShuffle", seed, ops)
    enc = ops.enc(X + Y + Xb + Yb + [hd])
    return dict(g=None, h=enc[-1], X=enc[:k], Y=enc[k:2 * k], Xbar=enc[2 * k:3 * k], Ybar=enc[3 * k:4 * k], proof=prf)


def test_dlog_prover_matches_the_bytes_prover(eng):
    k = 3
    a = honest_dlog(eng, k, "same")
    assert run(eng, [a], k) == [OK] == [oracle(a)]


@pytest.mark.parametrize("m,k", [(1, 1 << 16), (256, 256)])
def test_scale(eng, m, k):
    """honest shuffles at scale, and one corrupted copy each way"""
    nbase = min(m, 2)
    base = [honest_dlog(eng, k, "scale %d %d %d" % (m, k, i)) for i in range(nbase)]
    cases = [base[i % nbase] for i in range(m)]
    assert run(eng, cases, k) == [OK] * m
    c = base[0]
    its = sc.items(c["proof"])
    j = sc.item(k, "Theta", k + 7)
    bad_theta = dict(c, proof=sc.with_item(c["proof"], j, sc.add(its[j], sc.G)))
    swapped = dict(c, Xbar=[c["Xbar"][1], c["Xbar"][0]] + c["Xbar"][2:])
    torsion_x = dict(c, X=c["X"][:-1] + [sc.add(c["X"][-1], pc.T8)])
    got = run(eng, [bad_theta, swapped, torsion_x, c], k)
    assert got[:2] == [SIMPLE, PAIR] and got[3] == OK
    # Phi1 changes by -Zrho_{k-1} T8: the identity exactly when 8 divides Zrho_{k-1}
    assert got[2] in (OK, PAIR)
