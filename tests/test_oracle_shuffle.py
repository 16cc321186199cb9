"""CPU: the restatement of Neff's shuffle and its Fiat-Shamir transcript in tests/shuffle_cases.py -- honest proofs at the sizes
of the reference's shuffle_test.go, its two negative tests, the proof layout, protocol names, and a byte-level replay of the
transcript across rejected Pick draws."""
import random

import pytest

from oracle import ed25519 as ed
import pvss_cases as pc
import shuffle_cases as sc

L = sc.L


def pairs(k, seed, h):
    return sc.elgamal_pairs(k, random.Random(seed), h)


@pytest.mark.parametrize("k", [2, 3, 5])
def test_honest_pair_shuffle_verifies_and_swapped_outputs_do_not(k):
    h = pc.random_point(random.Random(k))
    X, Y = pairs(k, 10 + k, h)
    Xb, Yb, prf = sc.shuffle(None, h, X, Y, b"PairShuffle", "oracle %d" % k)
    assert len(prf) == sc.proof_len(k) == 32 * (12 * k + 3)
    assert sc.hash_verify(b"PairShuffle", None, h, X, Y, Xb, Yb, prf) == sc.OK
    sw = [Xb[1], Xb[0]] + Xb[2:]                          # shuffle_test.go: Xbar[0] and Xbar[1] swapped
    assert sc.hash_verify(b"PairShuffle", None, h, X, Y, sw, Yb, prf) == sc.PAIR


def test_given_g_and_h():
    rng = random.Random(3)
    g, h = pc.random_point(rng), pc.random_point(rng)
    X, Y = pairs(3, 4, h)
    Xb, Yb, prf = sc.shuffle(g, h, X, Y, b"PairShuffle", "given g")
    assert sc.hash_verify(b"PairShuffle", g, h, X, Y, Xb, Yb, prf) == sc.OK
    assert sc.hash_verify(b"PairShuffle", None, h, X, Y, Xb, Yb, prf) != sc.OK


def test_sequences_nq6_k5_and_the_replaced_input():
    nq, k = 6, 5
    rng = random.Random(65)
    h = pc.random_point(rng)
    X, Y = [], []
    for _ in range(nq):
        a, b = sc.elgamal_pairs(k, rng, h)
        X.append(a)
        Y.append(b)
    e = [rng.randrange(L) for _ in range(nq)]
    Xb, Yb, prf = sc.sequences_shuffle(None, h, X, Y, e, b"SequencesShuffle", "seq")
    xu, yu, xd, yd = sc.get_sequence_verifiable(X, Y, Xb, Yb, e)
    assert sc.hash_verify(b"SequencesShuffle", None, h, xu, yu, xd, yd, prf) == sc.OK
    X2 = [[pc.random_point(rng)] + X[0][1:]] + X[1:]      # shuffle_test.go: X[0][0] replaced
    xu2, yu2, xd2, yd2 = sc.get_sequence_verifiable(X2, Y, Xb, Yb, e)
    assert sc.hash_verify(b"SequencesShuffle", None, h, xu2, yu2, xd2, yd2, prf) == sc.PAIR


@pytest.mark.parametrize("proto", [b"PairShuffle", b"SequencesShuffle", b"", bytes(range(64)), bytes(range(65)),
                                   bytes(range(100, 230))])
def test_protocol_names(proto):
    h = pc.random_point(random.Random(5))
    X, Y = pairs(2, 6, h)
    Xb, Yb, prf = sc.shuffle(None, h, X, Y, proto, "proto")
    assert sc.hash_verify(proto, None, h, X, Y, Xb, Yb, prf) == sc.OK
    assert sc.hash_verify(proto + b"\x00", None, h, X, Y, Xb, Yb, prf) == sc.SIMPLE


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 128, 129, 500, 4096])
def test_fast_xof_root_is_the_explicit_one(n):
    rng = random.Random(n)
    seed = bytes(rng.getrandbits(8) for _ in range(min(n, 200)))
    extra = bytes(rng.getrandbits(8) for _ in range(n))
    a, b = sc.FastXof(seed, extra), pc.Xof(seed, extra)
    assert a.root == b.root
    assert a.read(300) == b.read(300)


def _replay(proto: bytes, proof: bytes, k: int):
    """proof.HashVerify's transcript for a shuffle, byte by byte on the explicit XOF: (zrho, zlambda, t, c, draws before each
    Reseed that were rejected)"""
    x = pc.Xof(proto)
    rejected = []

    def picks(n):
        out, rej = [], 0
        while len(out) < n:
            b = bytearray(x.read(32))
            b[0] &= 0x1F
            v = int.from_bytes(b, "big")
            if v < L:
                out.append(v)
            else:
                rej += 1
        rejected.append(rej)
        return out

    def reseed(msg):
        nonlocal x
        key = x.read(128)
        x = pc.Xof(key, msg)                              # New(key): key[:64] is the BLAKE2b key, key[64:] the first message

    o = [0, 32 * (4 * k + 3), 32 * (5 * k + 3), 32 * (8 * k + 4), 32 * (10 * k + 4)]
    reseed(proof[o[0]:o[1]]); zrho = picks(k)
    reseed(proof[o[1]:o[2]]); zl, = picks(1)
    reseed(proof[o[2]:o[3]]); t, = picks(1)
    reseed(proof[o[3]:o[4]]); c, = picks(1)
    return zrho, zl, t, c, rejected


def _transcript(proto: bytes, proof: bytes, k: int):
    v = sc.HashVerifier(proto, proof)
    v.get_points(4 * k + 3); zrho = v.pub_rand(k)
    v.get_points(k); zl, = v.pub_rand(1)
    v.get_scalars(k + 1); v.get_points(2 * k); t, = v.pub_rand(1)
    v.get_points(2 * k); c, = v.pub_rand(1)
    return zrho, zl, t, c


def test_transcript_across_rejected_draws_matches_a_byte_level_replay():
    k = 2
    h = pc.random_point(random.Random(8))
    X, Y = pairs(k, 9, h)
    seen = set()
    for i in range(40):
        proto = b"replay %d" % i
        Xb, Yb, prf = sc.shuffle(None, h, X, Y, proto, "replay %d" % i)
        zrho, zl, t, c, rej = _replay(proto, prf, k)
        assert _transcript(proto, prf, k) == (zrho, zl, t, c)
        assert sc.hash_verify(proto, None, h, X, Y, Xb, Yb, prf) == sc.OK
        if rej[0] or rej[1] or rej[2]:
            seen.add(tuple(bool(r) for r in rej[:3]))
        if (True, True, True) in seen or len(seen) >= 3:
            break
    assert any(s[1] for s in seen)                        # the Zlambda pick rejected a draw before the next Reseed


def test_undecodable_and_noncanonical_points():
    k = 2
    h = pc.random_point(random.Random(11))
    X, Y = pairs(k, 12, h)
    Xb, Yb, prf = sc.shuffle(None, h, X, Y, b"PairShuffle", "bad")
    bad = pc.undecodable()
    for name in ("Gamma", "A", "U", "D", "X", "Theta"):
        assert sc.hash_verify(b"PairShuffle", None, h, X, Y, Xb, Yb, sc.with_item(prf, sc.item(k, name), bad)) == sc.POINT
    assert sc.hash_verify(b"PairShuffle", None, h, [bad] + X[1:], Y, Xb, Yb, prf) == sc.POINT
    # the hash covers the raw bytes: the non-canonical identity and the canonical one are the same point, different transcripts
    j = sc.item(k, "D")
    a = sc.hash_verify(b"PairShuffle", None, h, X, Y, Xb, Yb, sc.with_item(prf, j, pc.IDENTITY))
    b = sc.hash_verify(b"PairShuffle", None, h, X, Y, Xb, Yb, sc.with_item(prf, j, pc.noncanonical_identity()))
    assert ed.decode(pc.IDENTITY) == ed.decode(pc.noncanonical_identity())
    assert a != sc.OK and b != sc.OK
