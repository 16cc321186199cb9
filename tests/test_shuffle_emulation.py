"""CPU: the shuffle verifier's device bodies (kyber_b200/csrc/shuffle.cuh) and host transcript (shuffle_transcript.h) compiled
for the host and checked against the restatement in tests/shuffle_cases.py -- thver with raw and e63-rule scalars, the Phi term
and the single multiplication on torsion points, the sequence term, the threaded Pick squeeze, the transcript, and
whole batches through every kernel body in order."""
import ctypes
import os
import random
import subprocess

import pytest

import ed25519_msm_cases as mc
import pvss_cases as pc
import shuffle_cases as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_shuffle.cpp")
L = sc.L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_shuffle") / "libemul_shuffle.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-pthread", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC,
                    "-o", so], check=True)
    lib = ctypes.CDLL(so)
    u32, sz, cp = ctypes.c_uint32, ctypes.c_size_t, ctypes.c_char_p
    lib.emul_transcript.argtypes = [sz, cp, cp, u32, cp, cp, cp, ctypes.c_uint]
    lib.emul_pick_many.argtypes = [cp, u32, sz, cp, ctypes.c_uint]
    lib.emul_pick_many.restype = ctypes.c_uint64
    lib.emul_thver.argtypes = [cp] * 5
    lib.emul_phi_term.argtypes = [cp] * 6
    lib.emul_sequence_term.argtypes = [u32, cp, cp, cp]
    lib.emul_shuffle_verify.argtypes = [sz, sz] + [cp] * 7 + [cp, u32, cp]
    return lib


def scalars(rng):
    return mc.crafted_high_scalars(rng) + [0, 1, L - 1, L, L + 1, (1 << 255) - 1, (1 << 256) - 1] + \
        [rng.getrandbits(256) for _ in range(4)]


def test_thver_raw_a_and_negated_b(lib):
    rng = random.Random(2)
    ss = scalars(rng)
    for j, a in enumerate(ss):
        b = ss[(3 * j + 1) % len(ss)]
        A, B = pc.random_point(rng, torsion=True), pc.random_point(rng, torsion=True)
        T = sc.add(*sc.py_mul([a, (-b) % L], [A, B]))
        assert lib.emul_thver(A, B, T, sc.le(a), sc.le(b)) == 1 == sc.thver(A, B, T, a, b)
        T2 = sc.add(T, pc.T8)
        assert lib.emul_thver(A, B, T2, sc.le(a), sc.le(b)) == 0 == sc.thver(A, B, T2, a, b)
        # negating the POINT B instead differs when B has a torsion part and b is not reduced
        T3 = sc.add(*sc.py_mul([a, b], [A, sc.neg(B)]))
        assert lib.emul_thver(A, B, T3, sc.le(a), sc.le(b)) == int(sc.thver(A, B, T3, a, b))


def test_phi_term_and_single_multiplication(lib):
    rng = random.Random(3)
    ss = scalars(rng)
    for j, zs in enumerate(ss):
        zr = ss[(5 * j + 2) % len(ss)]
        P, Q = pc.random_point(rng, torsion=True), pc.random_point(rng, torsion=True)
        out, om = ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
        assert lib.emul_phi_term(sc.le(zs), P, sc.le(zr), Q, out, om) == 1
        ps, pr = sc.py_mul([zs, zr], [P, Q])
        assert out.raw == sc.sub(ps, pr), (hex(zs), hex(zr))          # Sub negates the point
        assert om.raw == ps


def test_sequence_term(lib):
    rng = random.Random(4)
    for nq in (1, 2, 3, 6):
        pts = [pc.random_point(rng, torsion=True) for _ in range(nq)]
        e = [rng.choice(scalars(rng)) for _ in range(nq)]
        out = ctypes.create_string_buffer(32)
        assert lib.emul_sequence_term(nq, b"".join(pts), b"".join(sc.le(v) for v in e), out) == 1
        assert out.raw == sc.total(sc.py_mul(e, pts))
    assert lib.emul_sequence_term(1, pc.undecodable(), bytes(32), out) == 0


@pytest.mark.parametrize("n,nt", [(5, 1), (1500, 1), (1500, 4), (3000, 7)])
def test_threaded_pick_squeeze(lib, n, nt):
    seed = b"squeeze %d" % n
    out = ctypes.create_string_buffer(32 * n)
    pos = lib.emul_pick_many(seed, len(seed), n, out, nt)
    x = pc.Xof(seed)
    want = b"".join(pc.pick(x) for _ in range(n))
    assert out.raw == want
    assert pos * 32 == x.block * 64 - len(x.buf)                # the stream position after the last accepted draw


def _transcript(proto, proof, k):
    """the restated verifier's transcript over the proof bytes (points are not decoded: the transcript reads bytes only)"""
    v = sc.HashVerifier(proto, proof)
    v._take(4 * k + 3); zrho = v.pub_rand(k)
    v._take(k); v.pub_rand(1)
    v._take(3 * k + 1); t, = v.pub_rand(1)
    v._take(2 * k); c, = v.pub_rand(1)
    return b"".join(sc.le(z) for z in zrho), sc.le(t), sc.le(c)


@pytest.mark.parametrize("proto", [b"", b"PairShuffle", bytes(range(64)), bytes(range(65)), bytes(300)])
def test_host_transcript(lib, proto):
    k = 3
    h = pc.random_point(random.Random(5))
    X, Y = sc.elgamal_pairs(k, random.Random(6), h)
    _, _, prf = sc.shuffle(None, h, X, Y, proto, "emul transcript")
    zr, t, c = ctypes.create_string_buffer(32 * k), ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
    lib.emul_transcript(k, prf, proto, len(proto), zr, t, c, 1)
    assert (zr.raw, t.raw, c.raw) == _transcript(proto, prf, k)


def test_host_transcript_threaded_at_k_2000(lib):
    k = 2000
    proof = bytes(random.Random(7).getrandbits(8) for _ in range(sc.proof_len(k)))   # the transcript reads bytes only
    outs = []
    for nt in (1, 6):
        zr, t, c = ctypes.create_string_buffer(32 * k), ctypes.create_string_buffer(32), ctypes.create_string_buffer(32)
        lib.emul_transcript(k, proof, b"PairShuffle", 11, zr, t, c, nt)
        outs.append((zr.raw, t.raw, c.raw))
    assert outs[0] == outs[1] == _transcript(b"PairShuffle", proof, k)


def _verify(lib, cases, k, proto=b"PairShuffle"):
    m = len(cases)
    cat = lambda key: b"".join(b"".join(c[key]) for c in cases)
    gs = None if all(c["g"] is None for c in cases) else b"".join(c["g"] or sc.G for c in cases)
    hs = None if all(c["h"] is None for c in cases) else b"".join(c["h"] or sc.G for c in cases)
    st = ctypes.create_string_buffer(m)
    lib.emul_shuffle_verify(m, k, gs, hs, cat("X"), cat("Y"), cat("Xbar"), cat("Ybar"), b"".join(c["proof"] for c in cases),
                            proto, len(proto), st)
    return list(st.raw)


def test_whole_batch_against_the_restatement(lib):
    k = 2
    rng = random.Random(8)
    h = pc.random_point(rng)
    X, Y = sc.elgamal_pairs(k, rng, h)
    Xb, Yb, prf = sc.shuffle(None, h, X, Y, b"PairShuffle", "emul batch")
    c = dict(g=None, h=h, X=X, Y=Y, Xbar=Xb, Ybar=Yb, proof=prf)
    its = sc.items(prf)
    e63 = lambda v: sc.le((v & ((1 << 252) - 1)) | (0xB << 252))
    cases = [
        c,
        dict(c, Xbar=[Xb[1], Xb[0]]),
        dict(c, proof=sc.with_item(prf, sc.item(k, "Theta", 1), sc.add(its[sc.item(k, "Theta", 1)], pc.T8))),
        dict(c, proof=sc.with_item(prf, sc.item(k, "W", 0), pc.undecodable())),
        dict(c, proof=sc.with_item(prf, sc.item(k, "Zalpha", 0), e63(int.from_bytes(its[sc.item(k, "Zalpha", 0)], "little")))),
        dict(c, proof=sc.with_item(prf, sc.item(k, "Zalpha", 1), sc.le(int.from_bytes(its[sc.item(k, "Zalpha", 1)], "little") + L))),
        dict(c, X=[sc.add(X[0], pc.T8), X[1]]),
        dict(c, Ybar=[Yb[0], sc.add(Yb[1], mc.point(0, 4))]),
        dict(c, proof=sc.with_item(prf, sc.item(k, "D", 1), pc.noncanonical_identity())),
    ]
    got = _verify(lib, cases, k)
    want = [sc.hash_verify(b"PairShuffle", x["g"], x["h"], x["X"], x["Y"], x["Xbar"], x["Ybar"], x["proof"]) for x in cases]
    assert got == want
    assert got[0] == sc.OK and got[1] == sc.PAIR and got[3] == sc.POINT and got[5] == sc.OK


def test_whole_batch_with_given_g_and_more_than_one_chunk(lib):
    k = 130                                                  # two blocks of 128 in the Phi sums
    rng = random.Random(9)
    g = pc.random_point(rng)
    hd = rng.randrange(1, L)
    ops = sc.DlogOps(lambda ks: sc.py_mul(ks, [g] * len(ks)))   # dlogs to g
    X, Y = sc.elgamal_pairs(k, rng, hd, ops)
    Xb, Yb, prf = sc.shuffle(1, hd, X, Y, b"PairShuffle", "emul chunks", ops)
    enc = ops.enc(X + Y + Xb + Yb + [hd])
    c = dict(g=g, h=enc[-1], X=enc[:k], Y=enc[k:2 * k], Xbar=enc[2 * k:3 * k], Ybar=enc[3 * k:4 * k], proof=prf)
    bad = dict(c, Ybar=c["Ybar"][:129] + [c["Ybar"][0]])
    assert _verify(lib, [c, bad], k) == [sc.OK, sc.PAIR]
