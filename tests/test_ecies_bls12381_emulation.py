"""CPU: ECIES on BLS12-381's device bodies (kyber_b200/csrc/ecies_bls.cuh) compiled for the host and checked against the
restatement in tests/ecies_bls12381_oracle.py, for keys on G1 and on G2: the constant-time multiplication on every exceptional
case of the complete addition (the identity, P = Q, P = -Q, through scalars 0, 1, 2, r - 1, r - 2 and points at infinity and
+-small multiples of the generator), the constant-time compression, whole encryptions and decryptions, and the operation counts
of every constant-time helper, which must not depend on the key, r, R, dh, the tag's outcome or the message bytes."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import bls12381 as bls
import ecies_bls12381_oracle as eb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_ecies_bls.cpp")
R = bls.R
NCOUNT = 7
SELECT, WINDOW, SBOX, GHASH, ADD, DBL, INV = range(NCOUNT)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_ecies_bls") / "libemul_ecies_bls.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    i, u32, sz, cp = ctypes.c_int, ctypes.c_uint32, ctypes.c_size_t, ctypes.c_char_p
    lib.emul_counts.argtypes = [ctypes.c_void_p, i]
    lib.emul_mul.argtypes = [i, cp, cp, cp]
    lib.emul_compress.argtypes = [i, cp, cp, cp]
    lib.emul_decrypt.argtypes = [i, cp, sz, u32, cp, cp, cp]
    lib.emul_encrypt.argtypes = [i, sz, cp, cp, u32, cp, cp, cp]
    return lib


def counts(lib):
    c = (ctypes.c_uint64 * NCOUNT)()
    lib.emul_counts(c, 1)
    return tuple(c)


def decrypt(lib, group, priv, cts, clen):
    n = len(cts)
    msg, st = ctypes.create_string_buffer(max(n * (clen - 16), 1)), ctypes.create_string_buffer(n)
    lib.emul_decrypt(group - 1, priv, n, clen, b"".join(cts), msg, st)
    w = clen - 16
    return [(st.raw[i], msg.raw[w * i:w * i + w]) for i in range(n)]


def encrypt(lib, group, pubs, rs, msgs):
    n, ln, pl = len(msgs), len(msgs[0]), eb.POINT_LEN[group]
    out, st = ctypes.create_string_buffer(n * (pl + ln + 16)), ctypes.create_string_buffer(n)
    lib.emul_encrypt(group - 1, n, b"".join(pubs), b"".join(rs), ln, b"".join(msgs) or b"\x00", out, st)
    w = pl + ln + 16
    return [(st.raw[i], out.raw[w * i:w * i + w]) for i in range(n)]


def sb(k: int) -> bytes:
    return k.to_bytes(32, "big")


def scalars(rng):
    return [0, 1, 2, R - 1, R - 2, 1 << 254, rng.randrange(R), rng.randrange(R)]


def points(group, rng):
    """infinity, G, 2G, 3G, -G, -2G, a random point and its negative"""
    neg = bls.g1_neg if group == 1 else bls.g2_neg
    rnd = eb.mul(group, rng.randrange(1, R))
    return [None, eb.mul(group, 1), eb.mul(group, 2), eb.mul(group, 3), neg(eb.mul(group, 1)), neg(eb.mul(group, 2)), rnd, neg(rnd)]


@pytest.mark.parametrize("group", eb.GROUPS)
def test_multiplication_against_the_oracle(lib, group):
    rng = random.Random(10 + group)
    pl = eb.POINT_LEN[group]
    out = ctypes.create_string_buffer(pl)
    for k in scalars(rng):
        assert lib.emul_mul(group - 1, sb(k), None, out) == 0
        assert out.raw == eb.compress(group, eb.mul(group, k)), (group, hex(k))
        for p in points(group, rng):
            assert lib.emul_mul(group - 1, sb(k), eb.compress(group, p), out) == 0
            want = eb.compress(group, eb.mul(group, k, p) if p is not None else None)
            assert out.raw == want, (group, hex(k), p)


def _xy_bytes(group, pt) -> bytes:
    return bls.g1_to_affine_bytes(pt) if group == 1 else bls.g2_to_affine_bytes(pt)


@pytest.mark.parametrize("group", eb.GROUPS)
def test_compression_against_the_oracle(lib, group):
    """the encoding of (X : Y : Z) with Z != 1; compression only reads x and the sign of y, so the G2 cases with y.c1 = 0 (both
    halves of c0) and y.c1 != 0 with c0 in either half need not lie on the curve"""
    rng = random.Random(20 + group)
    pl = eb.POINT_LEN[group]
    pts = points(group, rng)
    if group == 2:
        x = eb.mul(2, 5)[0]
        small, large = 5, bls.P - 5
        pts += [(x, (small, 0)), (x, (large, 0)), (x, (large, small)), (x, (small, large)), (x, (0, 0))]
    else:
        x = eb.mul(1, 5)[0]
        pts += [(x, bls.HALF_P), (x, bls.HALF_P + 1), (x, 0)]
    out = ctypes.create_string_buffer(pl)
    for p in pts:
        for z in (1, 2, rng.randrange(1, bls.P)):
            lib.emul_compress(group - 1, _xy_bytes(group, p), z.to_bytes(48, "big"), out)
            assert out.raw == eb.compress(group, p), (group, p, z)


@pytest.mark.parametrize("group", eb.GROUPS)
def test_decrypt_against_the_oracle(lib, group):
    rng = random.Random(30 + group)
    pl = eb.POINT_LEN[group]
    for priv in (sb(0), sb(1), sb(R - 1), sb(rng.randrange(R))):
        pub = eb.public(group, priv)
        for n in (0, 32, 33):
            msgs = [rng.randbytes(n) for _ in range(3)]
            rs = [sb(rng.randrange(R)), sb(0), sb(R - 1)]
            cts = [eb.encrypt(group, pub, r, m)[1] for r, m in zip(rs, msgs)]
            bad = bytearray(cts[0]); bad[0] &= 0x7f                     # compression flag clear
            tag = bytearray(cts[0]); tag[-1] ^= 0x80
            body = bytearray(cts[2]); body[pl] ^= 0x01
            batch = cts + [bytes(bad), bytes(tag), bytes(body) if n else bytes(tag)]
            got = decrypt(lib, group, priv, batch, n + 16)
            assert got == [eb.decrypt(group, priv, c) for c in batch]
            assert [g for g in got[:3]] == [(eb.OK, m) for m in msgs]
            assert [g[0] for g in got[3:]] == [eb.POINT, eb.AUTH, eb.AUTH]


@pytest.mark.parametrize("group", eb.GROUPS)
def test_encrypt_against_the_oracle(lib, group):
    rng = random.Random(40 + group)
    for n in (0, 32, 1000):
        pubs = [eb.public(group, sb(rng.randrange(R))), eb.compress(group, None), eb.public(group, sb(1))]
        bad = bytearray(pubs[0]); bad[0] |= 0x40                         # infinity flag with a non-zero x
        pubs.append(bytes(bad))
        rs = [sb(rng.randrange(R)), sb(rng.randrange(R)), sb(0), sb(R - 1)]
        msgs = [rng.randbytes(n) for _ in pubs]
        got = encrypt(lib, group, pubs, rs, msgs)
        assert got == [eb.encrypt(group, p, r, m) for p, r, m in zip(pubs, rs, msgs)]
        assert [g[0] for g in got] == [eb.OK] * 3 + [eb.POINT]


@pytest.mark.parametrize("group", eb.GROUPS)
def test_operation_counts_do_not_depend_on_secrets_or_points(lib, group):
    """every key, r, R, dh, tag outcome and message of one length runs the same number of selections, windows, complete
    additions and doublings, Fermat inversions, S-box layers and GHASH blocks"""
    rng = random.Random(50 + group)
    keys = [sb(0), sb(1), sb(rng.randrange(R))]
    inf = eb.compress(group, None)
    Rs = [inf, eb.public(group, sb(rng.randrange(R)))]             # R at infinity (dh at infinity too) and R random
    msgs = [bytes(48), rng.randbytes(48)]
    counts(lib)
    dec, enc = set(), set()
    for k in keys:
        pub = eb.public(group, k)                                   # key 0: the public key, and so dh, at infinity
        for R_ in Rs:
            for m in msgs:
                good = eb.encrypt(group, pub, k, m)[1]              # (r = k: R = pub)
                ct = R_ + good[len(R_):]
                forged = ct[:-1] + bytes([ct[-1] ^ 1])
                for c in (good, ct, forged):
                    decrypt(lib, group, k, [c], 64)
                    dec.add(counts(lib))
            for m in msgs:
                for r in keys:
                    encrypt(lib, group, [pub], [r], [m])
                    enc.add(counts(lib))
    assert len(dec) == 1 and len(enc) == 1, (dec, enc)
    (d,), (e,) = dec, enc
    assert d[SELECT] == 65 and d[WINDOW] == 64 and d[ADD] == 6 + 65 and d[DBL] == 1 + 256 and d[INV] == 1
    assert e[SELECT] == 130 and e[WINDOW] == 128 and e[ADD] == 12 + 130 and e[DBL] == 2 + 512 and e[INV] == 2
    assert d[SBOX] == e[SBOX] == 13 + 14 * 3                             # SubWord x 13, then H with E(J0) and four counter blocks
    assert d[GHASH] == e[GHASH] == 4                                     # 48 bytes: three GHASH blocks and the length block
