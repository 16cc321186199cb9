"""CPU: the ring signature verifier's device bodies (kyber_b200/csrc/anon.cuh) compiled for the host and checked against the
restatement in tests/anon_cases.py -- the H1pre midstate and the Pick from its root across block boundaries, the link base,
the comb against geScalarMult with e63-rule scalars and torsion bases, and whole verifications through every body in order."""
import ctypes
import os
import random
import struct
import subprocess

import pytest

import anon_cases as ac
import ed25519_msm_cases as mc
import pvss_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_anon.cpp")
L = ac.L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_anon") / "libemul_anon.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    u32, sz, cp = ctypes.c_uint32, ctypes.c_size_t, ctypes.c_char_p
    lib.emul_h1.argtypes = [cp, u32, cp, u32, cp, cp, cp, cp]
    lib.emul_link_base.argtypes = [cp, u32, cp]
    lib.emul_comb.argtypes = [cp] * 5
    lib.emul_anon_verify.argtypes = [sz, cp, ctypes.c_int, cp, u32, sz, cp, cp, cp, u32, cp, cp]
    return lib


def test_h1_midstate_across_block_boundaries(lib):
    rng = random.Random(1)
    lens = [0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 193]
    for mlen in lens:
        for slen in [None] + lens:
            msg, scope = rng.randbytes(mlen), (rng.randbytes(slen) if slen is not None else None)
            tag, pg, ph = pc.random_point(rng), pc.random_point(rng), pc.random_point(rng)
            out = ctypes.create_string_buffer(32)
            lib.emul_h1(msg, mlen, scope, len(scope or b""), tag if scope is not None else None, pg, ph, out)
            want = ac.h1(msg, scope, tag if scope is not None else None, pg, ph if scope is not None else None)
            assert int.from_bytes(out.raw, "little") == want, (mlen, slen)


def test_link_base(lib):
    rng = random.Random(2)
    for scope in [b"", b"x", b"My Linkage Scope", rng.randbytes(64), rng.randbytes(65), rng.randbytes(200)] + \
            [rng.randbytes(rng.randrange(40)) for _ in range(6)]:
        out = ctypes.create_string_buffer(32)
        assert lib.emul_link_base(scope, len(scope), out) == 1
        assert out.raw == ac.link_base(scope), scope


def comb_scalars(rng):
    s = [0, 1, L - 1, L, rng.getrandbits(253)] + mc.crafted_high_scalars(rng)
    # e63 of exactly 0, 8, 9, 15 and 16
    by_digit = {}
    while len(by_digit) < 5:
        k = rng.getrandbits(256)
        d = mc.top_digit(k)
        if d in (0, 8, 9, 15, 16) and d not in by_digit:
            by_digit[d] = k
    return s + list(by_digit.values())


def test_comb_against_ge_scalar_mult(lib):
    rng = random.Random(3)
    ss = comb_scalars(rng)
    assert {mc.top_digit(k) for k in ss} >= {0, 8, 9, 15, 16}
    bases = [pc.G, pc.T8, mc.ZERO, pc.random_point(rng), pc.random_point(rng, torsion=True), mc.mixed_point(5)]
    for j, a in enumerate(ss):
        P = bases[j % len(bases)]
        out = ctypes.create_string_buffer(32)
        assert lib.emul_comb(mc.le([a]), P, None, None, out) == 0
        assert out.raw == ac.mul(a, P), (hex(a), P.hex())
        b = ss[(5 * j + 3) % len(ss)]
        Q = bases[(j + 2) % len(bases)]
        assert lib.emul_comb(mc.le([a]), P, mc.le([b]), Q, out) == 0
        assert out.raw == ac.add(ac.mul(a, P), ac.mul(b, Q))
    assert lib.emul_comb(mc.le([1]), pc.undecodable(), None, None, out) == -1


def run(lib, ring, msgs, sigs, scope, chunk=2):
    m, n = len(msgs), len(ring)
    offs, pos = [0], 0
    for x in msgs:
        pos += len(x)
        offs.append(pos)
    st, tags = ctypes.create_string_buffer(m), ctypes.create_string_buffer(32 * m)
    rc = lib.emul_anon_verify(n, b"".join(ring) or None, int(scope is not None), scope, len(scope or b""), m,
                              b"".join(msgs) or b"\0", struct.pack(f"<{m + 1}I", *offs), b"".join(sigs), chunk, st, tags)
    return rc, list(st.raw), [tags.raw[32 * j:32 * j + 32] for j in range(m)]


def expect(ring, msgs, sigs, scope):
    out = [ac.verify(x, ring, scope, s) for x, s in zip(msgs, sigs)]
    return [st for st, _ in out], [t if (t and scope is not None) else bytes(32) for _, t in out]


@pytest.mark.parametrize("scope", [None, b"", b"scope"], ids=["unlinkable", "empty-scope", "scope"])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 5])
def test_whole_verification(lib, n, scope):
    rng = random.Random(f"{n}/{scope}")
    if n:
        ring, msgs, sigs, _ = ac.signed_batch(f"emul/{n}/{scope}", n, 3, scope, msg_lens=(0, 64, 129))
    else:
        ring, msgs = [], [b"", b"m", rng.randbytes(70)]
        sigs = [rng.randbytes(32) + (pc.random_point(rng) if scope is not None else b"") for _ in msgs]
        sigs[1] = ac.with_scalar(sigs[1], 0, L + 5)                 # n = 0: any C0 verifies
    bad = list(sigs)
    bad.append(ac.flip(sigs[0], 0))                                 # C0
    if n:
        bad.append(ac.flip(sigs[1], 32 * rng.randrange(1, n + 1) + 3))  # an S_i
    if scope is not None:
        bad.append(sigs[2][:-32] + pc.undecodable())                # Tag that does not decode
        bad.append(sigs[2][:-32] + ac.add(sigs[2][-32:], pc.T8))    # Tag + T8
    ms = msgs + [msgs[j % len(msgs)] for j in range(len(bad) - len(sigs))]
    rc, st, tags = run(lib, ring, ms, bad, scope)
    assert rc == 0
    assert (st, tags) == expect(ring, ms, bad, scope)
    assert st[:3] == [ac.OK] * 3


def test_ring_key_that_does_not_decode(lib):
    ring, msgs, sigs, _ = ac.signed_batch("emul/badkey", 3, 1, None)
    rc, _, _ = run(lib, [ring[0], pc.undecodable(), ring[2]], msgs, sigs, None)
    assert rc == -1
