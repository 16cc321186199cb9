"""GPU: Boneh-Franklin IBE (CCA) on BLS12-381 through the C ABI against the restatement in oracle/ibe.py -- the drand timelock vector,
oracle-encrypt -> device-decrypt and device-encrypt -> oracle-decrypt on both groups (U, V, W byte for byte for a fixed sigma),
device round trips across the cooperative threshold (10240) and the fixed-G2 Miller loop, per-element statuses of a mixed batch,
a custom DST and the call errors."""
import random

import pytest

from kyber_b200.capi import B2KError, ERR_ARG, ERR_POINT
from oracle import bls12381 as o
from oracle import ibe

from test_oracle_ibe import TLOCK_BEACON, TLOCK_U, TLOCK_V, TLOCK_W, multi_iteration_case

pytestmark = pytest.mark.gpu


def _ops(on):
    return ((ibe.encrypt_cca_g1, ibe.decrypt_cca_g1) if on == 1 else (ibe.encrypt_cca_g2, ibe.decrypt_cca_g2))


def _bad_points(on, rng):
    """(off the curve, on the curve outside the subgroup) as compressed bytes of group `on`."""
    off = sub = None
    while off is None or sub is None:
        if on == 1:
            b = bytearray(rng.randrange(o.P).to_bytes(48, "big"))
            dec = o.g1_decompress
        else:
            b = bytearray(rng.randrange(o.P).to_bytes(48, "big") + rng.randrange(o.P).to_bytes(48, "big"))
            dec = o.g2_decompress
        b[0] |= 0x80
        b = bytes(b)
        try:
            dec(b, subgroup_check=False)
        except ValueError:
            off = off or b
            continue
        try:
            dec(b)
        except ValueError:
            sub = sub or b
    return off, sub


def test_tlock_vector(engine):
    """The drand vector (ibe_test.go:202-245): the device agrees with the oracle's full DecryptCCAonG1 (steps 1-2 give deadbeef...,
    the rP check does not hold for this U: PROOF, message zeroed)."""
    msgs, st = engine.bls12381_ibe_decrypt(1, TLOCK_BEACON, TLOCK_U, [TLOCK_V], [TLOCK_W])
    assert (msgs[0], st[0]) == ibe.decrypt_cca_g1(TLOCK_BEACON, TLOCK_U, TLOCK_V, TLOCK_W) == (bytes(16), ibe.PROOF)


@pytest.mark.parametrize("on", [1, 2])
def test_oracle_and_device_agree_both_ways(engine, on):
    rng = random.Random(40 + on)
    ident = b"round 1234"
    master, priv = ibe.keypair(on, rng.randrange(1, o.R), ident)
    enc, dec = _ops(on)
    s3, m3, _ = multi_iteration_case()
    cases = [(b"", b""), (b"x", b"y"), (rng.randbytes(12), rng.randbytes(12)), (rng.randbytes(32), rng.randbytes(32)), (m3, s3)]
    for msg, sigma in cases:
        # device encrypt with a fixed sigma == oracle encrypt, byte for byte
        u, v, w = engine.bls12381_ibe_encrypt(on, master, ident, [msg], [sigma])
        U, V, W = enc(master, ident, msg, sigma)
        assert (u, v[0], w[0]) == (U, V, W), len(msg)
        assert dec(priv, u, v[0], w[0]) == (msg, ibe.OK)
        # oracle ciphertext -> device decrypt
        got, st = engine.bls12381_ibe_decrypt(on, priv, U, [V], [W])
        assert (got[0], st[0]) == (msg, ibe.OK), len(msg)


@pytest.mark.parametrize("on,n", [(1, 1), (1, 10240), (1, 10241), (1, 1 << 16), (2, 1), (2, 10241)])
def test_device_round_trip(engine, on, n):
    rng = random.Random(n + on)
    ident = b"round %d" % n
    master, priv = ibe.keypair(on, rng.randrange(1, o.R), ident)
    ln = 16
    msgs = [rng.randbytes(ln) for _ in range(n)]
    sigmas = [rng.randbytes(ln) for _ in range(n)]
    u, v, w = engine.bls12381_ibe_encrypt(on, master, ident, msgs, sigmas)
    got, st = engine.bls12381_ibe_decrypt(on, priv, u, v, w)
    assert st == bytes(n)
    assert got == msgs
    ub = 48 * on
    enc, dec = _ops(on)
    for i in sorted({0, n // 2, n - 1}):                 # spot checks against the oracle at both ends of the batch
        assert (u[ub * i:ub * (i + 1)], v[i], w[i]) == enc(master, ident, msgs[i], sigmas[i])


@pytest.mark.parametrize("on,n", [(1, 12), (1, 10241 + 12), (2, 12)])
def test_mixed_batch_statuses(engine, on, n):
    """Every failure kind once, in a batch that is otherwise valid (n - 12 + 6 good ciphertexts); the large G1 batch takes the
    fixed-G2 Miller loop."""
    rng = random.Random(77 + n)
    ident = b"mixed"
    master, priv = ibe.keypair(on, rng.randrange(1, o.R), ident)
    msgs = [rng.randbytes(12) for _ in range(n)]
    u, v, w = engine.bls12381_ibe_encrypt(on, master, ident, msgs, [rng.randbytes(12) for _ in range(n)])
    ub = 48 * on
    us = [u[ub * i:ub * (i + 1)] for i in range(n)]
    off, sub = _bad_points(on, rng)
    want = [ibe.OK] * n
    v[1] = b"somenonsense"; want[1] = ibe.PROOF
    w[2] = b"somenonsense"; want[2] = ibe.PROOF
    us[3] = off; want[3] = ibe.POINT
    us[4] = sub; want[4] = ibe.POINT
    us[5] = o.g1_compress(None) if on == 1 else o.g2_compress(None); want[5] = ibe.PROOF
    us[6] = us[7]; want[6] = ibe.PROOF
    us[n - 1] = bytes(ub); want[n - 1] = ibe.POINT        # no compression flag
    got, st = engine.bls12381_ibe_decrypt(on, priv, b"".join(us), v, w)
    assert list(st) == want
    _, dec = _ops(on)
    for i in range(n):
        assert got[i] == (msgs[i] if want[i] == ibe.OK else bytes(12)), i
    for i in range(8):
        assert (got[i], st[i]) == dec(priv, us[i], v[i], w[i]), i


@pytest.mark.parametrize("on", [1, 2])
def test_custom_dst(engine, on):
    rng = random.Random(90 + on)
    dst = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_custom" if on == 1 else b"my-ibe-dst"
    ident = b"id with a dst"
    master, priv = ibe.keypair(on, rng.randrange(1, o.R), ident, dst)
    enc, _ = _ops(on)
    msg, sigma = rng.randbytes(20), rng.randbytes(20)
    u, v, w = engine.bls12381_ibe_encrypt(on, master, ident, [msg], [sigma], dst=dst)
    assert (u, v[0], w[0]) == enc(master, ident, msg, sigma, dst)
    assert engine.bls12381_ibe_decrypt(on, priv, u, v, w) == ([msg], b"\x00")
    # the default DST gives another identity point: the same key no longer decrypts
    u2, v2, w2 = engine.bls12381_ibe_encrypt(on, master, ident, [msg], [sigma])
    assert engine.bls12381_ibe_decrypt(on, priv, u2, v2, w2) == ([bytes(20)], bytes([ibe.PROOF]))


@pytest.mark.parametrize("on", [1, 2])
def test_call_errors(engine, on):
    rng = random.Random(5)
    master, priv = ibe.keypair(on, rng.randrange(1, o.R), b"id")
    u, v, w = engine.bls12381_ibe_encrypt(on, master, b"id", [b"abc"], [b"def"])
    off, _ = _bad_points(3 - on, rng)
    with pytest.raises(B2KError) as e:
        engine.bls12381_ibe_decrypt(on, off, u, v, w)
    assert e.value.code == ERR_POINT
    moff, _ = _bad_points(on, rng)
    with pytest.raises(B2KError) as e:
        engine.bls12381_ibe_encrypt(on, moff, b"id", [b"abc"], [b"def"])
    assert e.value.code == ERR_POINT
    with pytest.raises(B2KError) as e:
        engine.bls12381_ibe_decrypt(on, priv, u, [bytes(33)], [bytes(33)])
    assert e.value.code == ERR_ARG
    with pytest.raises(B2KError) as e:
        engine.bls12381_ibe_encrypt(on, master, b"id", [bytes(33)], [bytes(33)])
    assert e.value.code == ERR_ARG
    assert engine.bls12381_ibe_decrypt(on, priv, u, v, w) == ([b"abc"], b"\x00")     # the context is usable after the errors


def test_pair_fixed_g2_matches_pair(engine):
    rng = random.Random(8)
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(37)] + [None]
    for q in (o.g2_mul(rng.randrange(1, o.R)), None):
        g1 = b"".join(o.g1_to_affine_bytes(p) for p in pts)
        g2 = o.g2_to_affine_bytes(q)
        assert engine.bls12381_pair_fixed_g2(g1, g2) == engine.bls12381_pair(g1, g2 * len(pts))
