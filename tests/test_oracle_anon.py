"""CPU: the ring signature restatement (tests/anon_cases.py) against the reference's own fixtures -- the three Examples of
sign/anon/sig_test.go reproduced byte for byte with RandomStream = blake2xb.New(nil) -- and the verification rules a device
implementation must keep: raw scalars and the e63 rule, n = 0, and the canonical tag."""
import json
import os
import random

import pytest

import anon_cases as ac
import ed25519_msm_cases as mc
import pvss_cases as pc

HERE = os.path.dirname(os.path.abspath(__file__))
EX = {e["name"]: e for e in json.load(open(os.path.join(HERE, "golden", "anon_examples.json")))["examples"]}
L = ac.L


def replay(name):
    return ac.replay_example(EX[name])


@pytest.mark.parametrize("name", sorted(EX))
def test_examples_sign_byte_for_byte(name):
    _, _, _, sigs = replay(name)
    assert [s.hex() for s in sigs] == EX[name]["sigs"]


@pytest.mark.parametrize("name", sorted(EX))
def test_examples_verify(name):
    msg, ring, scope, sigs = replay(name)
    e = EX[name]
    for j, s in enumerate(sigs):
        st, tag = ac.verify(msg, ring, scope, s)
        assert st == ac.OK
        assert tag == (bytes.fromhex(e["tags"][j]) if scope is not None else b"")
        assert ac.verify(e["bad_message"].encode(), ring, scope, s) == (ac.INVALID, None)


def test_raw_scalars_and_the_e63_rule():
    ring, msgs, sigs, _ = ac.signed_batch("oracle/raw", 3, 1, None)
    msg, sig = msgs[0], sigs[0]
    s1 = int.from_bytes(sig[64:96], "little")
    kept = dropped = 0
    for v, e63 in ac.high_variants(s1):
        st, _ = ac.verify(msg, ring, None, ac.with_scalar(sig, 2, v))
        if e63 <= 8:
            assert mc.effective_scalar(v) % L == s1 and st == ac.OK
            kept += 1
        else:
            dropped += st == ac.INVALID
    assert kept and dropped
    c0 = int.from_bytes(sig[:32], "little")
    assert ac.verify(msg, ring, None, ac.with_scalar(sig, 0, c0 + L))[0] == ac.INVALID   # Scalar.Equal on raw bytes


def test_n_zero_accepts_any_c0():
    rng = random.Random(1)
    for c0 in (0, L, (1 << 256) - 1, rng.getrandbits(256)):
        assert ac.verify(b"m", [], None, mc.le([c0])) == (ac.OK, b"")
        tag = pc.random_point(rng)
        assert ac.verify(b"m", [], b"s", mc.le([c0]) + tag) == (ac.OK, tag)
        assert ac.verify(b"m", [], b"s", mc.le([c0]) + pc.undecodable()) == (ac.POINT, None)


def test_noncanonical_tag_is_hashed_and_returned_canonical():
    # a signer whose key is 0: its tag is the identity, which has the non-canonical encoding y = 1 + p
    rng = random.Random(2)
    ring, _ = ac.ring_with_signer(rng, 3, 1, 0)
    sig = ac.sign(b"vote", ring, b"poll", 1, 0, pc.Xof(b"seed"))
    assert sig[-32:] == pc.IDENTITY
    nc = sig[:-32] + pc.noncanonical_identity()
    assert ac.verify(b"vote", ring, b"poll", nc) == (ac.OK, pc.IDENTITY)


def test_torsion_ring_keys():
    rng = random.Random(3)
    x, _ = ac.keypair(rng)
    ring, clean = ac.ring_with_signer(rng, 4, 2, x, torsion=True)
    for scope in (None, b"s"):
        sig = ac.sign(b"t", ring, scope, 2, x, pc.Xof(b"t"))
        assert ac.verify(b"t", ring, scope, sig)[0] == ac.OK
        assert ac.verify(b"t", clean, scope, sig)[0] == ac.INVALID
