"""CPU: the DLEQ / PVSS restatement (tests/pvss_cases.py) against the reference's own output and hashlib.

- keyed BLAKE2Xb and Scalar.Pick reproduce Example_schnorr (examples/sig_test.go:93-120, tests/golden/pvss_schnorr_example.json);
- the root hash equals hashlib's BLAKE2b with the same key and node parameters, for keys of 0..64 bytes and seeds longer than 64
  bytes (the tail is written as message); the output blocks are oracle.ed25519.Blake2Xb's (hashlib refuses their depth 0), and
  the empty seed agrees with it;
- honest proofs and PVSS rounds verify in the restatement, and each kind of corruption gives the status it should."""
import hashlib
import json
import os
import random

import pytest

from oracle import ed25519 as ed
import pvss_cases as pc

HERE = os.path.dirname(os.path.abspath(__file__))


def _hashlib_root(seed: bytes) -> bytes:
    return hashlib.blake2b(seed[64:], digest_size=64, key=seed[:64], fanout=1, depth=1, leaf_size=0,
                           node_offset=0xFFFFFFFF << 32, node_depth=0, inner_size=0).digest()


def test_example_schnorr_is_reproduced():
    f = json.load(open(os.path.join(HERE, "golden", "pvss_schnorr_example.json")))
    rand = pc.Xof(f["seed"].encode())
    x = pc.pick_int(rand)                                    # private key
    v = pc.pick_int(rand)                                    # SchnorrSign's commitment
    t = ed.encode(ed.scalar_mult(v))
    c = pc.pick_int(pc.Xof(t, f["message"].encode()))        # hashSchnorr: XOF(encode(T)) then Write(message)
    r = (v - x * c) % ed.L
    assert c.to_bytes(32, "little").hex() == f["c"]
    assert r.to_bytes(32, "little").hex() == f["r"]


@pytest.mark.parametrize("klen", list(range(0, 65)) + [65, 100, 127, 128, 129, 200, 300])
def test_keyed_xof_matches_hashlib(klen):
    rng = random.Random(klen)
    seed = bytes(rng.getrandbits(8) for _ in range(klen))
    x = pc.Xof(seed)
    assert x.root == _hashlib_root(seed)
    # hashlib refuses the output blocks' depth 0; they are the unkeyed blocks oracle.ed25519.Blake2Xb (pinned by the dh KAT)
    # derives from its root, so a stream with the same root must be the same
    ref = ed.Blake2Xb(b"")
    ref.h0 = x.root
    assert x.read(64 * 3) == ref.read(64 * 3)


def test_empty_seed_agrees_with_the_message_form():
    assert pc.Xof(b"").read(256) == ed.Blake2Xb(b"").read(256)


def test_pick_rejects_about_half_the_draws():
    draws = [pc.pick_draws(bytes([i]) * 32) for i in range(200)]
    assert 1.5 < sum(draws) / len(draws) < 2.6
    assert max(draws) >= 3


def test_dleq_statuses():
    rng = random.Random(1)
    g, h = pc.random_point(rng), pc.random_point(rng, torsion=True)
    proof, xg, xh = pc.new_dleq_proof(g, h, rng.randrange(ed.L), rng.randrange(ed.L))
    assert pc.dleq_verify(g, h, xg, xh, proof) == pc.OK
    bad_r = proof[:32] + ((int.from_bytes(proof[32:64], "little") + 1) % ed.L).to_bytes(32, "little") + proof[64:]
    assert pc.dleq_verify(g, h, xg, xh, bad_r) == pc.INVALID
    assert pc.dleq_verify(h, g, xg, xh, proof) == pc.INVALID
    assert pc.dleq_verify(g, h, pc.undecodable(), xh, proof) == pc.POINT


def test_v_zero_proof_with_noncanonical_identities_verifies():
    rng = random.Random(2)
    g, h = pc.random_point(rng), pc.random_point(rng)
    proof, xg, xh = pc.new_dleq_proof(g, h, rng.randrange(ed.L), 0)
    assert proof[64:96] == proof[96:] == pc.IDENTITY
    nc = pc.noncanonical_identity()
    assert nc != pc.IDENTITY and pc.canon(nc) == pc.IDENTITY
    assert pc.dleq_verify(g, h, xg, xh, proof[:64] + nc + nc) == pc.OK


def test_pvss_round_trip():
    rng = random.Random(3)
    n, t = 5, 3
    h = pc.random_point(rng)
    priv = [rng.randrange(1, ed.L) for _ in range(n)]
    xs = [pc.base_mul(k) for k in priv]
    secret = rng.randrange(ed.L)
    commits, shares, s = pc.enc_shares(h, xs, secret, t, pc.RandomStream("round trip"))
    shs = [pc.eval_commits(commits, i + 1) for i in range(n)]
    vs = [v for _, v, _ in shares]
    proofs = [p for _, _, p in shares]
    assert pc.verify_enc_share_batch(h, commits, xs, shs, vs, proofs) == [pc.OK] * n
    swapped = vs[:]
    swapped[0], swapped[1] = swapped[1], swapped[0]
    assert pc.verify_enc_share_batch(h, commits, xs, shs, swapped, proofs) == [pc.CHALLENGE] * n
    dec = []
    for i in range(n):
        dv, p = pc.dec_share(priv[i], vs[i], rng.randrange(ed.L))
        dec.append((i, dv, p))
    assert [pc.verify_dec_share(pc.G, xs[i], vs[i], dv, p) for i, dv, p in dec] == [pc.OK] * n
    assert pc.recover_secret(pc.G, xs, vs, dec, t) == pc.base_mul(secret)
    broken = [(i, pc.base_mul(7), p) if i < n - t + 1 else (i, dv, p) for i, dv, p in dec]
    assert pc.recover_secret(pc.G, xs, vs, broken, t) is None
