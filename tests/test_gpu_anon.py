"""GPU: ring signature verification on edwards25519 (b2k_ed25519_anon_verify) against the restatement in tests/anon_cases.py.

Every status and tag is compared with the restated anon.Verify; the reference's three Examples verify with their printed tags."""
import json
import os
import random

import pytest

import anon_cases as ac
import ed25519_msm_cases as mc
import pvss_cases as pc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
L = ac.L
ZERO_TAG = bytes(32)


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def expect(ring, msgs, sigs, scope):
    out = [ac.verify(x, ring, scope, s) for x, s in zip(msgs, sigs)]
    return [st for st, _ in out], [t if (st == ac.OK and scope is not None) else ZERO_TAG for st, t in out]


def check(eng, ring, msgs, sigs, scope):
    st, tags = eng.ed25519_anon_verify(b"".join(ring), msgs, sigs, scope)
    got = (list(st), [tags[32 * j:32 * j + 32] for j in range(len(msgs))])
    want = expect(ring, msgs, sigs, scope)
    assert got == want
    return got[0]


def test_reference_examples(eng):
    ex = {e["name"]: e for e in json.load(open(os.path.join(HERE, "golden", "anon_examples.json")))["examples"]}
    for name, e in ex.items():
        msg, ring, scope, _ = ac.replay_example(e)
        sigs = [bytes.fromhex(s) for s in e["sigs"]]
        bad = e["bad_message"].encode()
        st, tags = eng.ed25519_anon_verify(b"".join(ring), [msg] * len(sigs) + [bad] * len(sigs), sigs + sigs, scope)
        assert list(st) == [ac.OK] * len(sigs) + [ac.INVALID] * len(sigs), name
        want = [bytes.fromhex(t) for t in e["tags"]] if scope is not None else [ZERO_TAG] * len(sigs)
        assert [tags[32 * j:32 * j + 32] for j in range(len(sigs))] == want
        assert tags[32 * len(sigs):] == bytes(32 * len(sigs))


MODES = [None, b"", b"ballot 2026"]
MODE_IDS = ["unlinkable", "empty-scope", "scope"]


@pytest.mark.parametrize("scope", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("n", [0, 1, 2, 3, 17, 300])
def test_ring_sizes(eng, n, scope):
    """300 positions cross the 128-position chunk boundary twice"""
    rng = random.Random(f"sizes/{n}/{scope}")
    if n:
        m = 2 if n > 100 else 4
        ring, msgs, sigs, _ = ac.signed_batch(f"gpu/{n}/{scope}", n, m, scope, msg_lens=(5, 80))
    else:
        ring, msgs = [], [b"", b"x", rng.randbytes(100)]
        sigs = [rng.randbytes(32) + (pc.random_point(rng) if scope is not None else b"") for _ in msgs]
        sigs[0] = ac.with_scalar(sigs[0], 0, L + 7)                 # n = 0 with C0 >= l: OK
        sigs[2] = ac.with_scalar(sigs[2], 0, (1 << 256) - 1)
    bad = [ac.flip(sigs[0], 5, 2)]
    if n:
        bad.append(ac.flip(sigs[1], 32 * rng.randrange(1, n + 1) + rng.randrange(32), rng.randrange(8)))
    st = check(eng, ring, msgs + msgs[:len(bad)], sigs + bad, scope)
    assert st[:len(sigs)] == [ac.OK] * len(sigs)


@pytest.mark.parametrize("scope_len", [None, 0, 1, 64, 65, 200])
def test_message_and_scope_lengths(eng, scope_len):
    rng = random.Random(f"lens/{scope_len}")
    scope = rng.randbytes(scope_len) if scope_len is not None else None
    lens = (0, 1, 63, 64, 65, 127, 128, 129, 1000)
    ring, msgs, sigs, _ = ac.signed_batch(f"gpu/lens/{scope_len}", 2, len(lens), scope, msg_lens=lens)
    wrong = [ac.flip(msgs[j], 0) if msgs[j] else b"\x00" for j in range(len(msgs))]
    st = check(eng, ring, msgs + wrong, sigs + sigs, scope)
    assert st == [ac.OK] * len(lens) + [ac.INVALID] * len(lens)


@pytest.mark.parametrize("scope", MODES, ids=MODE_IDS)
def test_corruptions(eng, scope):
    rng = random.Random(f"corrupt/{scope}")
    n = 5
    ring, msgs, sigs, who = ac.signed_batch(f"gpu/corrupt/{scope}", n, 4, scope)
    cases, cmsgs = [], []
    for j, s in enumerate(sigs):
        cases += [ac.flip(s, rng.randrange(32), rng.randrange(8)),                         # C0
                  ac.flip(s, 32 * rng.randrange(1, n + 1) + rng.randrange(32), rng.randrange(8))]   # an S_i
        cmsgs += [msgs[j]] * 2
        if scope is not None:
            cases.append(ac.flip(s, 32 * (n + 1) + rng.randrange(31), rng.randrange(8)))  # the Tag
            cmsgs.append(msgs[j])
        cases.append(s)                                                                   # the wrong message
        cmsgs.append(msgs[j] + b"!")
    st = check(eng, ring, cmsgs, cases, scope)
    assert ac.OK not in st
    # a signer outside the ring: the signer's key replaced by another
    other = list(ring)
    other[who[0]] = ac.keypair(rng)[1]
    assert check(eng, other, msgs[:1], sigs[:1], scope) == [ac.INVALID]


@pytest.mark.parametrize("scope", [None, b"s"], ids=["unlinkable", "linkable"])
def test_scalar_rules(eng, scope):
    ring, msgs, sigs, _ = ac.signed_batch(f"gpu/raw/{scope}", 3, 1, scope)
    msg, sig = msgs[0], sigs[0]
    cases, digits = [], []
    for slot in (1, 2, 3):
        s = int.from_bytes(sig[32 * slot:32 * slot + 32], "little")
        for v, e63 in ac.high_variants(s):
            cases.append(ac.with_scalar(sig, slot, v))
            digits.append(e63)
    c0 = int.from_bytes(sig[:32], "little")
    cases.append(ac.with_scalar(sig, 0, c0 + L))
    st = check(eng, ring, [msg] * len(cases), cases, scope)
    assert all(x == ac.OK for x, d in zip(st, digits) if d <= 8)
    assert ac.INVALID in st[:-1] and st[-1] == ac.INVALID


def test_torsion_and_tags(eng):
    rng = random.Random("torsion")
    x, _ = ac.keypair(rng)
    ring, clean = ac.ring_with_signer(rng, 6, 4, x, torsion=True)
    for scope in (None, b"poll"):
        sig = ac.sign(b"t", ring, scope, 4, x, pc.Xof(b"t"))
        assert check(eng, ring, [b"t"], [sig], scope) == [ac.OK]
        assert check(eng, clean, [b"t"], [sig], scope) == [ac.INVALID]
    sig = ac.sign(b"t", ring, b"poll", 4, x, pc.Xof(b"t2"))
    tag = sig[-32:]
    cases = [sig[:-32] + ac.add(tag, pc.T8), sig[:-32] + pc.undecodable(), sig]
    assert check(eng, ring, [b"t"] * 3, cases, b"poll") == [ac.INVALID, ac.POINT, ac.OK]
    # key 0: the tag is the identity, sent in its non-canonical encoding y = 1 + p
    ring0, _ = ac.ring_with_signer(rng, 3, 0, 0)
    sig0 = ac.sign(b"z", ring0, b"poll", 0, 0, pc.Xof(b"z"))
    nc = sig0[:-32] + pc.noncanonical_identity()
    st, tags = eng.ed25519_anon_verify(b"".join(ring0), [b"z"], [nc], b"poll")
    assert list(st) == [ac.OK] and tags == pc.IDENTITY
    check(eng, ring0, [b"z"], [nc], b"poll")


def test_large_tiled_batch(eng):
    """2^16 signatures tiled from 64 distinct ones (n = 8, linkable), 16 corrupted at seeded positions"""
    scope = b"proof of personhood"
    ring, msgs, sigs, _ = ac.signed_batch("gpu/tiled", 8, 64, scope, msg_lens=(0, 33, 70, 130))
    base_st, base_tags = expect(ring, msgs, sigs, scope)
    assert base_st == [ac.OK] * 64
    m = 1 << 16
    rng = random.Random(7)
    bad_at = sorted(rng.sample(range(m), 16))
    all_msgs = [msgs[j % 64] for j in range(m)]
    all_sigs = [sigs[j % 64] for j in range(m)]
    for j in bad_at:
        all_sigs[j] = ac.flip(all_sigs[j], rng.randrange(len(all_sigs[j])), rng.randrange(8))
    st, tags = eng.ed25519_anon_verify(b"".join(ring), all_msgs, all_sigs, scope)
    bad = set(bad_at)
    for j in range(m):
        if j in bad:
            want = expect(ring, [all_msgs[j]], [all_sigs[j]], scope)
            assert (st[j], tags[32 * j:32 * j + 32]) == (want[0][0], want[1][0])
            assert st[j] != ac.OK
        else:
            assert st[j] == ac.OK and tags[32 * j:32 * j + 32] == base_tags[j % 64]


def test_call_errors(eng):
    from kyber_b200.capi import B2KError, ERR_ARG, ERR_POINT
    ring, msgs, sigs, _ = ac.signed_batch("gpu/errors", 3, 2, b"s")
    bad_ring = ring[:1] + [pc.undecodable()] + ring[2:]
    with pytest.raises(B2KError) as e:
        eng.ed25519_anon_verify(b"".join(bad_ring), msgs, sigs, b"s")
    assert e.value.code == ERR_POINT
    with pytest.raises(B2KError) as e:
        eng.ed25519_anon_verify(b"".join(ring), [], [], b"s")         # m = 0
    assert e.value.code == ERR_ARG
    import ctypes
    st = ctypes.create_string_buffer(2)
    rc = eng.lib.b2k_ed25519_anon_verify(eng.h, 3, b"".join(ring), 1, b"s", 1, 2, None, None, b"".join(sigs), st, None)
    assert rc == ERR_ARG                                               # null messages / offsets
    assert check(eng, ring, msgs, sigs, b"s") == [ac.OK, ac.OK]        # the context still works
