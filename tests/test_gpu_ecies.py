"""GPU: ECIES on edwards25519 (b2k_ed25519_ecies_decrypt / _encrypt) against the restatement in oracle/ecies.py, byte for byte,
and the Pedersen DKG's ProcessDeals as one decryption call plus one PubPoly.Check call."""
import random

import pytest

import ed25519_msm_cases as mc
from oracle import ecies as ec
from oracle import ed25519 as ed

pytestmark = pytest.mark.gpu
L = ed.L
IDENT = ed.encode(ed.IDENT)


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def bad_point():
    return next(bytes([i]) + bytes(31) for i in range(2, 256) if ed.decode(bytes([i]) + bytes(31)) is None)


def test_decrypt_against_the_oracle(eng):
    rng = random.Random(1)
    priv = rng.randbytes(32)
    pub = ec.mul(priv)
    cts = [ec.encrypt(pub, rng.randbytes(32), rng.randbytes(32))[1] for _ in range(257)]
    msgs, st = eng.ed25519_ecies_decrypt(priv, cts, 48)
    assert list(zip(st, msgs)) == [ec.decrypt(priv, c) for c in cts]
    assert set(st) == {ec.OK}


def test_encrypt_against_the_oracle(eng):
    rng = random.Random(2)
    pubs = [ec.mul(rng.randbytes(32)) for _ in range(257)]
    rs = [rng.randbytes(32) for _ in pubs[:-3]] + [b"\xff" * 32, (0x8f << 248).to_bytes(32, "little"), bytes(32)]
    msgs = [rng.randbytes(32) for _ in pubs]
    cts, st = eng.ed25519_ecies_encrypt(pubs, rs, msgs)
    assert list(zip(st, cts)) == [ec.encrypt(p, r, m) for p, r, m in zip(pubs, rs, msgs)]


@pytest.mark.parametrize("length", [0, 32, 1000])
@pytest.mark.parametrize("n", [1, 4096, 1 << 16])
def test_round_trip(eng, n, length):
    rng = random.Random(n * 7 + length)
    priv = rng.randbytes(32)
    pub = ec.mul(priv)
    rs = [rng.randbytes(32) for _ in range(n)]
    msgs = [rng.randbytes(length) for _ in range(n)]
    cts, st = eng.ed25519_ecies_encrypt([pub] * n, rs, msgs)
    assert st == bytes(n)
    for i in {0, n // 2, n - 1}:                                      # spot checks against the oracle
        assert cts[i] == ec.encrypt(pub, rs[i], msgs[i])[1]
    back, st = eng.ed25519_ecies_decrypt(priv, cts, length + 16)
    assert st == bytes(n) and back == msgs


def test_mixed_batch(eng):
    rng = random.Random(3)
    priv = rng.randbytes(32)
    pub = ec.mul(priv)
    good = [ec.encrypt(pub, rng.randbytes(32), rng.randbytes(40))[1] for _ in range(6)]
    flipped_tag = bytearray(good[1]); flipped_tag[-3] ^= 0x10
    flipped_body = bytearray(good[2]); flipped_body[40] ^= 0x01
    batch = [good[0], bad_point() + good[0][32:], bytes(flipped_tag), bytes(flipped_body), ec.mul(rng.randbytes(32)) + good[3][32:],
             IDENT + good[4][32:], mc.T8 + good[4][32:], bytes(32) + good[5][32:], good[5]]
    msgs, st = eng.ed25519_ecies_decrypt(priv, batch, 56)
    want = [ec.decrypt(priv, c) for c in batch]
    assert list(zip(st, msgs)) == want
    assert list(st) == [ec.OK, ec.POINT, ec.AUTH, ec.AUTH, ec.AUTH, ec.AUTH, ec.AUTH, ec.AUTH, ec.OK]


def test_encrypt_to_small_order_and_bad_keys(eng):
    rng = random.Random(4)
    pubs = [IDENT, mc.T8, bytes(32), bad_point(), ec.mul(rng.randbytes(32))]
    rs = [rng.randbytes(32) for _ in pubs]
    msgs = [rng.randbytes(32) for _ in pubs]
    cts, st = eng.ed25519_ecies_encrypt(pubs, rs, msgs)
    assert list(zip(st, cts)) == [ec.encrypt(p, r, m) for p, r, m in zip(pubs, rs, msgs)]
    assert list(st) == [ec.OK, ec.OK, ec.OK, ec.POINT, ec.OK]
    # r times the identity is the identity: the key comes from its encoding, so the body opens without any private key
    key, nonce = ec.derive(IDENT)
    assert ec.gcm_open(key, nonce, cts[0][32:]) == msgs[0]


def test_call_errors(eng):
    import ctypes
    from kyber_b200.capi import B2KError
    with pytest.raises(B2KError):
        eng.ed25519_ecies_decrypt(bytes(32), [], 48)                 # n = 0
    with pytest.raises(B2KError):
        eng.ed25519_ecies_decrypt(bytes(32), [bytes(47)], 15)        # shorter than a tag
    with pytest.raises(B2KError):
        eng.ed25519_ecies_encrypt([IDENT], [bytes(32)], [bytes(ec.MAX_LEN + 1)])
    with pytest.raises(B2KError):
        eng.ed25519_ecies_encrypt([], [], [])
    buf = ctypes.create_string_buffer(256)
    assert eng.lib.b2k_ed25519_ecies_decrypt(eng.h, None, 1, 48, buf, buf, buf) != 0
    assert eng.lib.b2k_ed25519_ecies_decrypt(eng.h, buf, 1, ec.MAX_LEN + 17, buf, buf, buf) != 0
    assert eng.lib.b2k_ed25519_ecies_encrypt(eng.h, 1, buf, None, 32, buf, buf, buf) != 0
    assert eng.lib.b2k_ed25519_ecies_decrypt(eng.h, buf, (1 << 64) - 1, 48, buf, buf, buf) != 0   # n len overflows


def test_dkg_process_deals(eng):
    """64 dealers with t = 22 deal to node nidx; one share is wrong and one ciphertext tampered.  Deals() is one encryption
    call, ProcessDeals one decryption call plus one PubPoly.Check over the dealers' commitments at the single index nidx."""
    rng = random.Random(5)
    m, t, nidx = 64, 22, 9
    priv = rng.randbytes(32)
    pub = ec.mul(priv)
    polys = [[rng.randrange(L) for _ in range(t)] for _ in range(m)]
    commits = b"".join(ec.mul(a.to_bytes(32, "little")) for f in polys for a in f)
    x = nidx + 1
    shares = [sum(a * pow(x, j, L) for j, a in enumerate(f)) % L for f in polys]
    shares[7] = (shares[7] + 1) % L                                  # a dealer that deals a wrong share
    plain = [s.to_bytes(32, "little") for s in shares]
    cts, st = eng.ed25519_ecies_encrypt([pub] * m, [rng.randbytes(32) for _ in range(m)], plain)
    assert st == bytes(m)
    tampered = bytearray(cts[30]); tampered[50] ^= 0x04
    cts[30] = bytes(tampered)
    got, dst = eng.ed25519_ecies_decrypt(priv, cts, 48)
    ok = eng.ed25519_pubpoly_check(commits, t, [[nidx]] * m, b"".join(got))
    verdict = [d == ec.OK and o == 1 for d, o in zip(dst, ok)]
    want = []
    for j in range(m):                                               # the oracle's ProcessDeals, dealer by dealer
        s, msg = ec.decrypt(priv, cts[j])
        if s != ec.OK:
            want.append(False)
            continue
        comm = ed.IDENT
        for k, a in enumerate(polys[j]):
            comm = ed.add(comm, ed.scalar_mult(a * pow(x, k, L) % L))
        want.append(ec.mul(msg) == ed.encode(comm))
    assert verdict == want
    assert [j for j in range(m) if not verdict[j]] == [7, 30]
    assert dst[30] == ec.AUTH and dst[7] == ec.OK
