"""GPU: ECIES on BLS12-381 with keys on G1 and on G2 (b2k_bls12381_g{1,2}_ecies_decrypt / _encrypt) against the restatement in
tests/ecies_bls12381_oracle.py, byte for byte: scalars 0, 1 and r - 1, infinity as R and as the public key, every encoding
UnmarshalBinary refuses, tampered bodies and tags, every length class, the call errors, round trips up to 2^16 ciphertexts,
and the Pedersen DKG's ProcessDeals on BLS12-381 keys as one decryption call plus one PubPoly.Check call."""
import ctypes
import random

import pytest

from oracle import bls12381 as bls
import ecies_bls12381_oracle as eb
import schnorr_cases as sc

pytestmark = pytest.mark.gpu
R = bls.R
GROUPS = eb.GROUPS


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def sb(k: int) -> bytes:
    return k.to_bytes(32, "big")


def pub_batch(eng, group, ks):
    """the compressed public keys k G, computed on the device (the round trips check them against the oracle's)"""
    gen = bls.g1_to_affine_bytes(bls.G1) if group == 1 else bls.g2_to_affine_bytes(bls.G2)
    mul = eng.bls12381_g1_mul_batch if group == 1 else eng.bls12381_g2_mul_batch
    out = mul(b"".join(sb(k) for k in ks), gen * len(ks))
    pl = eb.POINT_LEN[group]
    return [out[pl * i:pl * i + pl] for i in range(len(ks))]


@pytest.mark.parametrize("group", GROUPS)
def test_decrypt_against_the_oracle(eng, group):
    rng = random.Random(100 + group)
    pl = eb.POINT_LEN[group]
    inf = eb.compress(group, None)
    priv = sb(rng.randrange(R))
    pub = eb.public(group, priv)
    rs = [sb(0), sb(1), sb(R - 1)] + [sb(rng.randrange(R)) for _ in range(254)]
    msgs = [rng.randbytes(32) for _ in rs]
    cts = [eb.encrypt(group, pub, r, m)[1] for r, m in zip(rs, msgs)]
    cts[10] = inf + cts[10][pl:]                                     # R at infinity: dh at infinity, the tag fails
    key, nonce = eb.derive(inf)
    from oracle import ecies as ec
    cts[11] = inf + ec.gcm_seal(key, nonce, msgs[11])               # R at infinity, sealed under dh = infinity: OK
    got, st = eng.bls12381_ecies_decrypt(group, priv, cts, 48)
    assert list(zip(st, got)) == [eb.decrypt(group, priv, c) for c in cts]
    assert st[10] == eb.AUTH and [st[i] for i in range(len(cts)) if i != 10] == [eb.OK] * (len(cts) - 1)
    for k in (0, 1, R - 1):                                          # the extreme private keys, infinity among them
        p = eb.public(group, sb(k))
        cts = [eb.encrypt(group, p, r, m)[1] for r, m in zip(rs[:4], msgs[:4])]
        got, st = eng.bls12381_ecies_decrypt(group, sb(k), cts, 48)
        assert st == bytes(4) and got == msgs[:4], k


@pytest.mark.parametrize("group", GROUPS)
def test_encrypt_against_the_oracle(eng, group):
    rng = random.Random(200 + group)
    ks = [rng.randrange(1, R) for _ in range(254)]
    pubs = [eb.compress(group, None), eb.public(group, sb(1)), eb.public(group, sb(R - 1))] + pub_batch(eng, group, ks)
    rs = [sb(rng.randrange(R)) for _ in range(254)] + [sb(0), sb(1), sb(R - 1)]
    msgs = [rng.randbytes(32) for _ in pubs]
    cts, st = eng.bls12381_ecies_encrypt(group, pubs, rs, msgs)
    assert list(zip(st, cts)) == [eb.encrypt(group, p, r, m) for p, r, m in zip(pubs, rs, msgs)]
    assert st == bytes(len(pubs))


@pytest.mark.parametrize("group", GROUPS)
def test_every_point_rejection(eng, group):
    """each encoding UnmarshalBinary refuses is POINT, as R and as the public key, with zeroed outputs"""
    rng = random.Random(300 + group)
    pl = eb.POINT_LEN[group]
    name = f"bls12381_g{group}"
    bad = [b for _, b in sc.bad_encodings(name)]
    assert len(bad) == 7
    priv = sb(rng.randrange(R))
    good = eb.encrypt(group, eb.public(group, priv), sb(rng.randrange(R)), rng.randbytes(32))[1]
    cts = [b + good[pl:] for b in bad] + [good]
    got, st = eng.bls12381_ecies_decrypt(group, priv, cts, 48)
    assert list(zip(st, got)) == [eb.decrypt(group, priv, c) for c in cts]
    assert list(st) == [eb.POINT] * 7 + [eb.OK] and got[:7] == [bytes(32)] * 7
    msgs = [rng.randbytes(32) for _ in bad]
    cts, st = eng.bls12381_ecies_encrypt(group, bad, [sb(rng.randrange(R)) for _ in bad], msgs)
    assert st == bytes([eb.POINT]) * 7 and cts == [bytes(pl + 48)] * 7


@pytest.mark.parametrize("group", GROUPS)
def test_auth_failures(eng, group):
    rng = random.Random(400 + group)
    pl = eb.POINT_LEN[group]
    priv = sb(rng.randrange(R))
    pub = eb.public(group, priv)
    good = [eb.encrypt(group, pub, sb(rng.randrange(R)), rng.randbytes(40))[1] for _ in range(3)]
    body = bytearray(good[0]); body[pl + 7] ^= 0x20
    tag = bytearray(good[1]); tag[-5] ^= 0x01
    cts = [bytes(body), bytes(tag), good[2]]
    got, st = eng.bls12381_ecies_decrypt(group, priv, cts, 56)
    assert list(zip(st, got)) == [eb.decrypt(group, priv, c) for c in cts]
    assert list(st) == [eb.AUTH, eb.AUTH, eb.OK] and got[:2] == [bytes(40)] * 2


@pytest.mark.parametrize("length", [0, 32, 1000, eb.MAX_LEN])
@pytest.mark.parametrize("group", GROUPS)
def test_lengths(eng, group, length):
    rng = random.Random(500 + group + length)
    priv = sb(rng.randrange(R))
    pub = eb.public(group, priv)
    rs = [sb(rng.randrange(R)) for _ in range(3)]
    msgs = [rng.randbytes(length) for _ in rs]
    cts, st = eng.bls12381_ecies_encrypt(group, [pub] * 3, rs, msgs)
    assert st == bytes(3)
    assert cts[1] == eb.encrypt(group, pub, rs[1], msgs[1])[1]
    got, st = eng.bls12381_ecies_decrypt(group, priv, cts, length + 16)
    assert st == bytes(3) and got == msgs
    assert eb.decrypt(group, priv, cts[2]) == (eb.OK, msgs[2])


@pytest.mark.parametrize("group", GROUPS)
def test_call_errors(eng, group):
    from kyber_b200.capi import B2KError
    pl = eb.POINT_LEN[group]
    dec = getattr(eng.lib, f"b2k_bls12381_g{group}_ecies_decrypt")
    enc = getattr(eng.lib, f"b2k_bls12381_g{group}_ecies_encrypt")
    pub = eb.public(group, sb(3))
    ct = eb.encrypt(group, pub, sb(5), bytes(32))[1]
    with pytest.raises(B2KError) as e:
        eng.bls12381_ecies_decrypt(group, sb(R), [ct], 48)            # priv = r
    assert e.value.code == -3
    with pytest.raises(B2KError) as e:
        eng.bls12381_ecies_encrypt(group, [pub] * 3, [sb(1), sb(R), sb(2)], [bytes(32)] * 3)    # one r_i = r
    assert e.value.code == -3
    buf = ctypes.create_string_buffer(1 << 10)
    out = ctypes.create_string_buffer(1 << 10)
    assert dec(eng.h, sb(R + 1), 1, 48, ct, out, out) == -3
    assert enc(eng.h, 1, pub, b"\xff" * 32, 32, buf, out, out) == -3
    assert dec(eng.h, None, 1, 48, buf, out, out) == -2                          # a null pointer
    assert enc(eng.h, 1, buf, None, 32, buf, out, out) == -2
    assert dec(eng.h, sb(1), 0, 48, buf, out, out) == -2                         # n = 0
    assert enc(eng.h, 0, buf, buf, 32, buf, out, out) == -2
    assert dec(eng.h, sb(1), 1, 15, buf, out, out) == -2                         # shorter than a tag
    assert dec(eng.h, sb(1), 1, eb.MAX_LEN + 17, buf, out, out) == -2            # longer than the limit
    assert enc(eng.h, 1, buf, buf, eb.MAX_LEN + 1, buf, out, out) == -2
    assert dec(eng.h, sb(1), (1 << 64) - 1, 48, buf, out, out) == -2             # n len overflows
    assert enc(eng.h, (1 << 62), buf, buf, 1000, buf, out, out) == -2
    got, st = eng.bls12381_ecies_decrypt(group, sb(3), [ct], 48)                 # the context still works
    assert st == bytes(1) and got == [bytes(32)] and len(ct) == pl + 48


@pytest.mark.parametrize("length", [32, 1000])
@pytest.mark.parametrize("n", [1, 4096, 1 << 16])
@pytest.mark.parametrize("group", GROUPS)
def test_round_trip(eng, group, n, length):
    rng = random.Random(n * 7 + length + group)
    priv = sb(rng.randrange(R))
    pub = pub_batch(eng, group, [int.from_bytes(priv, "big")])[0]
    assert pub == eb.public(group, priv)
    rs = [sb(rng.randrange(R)) for _ in range(n)]
    msgs = [rng.randbytes(length) for _ in range(n)]
    cts, st = eng.bls12381_ecies_encrypt(group, [pub] * n, rs, msgs)
    assert st == bytes(n)
    for i in {0, n // 2, n - 1}:                                      # spot checks against the oracle
        assert cts[i] == eb.encrypt(group, pub, rs[i], msgs[i])[1]
    back, st = eng.bls12381_ecies_decrypt(group, priv, cts, length + 16)
    assert st == bytes(n) and back == msgs


@pytest.mark.parametrize("group", GROUPS)
def test_dkg_process_deals(eng, group):
    """64 dealers with t = 22 deal 32-byte big-endian shares to node nidx, whose key lies in the group (G1: drand's default);
    one share is wrong and one ciphertext tampered.  Deals() is one encryption call, ProcessDeals one decryption call plus one
    PubPoly.Check over the dealers' commitments at the single index nidx."""
    rng = random.Random(600 + group)
    m, t, nidx = 64, 22, 9
    priv = sb(rng.randrange(R))
    pub = eb.public(group, priv)
    polys = [[rng.randrange(R) for _ in range(t)] for _ in range(m)]
    gen = bls.g1_to_affine_bytes(bls.G1) if group == 1 else bls.g2_to_affine_bytes(bls.G2)
    mul = eng.bls12381_g1_mul_batch_affine if group == 1 else eng.bls12381_g2_mul_batch_affine
    commits = mul(b"".join(sb(a) for f in polys for a in f), gen * (m * t))    # C_jk = a_jk G, operand form
    x = nidx + 1
    shares = [sum(a * pow(x, k, R) for k, a in enumerate(f)) % R for f in polys]
    shares[7] = (shares[7] + 1) % R                                  # a dealer that deals a wrong share
    plain = [sb(s) for s in shares]
    cts, st = eng.bls12381_ecies_encrypt(group, [pub] * m, [sb(rng.randrange(R)) for _ in range(m)], plain)
    assert st == bytes(m)
    tampered = bytearray(cts[30]); tampered[eb.POINT_LEN[group] + 20] ^= 0x04
    cts[30] = bytes(tampered)
    got, dst = eng.bls12381_ecies_decrypt(group, priv, cts, 48)
    ok = eng.pubpoly_check(f"bls12381_g{group}", commits, t, [[nidx]] * m, b"".join(got))
    verdict = [d == eb.OK and o == 1 for d, o in zip(dst, ok)]
    want = []
    for j in range(m):                                               # the oracle's ProcessDeals, dealer by dealer
        s, msg = eb.decrypt(group, priv, cts[j])
        if s != eb.OK:
            want.append(False)
            continue
        comm = None                                                  # PubPoly.Eval(nidx) = sum_k x^k C_k
        for k in range(t):
            ck = bls.g1_from_affine_bytes(commits[96 * (j * t + k):96 * (j * t + k + 1)]) if group == 1 else \
                bls.g2_from_affine_bytes(commits[192 * (j * t + k):192 * (j * t + k + 1)])
            term = eb.mul(group, pow(x, k, R), ck)
            comm = bls.g1_add(comm, term) if group == 1 else bls.g2_add(comm, term)
        want.append(eb.mul(group, int.from_bytes(msg, "big")) == comm)
    assert verdict == want
    assert [j for j in range(m) if not verdict[j]] == [7, 30]
    assert dst[30] == eb.AUTH and dst[7] == eb.OK
