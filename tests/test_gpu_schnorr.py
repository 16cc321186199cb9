"""GPU: batched sign/schnorr verification over BLS12-381 keys on G1 and G2 (b2k_bls12381_g{1,2}_schnorr_verify / _dev,
k_schnorr_verify) returns, for every signature, the first failing check of schnorr.VerifyWithChecks -- checked against the
oracle (tests/schnorr_oracle.py) on every shared case, in mixed batches, and at 2^16 signatures.  On edwards25519, the
existing b2k_ed25519_verify is the device path of sign/schnorr: its statuses are checked against the Schnorr oracle."""
import hashlib
import struct

import pytest

from oracle import bls12381 as bls
from oracle import eddsa as oe
import schnorr_cases as cases
import schnorr_oracle as so

pytestmark = pytest.mark.gpu
PL = so.POINT_LEN


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def expected():
    return {g: [(name, pk, m, s, so.verify_with_checks(g, pk, m, s)) for name, pk, m, s in cases.cases(g)] for g in so.GROUPS}


def _run(eng, group, items):
    return list(eng.schnorr_verify(group, b"".join(c[1] for c in items), [c[2] for c in items], b"".join(c[3] for c in items)))


def _run_dev(eng, group, items):
    import torch
    n = len(items)
    blob, offs = eng._pack_msgs([c[2] for c in items])
    dev = lambda b: torch.frombuffer(bytearray(b) or bytearray(1), dtype=torch.uint8).cuda()
    d_pk, d_msg, d_off = dev(b"".join(c[1] for c in items)), dev(blob), dev(offs)
    d_sig = dev(b"".join(c[3] for c in items))
    d_st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.schnorr_verify_dev(group, n, d_pk.data_ptr(), d_msg.data_ptr(), d_off.data_ptr(), d_sig.data_ptr(), d_st.data_ptr())
    eng.synchronize()
    return list(bytes(d_st.cpu().numpy()))


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_every_case_host_and_dev_in_one_batch_and_one_by_one(eng, expected, group):
    items = expected[group]
    want = [c[4] for c in items]
    assert set(want) == {0, 1, 2, 3, 4}
    for got in (_run(eng, group, items), _run_dev(eng, group, items)):
        for (name, *_), g, w in zip(items, got, want):
            assert g == w, (group, name, g, w)
    for name, pk, m, s, w in items:
        assert _run(eng, group, [(name, pk, m, s)]) == [w], (group, name)


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_mixed_batches_of_statuses_and_lengths(eng, expected, group):
    import random
    rng = random.Random(11)
    items = expected[group]
    for size in (3, 127, 128, 129, 1000):
        batch = [rng.choice(items) for _ in range(size)]
        assert _run(eng, group, batch) == [c[4] for c in batch], (group, size)


def _base(group, count):
    """count distinct valid (pk, 32-byte msg, sig) over 8 keys"""
    out = []
    for i in range(count):
        x = int.from_bytes(hashlib.sha256(b"key %d" % (i % 8)).digest(), "big") % bls.R
        m = hashlib.sha256(b"bundle %d" % i).digest()
        k = int.from_bytes(hashlib.sha256(b"nonce %d" % i).digest(), "big") % bls.R
        out.append((so.public_key(group, x), m, so.sign(group, x, m, k)))
    return out


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_2_16_signatures_with_corruptions_at_known_positions(eng, group):
    n, pl = 1 << 16, PL[group]
    base = _base(group, 64)
    pks = bytearray(b"".join(c[0] for c in base) * (n // 64))
    msgs = [c[1] for c in base] * (n // 64)
    sigs = bytearray(b"".join(c[2] for c in base) * (n // 64))
    bad_point = bytes([0xE0]) + bytes(pl - 1)
    where = {0: "msg", 63: "s", 64: "R", 65: "pk", 4095: "s+r", n // 2 + 7: "R", n - 33: "pk", n - 1: "msg"}
    want = {}
    for i, kind in where.items():
        pk, m, s = bytes(pks[pl * i:pl * (i + 1)]), msgs[i], bytes(sigs[(pl + 32) * i:(pl + 32) * (i + 1)])
        if kind == "msg":
            m = bytes([m[0] ^ 1]) + m[1:]
        elif kind == "s":
            s = s[:pl] + ((int.from_bytes(s[pl:], "big") + 1) % bls.R).to_bytes(32, "big")
        elif kind == "s+r":
            s = s[:pl] + (int.from_bytes(s[pl:], "big") + bls.R).to_bytes(32, "big")
        elif kind == "R":
            s = bad_point + s[pl:]
        else:
            pk = bad_point
        pks[pl * i:pl * (i + 1)], msgs[i], sigs[(pl + 32) * i:(pl + 32) * (i + 1)] = pk, m, s
        want[i] = so.verify_with_checks(group, pk, m, s)
    assert sorted(set(want.values())) == [1, 2, 3, 4]
    items = [(None, bytes(pks[pl * i:pl * (i + 1)]), msgs[i], bytes(sigs[(pl + 32) * i:(pl + 32) * (i + 1)])) for i in range(n)]
    for got in (_run(eng, group, items), _run_dev(eng, group, items)):
        assert {i: g for i, g in enumerate(got) if g != 0} == want


def test_ed25519_verify_is_the_schnorr_path_on_edwards25519(eng, expected):
    """status 0 <=> Schnorr OK, 8 <=> Schnorr invalid, 1-7 only where Schnorr fails before the equation: the mapping the
    edwards25519 Go adapter applies"""
    items = expected["ed25519"]
    got = list(eng.ed25519_verify(b"".join(c[1] for c in items), [c[2] for c in items], b"".join(c[3] for c in items)))
    seen = set()
    for (name, *_, want), g in zip(items, got):
        seen.add(g)
        assert (g == oe.OK) == (want == oe.OK), name
        assert (g == oe.NOT_EQUAL) == (want == oe.NOT_EQUAL), name
        if g not in (oe.OK, oe.NOT_EQUAL):
            assert so.fails_before_equation("ed25519", want), name
    assert {0, 8} <= seen and len(seen - {0, 8}) >= 4


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_refusals_then_a_correct_call(eng, expected, group):
    from kyber_b200.capi import ERR_ARG, _buf
    name, pk, msg, sig, _ = expected[group][2]
    lib, h = eng.lib, eng.h
    host, dev = getattr(lib, f"b2k_{group}_schnorr_verify"), getattr(lib, f"b2k_{group}_schnorr_verify_dev")
    st = bytearray(2)
    blob, offs = eng._pack_msgs([msg, msg])
    bufs = [_buf(x) for x in (pk * 2, blob, offs, sig * 2, st)]
    p = [b[0] for b in bufs]
    assert host(h, 0, *p) == ERR_ARG
    pd, kd = _buf(struct.pack("<3I", 0, 1, 0))
    assert host(h, 2, p[0], p[1], pd, p[3], p[4]) == ERR_ARG
    assert host(h, 2, p[0], p[1], p[2], None, p[4]) == ERR_ARG
    assert host(h, 2, None, p[1], p[2], p[3], p[4]) == ERR_ARG
    assert dev(h, 2, p[0], p[1], p[2], p[3], None) == ERR_ARG
    assert dev(h, 0, p[0], p[1], p[2], p[3], p[4]) == ERR_ARG
    assert host(h, 2, *p) == 0 and bytes(st) == b"\x00\x00"
