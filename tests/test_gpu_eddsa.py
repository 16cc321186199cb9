"""GPU: batched Ed25519 verification (b2k_ed25519_verify / _dev, k_ed25519_verify) returns, for every signature, the code of
the first failing check of eddsa.VerifyWithChecks -- checked against the oracle (oracle/eddsa.py) on the reference's
fixtures, on crafted cases for every rejection path, on the cofactorless equation, around the SHA-512 padding and at scale."""
import ctypes
import os
import struct
import subprocess

import pytest

from oracle import eddsa as oe
import eddsa_cases as cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fixture_cases():
    """every fixture with a 32-byte key and a 64-byte signature (other lengths are the caller's checks)"""
    items = [("rfc%d" % i, pk, m, s) for i, (_, pk, m, s) in enumerate(cases.rfc8032())]
    items += [("sign.input %d" % i, pk, m, s) for i, (_, pk, m, s) in enumerate(cases.sign_input())]
    items += [("wycheproof %d" % tc, pk, m, s) for tc, pk, m, s, _ in cases.wycheproof() if len(s) == 64 and len(pk) == 32]
    items += [c[:4] for c in cases.inline()]
    return [(name, pk, m, s, oe.verify_with_checks(pk, m, s)) for name, pk, m, s in items]


def _run(eng, items):
    return list(eng.ed25519_verify(b"".join(c[1] for c in items), [c[2] for c in items], b"".join(c[3] for c in items)))


def _assert_batch_and_single(eng, items):
    got = _run(eng, items)
    for (name, *_, want), g in zip(items, got):
        assert g == want, name
    for name, pk, m, s, want in items:
        assert _run(eng, [(name, pk, m, s)]) == [want], name


def test_fixtures_in_one_batch_and_one_by_one(eng, fixture_cases):
    assert len(fixture_cases) > 1150
    assert sum(c[4] == 0 for c in fixture_cases) >= 1024 + 5 + 80
    _assert_batch_and_single(eng, fixture_cases)


def test_inline_vectors_give_their_expected_errors(eng):
    name_to_code = {v: k for k, v in oe.ERR_NAMES.items()}
    inl = cases.inline()
    got = _run(eng, [c[:4] for c in inl])
    assert got == [name_to_code[c[4]] for c in inl]


def test_crafted_cases(eng):
    items = [(n, pk, m, s, oe.verify_with_checks(pk, m, s)) for n, pk, m, s in cases.crafted()]
    expect_prefix = {"s + l": 1, "s bit 255": 1, "s = l": 1, "s = l - 1": 8, "R non-canonical": 2, "R no sqrt": 3,
                     "R small order": 4, "pk non-canonical": 5, "pk no sqrt": 6, "pk small order": 7, "msg bit": 8,
                     "valid": 0, "empty message": 0}
    for name, *_, want in items:             # the oracle's code is the category the case was built for
        for pre, code in expect_prefix.items():
            if name == pre or (name.startswith(pre + " ") and name[len(pre) + 1:].isdigit()):
                assert want == code, name
    assert {c[4] for c in items} == set(range(9))
    _assert_batch_and_single(eng, items)


def test_cofactorless_equation(eng):
    cc = cases.cofactor_cases()
    got = _run(eng, [c[:4] for c in cc])
    assert any(h8 == 0 for *_, h8 in cc) and sum(h8 != 0 for *_, h8 in cc) >= 8
    assert got == [0 if h8 == 0 else 8 for *_, h8 in cc]


def test_message_lengths_around_the_padding(eng):
    items = [(n, pk, m, s, 0) for n, pk, m, s in cases.lengths_cases()]
    flipped = [(n + " flipped", pk, m[:-1] + bytes([m[-1] ^ 1]), s, 8) for n, pk, m, s, _ in items]
    _assert_batch_and_single(eng, items + flipped)


def _distinct_signatures(count):
    """count distinct (pk, 32-byte msg, sig), signed by libsodium where PyNaCl is importable, else by the oracle"""
    import hashlib
    out = []
    try:
        import nacl.signing
        for i in range(count):
            seed = hashlib.sha256(b"scale seed %d" % (i % 64)).digest()
            msg = hashlib.sha256(b"scale msg %d" % i).digest()
            k = nacl.signing.SigningKey(seed)
            out.append((bytes(k.verify_key), msg, k.sign(msg).signature))
    except ImportError:
        for i in range(count):
            seed = hashlib.sha256(b"scale seed %d" % (i % 64)).digest()
            msg = hashlib.sha256(b"scale msg %d" % i).digest()
            out.append((oe.keygen(seed)[2], msg, oe.sign(seed, msg)))
    return out


@pytest.fixture(scope="module")
def base4096():
    base = _distinct_signatures(4096)
    for pk, m, s in base[:8]:
        assert oe.verify_with_checks(pk, m, s) == 0
    return base


def _corrupt(pk, m, s, kind):
    if kind == "msg":
        return pk, bytes([m[0] ^ 1]) + m[1:], s
    if kind == "s":
        return pk, m, s[:32] + (int.from_bytes(s[32:], "little") + oe.L).to_bytes(32, "little")
    if kind == "R":
        return pk, m, b"\xee" + b"\xff" * 30 + b"\x7f" + s[32:]
    return b"\x01" + b"\x00" * 31, m, s                          # small-order key


@pytest.mark.parametrize("n", [1 << 16, 1 << 20])
def test_scale_with_corruptions_host_and_dev(eng, base4096, n):
    import torch
    pks = bytearray(b"".join(c[0] for c in base4096) * (n // 4096))
    msgs = [c[1] for c in base4096] * (n // 4096)
    sigs = bytearray(b"".join(c[2] for c in base4096) * (n // 4096))
    kinds = ["msg", "s", "R", "pk"]
    where = {0: "msg", 31: "s", 32: "R", 33: "pk", 4095: "msg", 4096: "s", n // 2 + 7: "R", n - 33: "pk", n - 1: "msg"}
    want = {}
    for i, kind in where.items():
        pk, m, s = _corrupt(pks[32 * i:32 * i + 32], msgs[i], sigs[64 * i:64 * i + 64], kind)
        pks[32 * i:32 * i + 32], msgs[i], sigs[64 * i:64 * i + 64] = pk, m, s
        want[i] = oe.verify_with_checks(bytes(pk), m, bytes(s))
    assert sorted(set(want.values())) == [1, 2, 7, 8] and set(kinds) == set(where.values())
    got = eng.ed25519_verify(bytes(pks), msgs, bytes(sigs))
    bad = {i: got[i] for i in range(n) if got[i] != 0}
    assert bad == want
    # the device-pointer form on the same inputs
    blob, offs = eng._pack_msgs(msgs)
    dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    d_pk, d_msg, d_off, d_sig = dev(pks), dev(blob), dev(offs), dev(sigs)
    d_st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.ed25519_verify_dev(n, d_pk.data_ptr(), d_msg.data_ptr(), d_off.data_ptr(), d_sig.data_ptr(), d_st.data_ptr())
    eng.synchronize()
    assert bytes(d_st.cpu().numpy()) == got


def test_refusals_then_a_correct_call(eng):
    from kyber_b200.capi import ERR_ARG, _buf
    _, pk, msg, sig = cases.rfc8032()[1]
    lib, h = eng.lib, eng.h
    st = bytearray(2)
    blob, offs = eng._pack_msgs([msg, msg])
    bufs = [_buf(x) for x in (pk * 2, blob, offs, sig * 2, st)]
    p = [b[0] for b in bufs]
    assert lib.b2k_ed25519_verify(h, 0, *p) == ERR_ARG
    dec = struct.pack("<3I", 0, 1, 0)
    pd, kd = _buf(dec)
    assert lib.b2k_ed25519_verify(h, 2, p[0], p[1], pd, p[3], p[4]) == ERR_ARG
    assert lib.b2k_ed25519_verify(h, 2, p[0], p[1], p[2], None, p[4]) == ERR_ARG
    assert lib.b2k_ed25519_verify_dev(h, 2, p[0], p[1], p[2], p[3], None) == ERR_ARG
    assert lib.b2k_ed25519_verify_dev(h, 0, p[0], p[1], p[2], p[3], p[4]) == ERR_ARG
    assert lib.b2k_ed25519_verify(h, 2, *p) == 0 and bytes(st) == b"\x00\x00"


def test_cpp_mirror_verify_batch(tmp_path):
    exe = str(tmp_path / "test_eddsa")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "test_eddsa.cpp"), "-o", exe,
                    "-L" + os.path.join(ROOT, "kyber_b200"), "-lb2kyber", "-Wl,-rpath," + os.path.join(ROOT, "kyber_b200"),
                    "-L/usr/local/cuda/lib64", "-lcudart"], check=True)
    rfc = [(pk, m, s, 0) for _, pk, m, s in cases.rfc8032()]
    _, pk, m, s = cases.rfc8032()[2]
    rfc.append((pk, bytes([m[0] ^ 1]) + m[1:], s, 8))
    path = tmp_path / "cases.txt"
    path.write_text("".join("%s %s %s %d\n" % (pk.hex(), m.hex() or "-", s.hex(), c) for pk, m, s, c in rfc))
    r = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PASSED" in r.stdout and r.stdout.count("ok ") == len(rfc) + 1
