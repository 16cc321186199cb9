"""CPU: ECIES's device bodies (kyber_b200/csrc/ecies.cuh) compiled for the host and checked against the restatement in
oracle/ecies.py -- the AES-256 block, GCM Seal and Open across block edges, HKDF, both constant-time multiplications against
point_mul (top-bit scalars, the identity, small-order points, all-zero bytes), whole encryptions and decryptions, and the
operation counts of the constant-time helpers, which must not depend on the key, r, the point or the message."""
import ctypes
import os
import random
import subprocess
import sys

import pytest

import ed25519_msm_cases as mc
from oracle import ecies as ec
from oracle import ed25519 as ed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_ecies.cpp")
LENGTHS = [0, 1, 15, 16, 17, 31, 32, 33, 4096]
IDENT = ed.encode(ed.IDENT)
T8 = mc.T8                                                  # a point of order 8


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("emul_ecies")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_ecies_table
    gen_ecies_table.main(str(d / "ecies_base_comb.inc"))       # the table build() generates, for a tree not built yet
    so = str(d / "libemul_ecies.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", "-I", str(d), SRC,
                    "-o", so], check=True)
    lib = ctypes.CDLL(so)
    u32, sz, cp = ctypes.c_uint32, ctypes.c_size_t, ctypes.c_char_p
    lib.emul_counts.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.emul_aes256.argtypes = [cp] * 3
    lib.emul_kdf.argtypes = [cp, cp]
    lib.emul_gcm_seal.argtypes = [cp, cp, u32, cp]
    lib.emul_gcm_open.argtypes = [cp, cp, u32, cp]
    lib.emul_mul_var.argtypes = [cp] * 3
    lib.emul_mul_base.argtypes = [cp] * 2
    lib.emul_decrypt.argtypes = [cp, sz, u32, cp, cp, cp]
    lib.emul_encrypt.argtypes = [sz, cp, cp, u32, cp, cp, cp]
    return lib


def counts(lib):
    c = (ctypes.c_uint64 * 4)()
    lib.emul_counts(c, 1)
    return tuple(c)


def decrypt(lib, priv, cts, clen):
    n = len(cts)
    msg, st = ctypes.create_string_buffer(max(n * (clen - 16), 1)), ctypes.create_string_buffer(n)
    lib.emul_decrypt(priv, n, clen, b"".join(cts), msg, st)
    w = clen - 16
    return [(st.raw[i], msg.raw[w * i:w * i + w]) for i in range(n)]


def encrypt(lib, pubs, rs, msgs):
    n, ln = len(msgs), len(msgs[0])
    out, st = ctypes.create_string_buffer(max(n * (ln + 48), 1)), ctypes.create_string_buffer(n)
    lib.emul_encrypt(n, b"".join(pubs), b"".join(rs), ln, b"".join(msgs) or b"\x00", out, st)
    w = ln + 48
    return [(st.raw[i], out.raw[w * i:w * i + w]) for i in range(n)]


def test_aes256_block(lib):
    out = ctypes.create_string_buffer(16)
    lib.emul_aes256(bytes(range(32)), bytes.fromhex("00112233445566778899aabbccddeeff"), out)
    assert out.raw == bytes.fromhex("8ea2b7ca516745bfeafc49904b496089")
    rng = random.Random(1)
    for _ in range(20):
        key, blk = rng.randbytes(32), rng.randbytes(16)
        lib.emul_aes256(key, blk, out)
        assert out.raw == ec.aes256_encrypt_block(key, blk)


def test_hkdf(lib):
    rng = random.Random(2)
    out = ctypes.create_string_buffer(44)
    for dh in [bytes(32), b"\xff" * 32] + [rng.randbytes(32) for _ in range(10)]:
        lib.emul_kdf(dh, out)
        assert out.raw == ec.hkdf_sha256(dh, 44)


@pytest.mark.parametrize("n", LENGTHS)
def test_gcm_seal_and_open(lib, n):
    rng = random.Random(100 + n)
    k44, msg = rng.randbytes(44), rng.randbytes(n)
    out = ctypes.create_string_buffer(n + 16)
    lib.emul_gcm_seal(k44, msg, n, out)
    assert out.raw == ec.gcm_seal(k44[:32], k44[32:], msg)
    back = ctypes.create_string_buffer(max(n, 1))
    assert lib.emul_gcm_open(k44, out.raw, n + 16, back) == 1 and back.raw[:n] == msg
    for pos in {0, n // 2, n + 15}:
        bad = bytearray(out.raw)
        bad[pos] ^= 0x01
        back = ctypes.create_string_buffer(b"\xaa" * max(n, 1))
        assert lib.emul_gcm_open(k44, bytes(bad), n + 16, back) == 0
        assert back.raw[:n] == bytes(n)


def scalars(rng):
    return [bytes(32), (1).to_bytes(32, "little"), ed.L.to_bytes(32, "little"), b"\xff" * 32, (0x8f << 248).to_bytes(32, "little"),
            (0x80 << 248).to_bytes(32, "little"), ((0x97 << 248) | rng.getrandbits(240)).to_bytes(32, "little")] + \
        [rng.randbytes(32) for _ in range(6)]


def test_multiplications(lib):
    rng = random.Random(3)
    pts = [IDENT, T8, bytes(32), ec.mul(rng.randbytes(32)), ed.encode(ed.add(ed.decode(ec.mul(rng.randbytes(32))), ed.decode(T8)))]
    out = ctypes.create_string_buffer(32)
    for k in scalars(rng):
        lib.emul_mul_base(k, out)
        assert out.raw == ec.mul(k), k.hex()
        for p in pts:
            assert lib.emul_mul_var(k, p, out) == 0
            assert out.raw == ec.mul(k, ed.decode(p)), (k.hex(), p.hex())


def test_decrypt_against_the_oracle(lib):
    rng = random.Random(4)
    priv = rng.randbytes(32)
    pub = ec.mul(priv)
    for n in (0, 32, 33, 1000):
        msgs = [rng.randbytes(n) for _ in range(4)]
        rs = [rng.randbytes(32) for _ in range(4)]
        cts = [ec.encrypt(pub, r, m)[1] for r, m in zip(rs, msgs)]
        bad_r = next(bytes([i]) + bytes(31) for i in range(2, 256) if ed.decode(bytes([i]) + bytes(31)) is None)
        flipped = bytearray(cts[1]); flipped[-1] ^= 0x80
        body = bytearray(cts[2]); body[32] ^= 0x01
        other = ec.mul(rng.randbytes(32)) + cts[3][32:]
        batch = cts + [bad_r + cts[0][32:], bytes(flipped), bytes(body), other, IDENT + cts[0][32:], bytes(32) + cts[0][32:]]
        got = decrypt(lib, priv, batch, n + 16)
        assert got == [ec.decrypt(priv, c) for c in batch]
        assert [g[0] for g in got[:4]] == [ec.OK] * 4 and [g[1] for g in got[:4]] == msgs


def test_encrypt_against_the_oracle(lib):
    rng = random.Random(5)
    for n in (0, 32, 1000):
        pubs = [ec.mul(rng.randbytes(32)) for _ in range(3)] + [IDENT, T8, bytes(32)]
        bad = next(bytes([i]) + bytes(31) for i in range(2, 256) if ed.decode(bytes([i]) + bytes(31)) is None)
        pubs.append(bad)
        rs = [rng.randbytes(32) for _ in pubs[:-2]] + [b"\xff" * 32, rng.randbytes(32)]
        msgs = [rng.randbytes(n) for _ in pubs]
        got = encrypt(lib, pubs, rs, msgs)
        assert got == [ec.encrypt(p, r, m) for p, r, m in zip(pubs, rs, msgs)]


def test_operation_counts_do_not_depend_on_secrets_or_points(lib):
    """every key, r, R and message of one length runs the same number of selections, windows, S-box layers and GHASH blocks"""
    rng = random.Random(6)
    keys = [bytes(32), b"\xff" * 32, (1 << 255).to_bytes(32, "little"), (0x8f << 248).to_bytes(32, "little"), rng.randbytes(32)]
    points = [IDENT, T8, bytes(32), ec.mul(rng.randbytes(32))]
    counts(lib)
    seen = set()
    for k in keys:
        for p in points:
            decrypt(lib, k, [p + rng.randbytes(48)], 48)
            seen.add(("dec", counts(lib)))
            encrypt(lib, [p], [k], [rng.randbytes(32)])
            seen.add(("enc", counts(lib)))
    dec = {c for w, c in seen if w == "dec"}
    enc = {c for w, c in seen if w == "enc"}
    assert len(dec) == 1 and len(enc) == 1, seen
    (d,), (e,) = dec, enc
    assert d[0] == 64 and d[1] == 63 and e[0] == 128 and e[1] == 64     # selections and windows of each multiplication
    assert d[2] == e[2] == 13 + 14 * 2                                   # SubWord x 13, then H with E(J0) and two counter blocks
    assert d[3] == e[3] == 3                                             # 32 bytes: two GHASH blocks and the length block
