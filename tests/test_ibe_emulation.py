"""CPU: the IBE device code (kyber_b200/csrc/ibe.cuh) compiled for the host -- the fixed-G2 Miller loop against miller_loop<1>
(both through the final exponentiation), the decrypt-finish and encrypt bodies against oracle/ibe.py (including an H3 that
rejects candidates) and compression round trips through g1/g2_decompress."""
import ctypes
import random
import subprocess

import pytest

from oracle import bls12381 as o
from oracle import ibe
from test_oracle_ibe import multi_iteration_case

import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_ibe.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_ibe") / "libemul_ibe.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    cp, u32, i = ctypes.c_char_p, ctypes.c_uint32, ctypes.c_int
    lib.emul_ibe_pair.argtypes = [cp, cp, i, cp]
    lib.emul_ibe_decrypt_finish.argtypes = [i, cp, cp, cp, cp, u32, cp]
    lib.emul_ibe_encrypt_body.argtypes = [i, cp, cp, u32, cp, cp, cp]
    lib.emul_ibe_recompress.argtypes = [i, cp, cp]
    return lib


def _pair(lib, p, q, fixed):
    out = ctypes.create_string_buffer(576)
    lib.emul_ibe_pair(o.g1_to_affine_bytes(p), o.g2_to_affine_bytes(q), fixed, out)
    return out.raw


def test_fixed_q_miller_loop_matches_miller_loop(lib):
    rng = random.Random(1)
    q = o.g2_mul(rng.randrange(1, o.R))
    cases = [(o.g1_mul(rng.randrange(1, o.R)), q) for _ in range(3)]
    cases += [(o.G1, o.G2), (None, q), (o.g1_mul(5), None)]
    for p, qq in cases:
        got = _pair(lib, p, qq, 1)
        assert got == _pair(lib, p, qq, 0)
        assert got == o.gt_to_bytes(o.pairing_reference(p, qq))


def _finish(lib, group, gt, u, v, w):
    msg = ctypes.create_string_buffer(max(len(w), 1))
    st = lib.emul_ibe_decrypt_finish(group, gt, u, v, w, len(w), msg)
    return msg.raw[:len(w)], st


@pytest.mark.parametrize("group", [1, 2])
def test_finish_and_encrypt_bodies_match_the_oracle(lib, group):
    rng = random.Random(10 + group)
    ident = b"emul"
    master, priv = ibe.keypair(group, rng.randrange(1, o.R), ident)
    key = (o.g2_decompress if group == 1 else o.g1_decompress)(priv)
    s3, m3, it = multi_iteration_case()
    assert it >= 2
    cases = [(b"", b""), (rng.randbytes(1), rng.randbytes(1)), (rng.randbytes(32), rng.randbytes(32)), (m3, s3)]
    ub = 48 * group
    for msg, sigma in cases:
        U, V, W = (ibe.encrypt_cca_g1 if group == 1 else ibe.encrypt_cca_g2)(master, ident, msg, sigma)
        u, r, w = ctypes.create_string_buffer(ub), ctypes.create_string_buffer(32), ctypes.create_string_buffer(max(len(msg), 1))
        assert lib.emul_ibe_encrypt_body(group, msg, sigma, len(msg), u, r, w) == 1
        assert u.raw == U and w.raw[:len(msg)] == W
        assert int.from_bytes(r.raw, "big") == ibe.h3(sigma, msg)
        Up = (o.g1_decompress if group == 1 else o.g2_decompress)(U)
        gt = o.gt_to_bytes(ibe.pair(Up, key) if group == 1 else ibe.pair(key, Up))
        assert _finish(lib, group, gt, U, V, W) == (msg, ibe.OK)
        if msg:
            bad = bytes([V[0] ^ 1]) + V[1:]
            assert _finish(lib, group, gt, U, bad, W) == (bytes(len(msg)), ibe.PROOF)
    assert _finish(lib, group, bytes(576), bytes(ub), b"ab", b"cd") == (bytes(2), ibe.POINT)


@pytest.mark.parametrize("group", [1, 2])
def test_compression_round_trips(lib, group):
    rng = random.Random(20 + group)
    pts = [None] + [(o.g1_mul if group == 1 else o.g2_mul)(rng.randrange(1, o.R)) for _ in range(8)]
    for p in pts:
        c = o.g1_compress(p) if group == 1 else o.g2_compress(p)
        out = ctypes.create_string_buffer(48 * group)
        assert lib.emul_ibe_recompress(group, c, out) == 1
        assert out.raw == c
