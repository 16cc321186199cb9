"""CPU: the sign/bdn masked-sum bodies (kyber_b200/csrc/bdn.cuh) compiled for the host on BLS12-381 G1 and checked against the
plain masked sum of tests/bdn_cases.py -- empty, single-bit and full masks, popcount exactly n/2 and n/2 + 1, bits beyond n,
duplicate keys, a key with its negation, an infinity term, and rosters that are not multiples of 8 or of a 1024-member slice."""
import ctypes
import os
import random
import subprocess

import pytest

import bdn_cases as bc
from oracle import bls12381 as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_bdn.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_bdn") / "libemul_bdn.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    u32, cp = ctypes.c_uint32, ctypes.c_char_p
    lib.emul_bdn_aggregate.argtypes = [u32, cp, u32, cp, cp, cp]
    lib.emul_bdn_aggregate.restype = ctypes.c_int
    return lib


def _enc(p) -> bytes:
    return bytes(96) if p is None else p[0].to_bytes(48, "big") + p[1].to_bytes(48, "big")


def _roster(n: int, rng: random.Random):
    """random multiples of the base, with a duplicate, a key next to its negation and an infinity term"""
    step = o.g1_mul(rng.randrange(1, o.R))
    pts, acc = [], None
    for i in range(n):
        acc = o.g1_add(acc, step) if i % 5 else o.g1_mul(rng.randrange(1, o.R))
        pts.append(acc)
    if n >= 8:
        pts[2] = pts[1]
        pts[4] = o.g1_neg(pts[3])
        pts[6] = None
    return pts


def _run(lib, pts, masks):
    n, m = len(pts), len(masks)
    out, comp = ctypes.create_string_buffer(96 * m), ctypes.create_string_buffer(m)
    assert lib.emul_bdn_aggregate(n, b"".join(_enc(p) for p in pts), m, b"".join(masks), out, comp) == 0
    return [out.raw[96 * k:96 * k + 96] for k in range(m)], list(comp.raw)


@pytest.mark.parametrize("n", [1, 7, 8, 13, 64, 100, 1023, 1025])
def test_masked_sums_against_the_plain_sum(lib, n):
    rng = random.Random(n)
    pts = _roster(n, rng)
    masks = [bc.mask_of(n, []), bc.mask_of(n, range(n))] + bc.edge_masks(n, rng) + bc.random_masks(n, 12, rng)
    if n >= 8:
        masks += [bc.mask_of(n, [1, 2]), bc.mask_of(n, [3, 4]), bc.mask_of(n, [6]), bc.mask_of(n, [0, 1, 2, 3, 4, 5, 6])]
    got, comp = _run(lib, pts, masks)
    for k, mk in enumerate(masks):
        assert got[k] == _enc(bc.aggregate_public_keys(pts, mk, n, o.g1_add)), k
        pop = sum(bc.bit(mk, i) for i in range(n))
        assert comp[k] == (1 if 2 * pop > n else 0), k


def test_complement_threshold_and_ignored_bits(lib):
    n = 13
    rng = random.Random(3)
    pts = _roster(n, rng)
    half = bc.mask_of(n, range(6))                    # popcount 6 = floor(n/2): summed directly
    over = bc.mask_of(n, range(7))                    # 7 > n/2: through the complement
    junk = bytearray(over)
    junk[-1] |= 0xE0                                  # bits 13..15 lie beyond n
    got, comp = _run(lib, pts, [half, over, bytes(junk)])
    assert comp == [0, 1, 1]
    assert got[1] == got[2] == _enc(bc.aggregate_public_keys(pts, over, n, o.g1_add))
    even = _roster(12, rng)
    got, comp = _run(lib, even, [bc.mask_of(12, range(6)), bc.mask_of(12, range(7))])
    assert comp == [0, 1]                             # exactly n/2 direct, n/2 + 1 complemented
    assert got[0] == _enc(bc.aggregate_public_keys(even, bc.mask_of(12, range(6)), 12, o.g1_add))
    assert got[1] == _enc(bc.aggregate_public_keys(even, bc.mask_of(12, range(7)), 12, o.g1_add))


def test_malformed_term_is_refused(lib):
    pts = _roster(9, random.Random(4))
    blob = bytearray(b"".join(_enc(p) for p in pts))
    blob[96 + 95] ^= 1
    out, comp = ctypes.create_string_buffer(96), ctypes.create_string_buffer(1)
    assert lib.emul_bdn_aggregate(9, bytes(blob), 1, bc.mask_of(9, [0]), out, comp) == -1
