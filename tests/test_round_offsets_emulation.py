"""CPU tests of the MSM's affine pair-tree rounds with every round's bucket offsets taken from ONE multi-column scan of the
histogram (kernels.cuh: k_scan_*, column y = ceil(counts / 2^y); msm_host.cuh enqueues no count or scan per round): the scan
columns equal the offsets that halving every bucket round by round gives, and the whole MSM on them matches the oracle
(tests/host_emul/emul_round_offsets.cpp, the device bodies compiled for the host)."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import bls12381 as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")


@pytest.fixture(scope="module")
def lib():
    src = os.path.join(EMU, "emul_round_offsets.cpp")
    so = os.path.join(EMU, "libemul_round_offsets.so")
    newest = max([os.path.getmtime(src)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cuh")])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", src, "-o", so],
                       check=True)
    return ctypes.CDLL(so)


def _halving_offsets(counts, rounds):
    """the offsets of round 1..R as the rounds produce them: every bucket of k operands keeps ceil(k / 2) per round"""
    cols, cur = [], list(counts)
    for _ in range(rounds):
        cur = [(k + 1) // 2 for k in cur]
        offs, run = [], 0
        for k in cur:
            offs.append(run)
            run += k
        cols.append(offs + [run])
    return cols


@pytest.mark.parametrize("total,rounds", [(1, 1), (1000, 3), (1024, 2), (3000, 8), (4097, 5)])
def test_scan_columns_equal_round_by_round_halving(lib, total, rounds):
    rng = random.Random(total * 31 + rounds)
    counts = [rng.choice([0, 1, 2, 3, 255, 256, 257, rng.randrange(1 << 12), rng.randrange(1 << 24)]) for _ in range(total)]
    out = (ctypes.c_uint32 * ((rounds + 1) * (total + 1)))()
    lib.emul_scan_columns((ctypes.c_uint32 * total)(*counts), ctypes.c_uint32(total), rounds, out)
    cols = [list(out[y * (total + 1):(y + 1) * (total + 1)]) for y in range(rounds + 1)]
    run, col0 = 0, []
    for k in counts:
        col0.append(run)
        run += k
    assert cols[0] == col0 + [run]
    assert cols[1:] == _halving_offsets(counts, rounds)


def test_msm_on_precomputed_round_offsets(lib):
    """split rounds (forward / invert / backward, plain and cp.async-staged) on the offsets of the one scan give the oracle's MSM,
    including repeated points in one bucket, P and -P, operands at infinity and all-equal scalars, over several R and batch widths"""
    rng = random.Random(23)
    n = 48
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[5] = None
    pts[6] = pts[7] = pts[8] = pts[9]
    pts[10] = o.g1_neg(pts[11])
    pts[13] = (0, 2)
    pts[14] = (0, o.P - 2)
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    sets = ([rng.randrange(o.R) for _ in range(n)], [0x123456789ABCDEF] * n, [rng.randrange(1 << 9) for _ in range(n)])
    for ks in sets:
        sb = b"".join(o.scalar_to_bytes(k) for k in ks)
        want = o.g1_compress(o.g1_msm(ks, pts))
        for c, m, L, rounds, pbatch in ((4, 2, 3, 1, 3), (4, 2, 2, 2, 9), (5, 4, 4, 3, 24), (8, 8, 5, 6, 192), (3, 2, 1, 8, 15), (4, 2, 3, 0, 1)):
            for staged in (0, 1):
                o48 = ctypes.create_string_buffer(48)
                rc = lib.emul_bls12381_g1_msm_affine_onescan(ctypes.c_size_t(n), sb, pb, c, m, L, rounds, pbatch, staged, o48)
                assert rc == 0 and o48.raw == want, (c, m, L, rounds, pbatch, staged)
