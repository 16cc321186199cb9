"""CPU tests of the MSM's bucket sort (kyber_b200/csrc/msm_sort.cuh): the digit columns and histogram of the point-load pass, the
coarse partition and the bin sort, run block by block with the device bodies compiled for the host
(tests/host_emul/emul_msm_sort.cpp), against the plain counting sort: the same bucket offsets and, in every bucket, the same
multiset of (index | sign) entries."""
import ctypes
import os
import random
import subprocess

import pytest

import msm_cases as mc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")

WINDOWS = (4, 5, 7, 12, 16)


@pytest.fixture(scope="module")
def lib():
    src = os.path.join(EMU, "emul_msm_sort.cpp")
    so = os.path.join(EMU, "libemul_msm_sort.so")
    newest = max([os.path.getmtime(src)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cuh")])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", src, "-o", so],
                       check=True)
    return ctypes.CDLL(so)


def _check(lib, scalars, c, bits):
    stats = (ctypes.c_uint64 * 4)()
    rc = lib.emul_msm_sort_check(ctypes.c_size_t(len(scalars)), mc.scalars_to_bytes(scalars), c, bits, stats)
    assert rc == 0, (c, bits, len(scalars), rc)
    return list(stats)


G = mc.GROUPS["bls12381_g1"]


@pytest.mark.parametrize("c", WINDOWS)
@pytest.mark.parametrize("name", mc.SETS)
@pytest.mark.parametrize("n", (1, 127, 2000))
def test_sort_matches_counting_sort(lib, name, n, c):
    if name == "plus_minus" and n % 2:
        n += 1
    _, s = mc.build_set(G, name, n, mc.multipliers(G, 16))
    _check(lib, s, c, G.scalar_bits)


@pytest.mark.parametrize("c", WINDOWS)
@pytest.mark.parametrize("name", ("uniform", "equal", "bdn128"))
def test_sort_matches_counting_sort_2p16(lib, name, c):
    """2^16 pairs: 16 partition tiles and, at c = 16, bin-sort tiles inside coarse bins; the equal set puts every entry of a
    window into one bucket (a bin 2^16 entries deep), the 128-bit factors crowd the lower windows"""
    _, s = mc.build_set(G, name, 1 << 16, mc.multipliers(G, 16))
    entries, big, mean, _ = _check(lib, s, c, G.scalar_bits)
    if name == "equal":
        assert big == 1 << 16


def test_sort_bin_far_above_average(lib):
    """one coarse bin holds half of all entries, the rest spread thin: the hot bin spans many bin-sort tiles that share its
    buckets, and the sparse tiles cross many bins (buckets past the shared slots reserve one by one)"""
    rng = random.Random(5)
    n = 3 * (1 << 14)
    hot = rng.randrange(G.r)
    s = [hot if i % 2 == 0 else rng.randrange(G.r) for i in range(n)]
    entries, big, mean, _ = _check(lib, s, 16, G.scalar_bits)
    assert big > 8 * mean


def test_sort_sparse_tiles_reserve_past_the_slots(lib):
    """few pairs under a wide window: a bin-sort tile spans every window, so most buckets lie past its shared slots"""
    rng = random.Random(9)
    s = [rng.randrange(G.r) for _ in range(300)]
    _, _, _, spill = _check(lib, s, 16, G.scalar_bits)
    assert spill > 0


@pytest.mark.parametrize("bits", (127, 254, 256))
def test_sort_other_scalar_widths(lib, bits):
    """the GLV halves of BLS12-381 G1 (127 bits) and the bn254 / bn256 orders (254, 256 bits: the top carry window at c = 4)"""
    rng = random.Random(bits)
    s = [rng.randrange(1 << bits) for _ in range(3000)] + [(1 << bits) - 1] * 50
    for c in WINDOWS:
        _check(lib, s, c, bits)
