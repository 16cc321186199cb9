"""CPU: the edwards25519 MSM and share/poly device code (kyber_b200/csrc/ed_msm.cuh, lagrange.cuh) compiled for the host and
run stage by stage in the order of the kernels of b2k_ed25519_msm.cu -- load and scalar rule, balanced slices with buckets cut
by forced short slices, serial and block-parallel fix-up, chunked reduction, window sums, Horner -- against the oracle."""
import ctypes
import os
import random
import subprocess
import struct

import pytest

from oracle import ed25519 as ed
from oracle import share_poly
import ed25519_msm_cases as cases
from msm_cases import signed_digits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_ed_msm.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_ed_msm") / "libemul_ed_msm.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    lib.emul_ed_load.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_char_p]
    lib.emul_ed_msm.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_uint32,
                                ctypes.c_int, ctypes.c_char_p, ctypes.c_void_p]
    lib.emul_ed_lagrange.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_char_p]
    lib.emul_ed_pubpoly_eval.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    lib.emul_ed_pubpoly_check.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    lib.emul_ed_ge_scalar_mult_base.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
    return lib


WINDOWS = (4, 5, 8, 12, 16)


def _msm(lib, scalars, pts: bytes, c, m, L, serial_max=64):
    out, stats = ctypes.create_string_buffer(32), (ctypes.c_uint32 * 2)()
    bad = lib.emul_ed_msm(len(scalars), cases.le(scalars), pts, c, m, L, serial_max, out, stats)
    return out.raw, bad, (stats[0], stats[1])


@pytest.mark.parametrize("c", WINDOWS)
def test_load_pass_digits_and_niels_form(lib, c):
    rng = random.Random(c)
    W = (256 + c) // c
    ks = cases.crafted_high_scalars(rng) + [rng.getrandbits(256) for _ in range(40)] + [0, (1 << 256) - 1]
    pts = [cases.point(rng.randrange(ed.L), rng.randrange(8)) for _ in range(6)] + [cases.IDENTITY, cases.ZERO, (2).to_bytes(32, "little")]
    for i, k in enumerate(ks):
        p = pts[i % len(pts)]
        digits = (ctypes.c_int16 * W)()
        niels = ctypes.create_string_buffer(96)
        ok = lib.emul_ed_load(k.to_bytes(32, "little"), p, c, digits, niels)
        assert list(digits) == signed_digits(cases.effective_scalar(k), c, 256), (hex(k), c)
        dp = ed.decode(p)
        assert ok == (dp is not None)
        x, y = dp if dp is not None else (0, 1)
        want = b"".join(v.to_bytes(32, "little") for v in ((y + x) % ed.P, (y - x) % ed.P, 2 * ed.D * x * y % ed.P))
        assert niels.raw == want


# (set, n, c, chunk m, slice length L, serial fix-up limit): forced short slices cut buckets; serial_max 2 sends every bucket
# with more than two partials to the block-parallel path
PLANS = [(s, n, c, m, L, sm) for s in cases.SETS for (n, c, m, L, sm) in
         ((2, 4, 1, 1, 64), (300, 5, 4, 3, 64), (300, 8, 16, 7, 2), (700, 12, 64, 5, 2))]
PLANS += [(s, n, 16, 16, L, 64) for s in ("uniform", "equal", "high") for (n, L) in ((1, 4), (1000, 64))]   # c = 16: 2^15 buckets a window


@pytest.mark.parametrize("name,n,c,m,L,smax", PLANS)
def test_msm_matches_the_oracle(lib, name, n, c, m, L, smax):
    if name == "plus_minus" and n % 2:
        n += 1
    scalars, ab = cases.build_set(name, n)
    got, bad, (cut, big) = _msm(lib, scalars, cases.points(ab), c, m, L, smax)
    assert bad == 0
    assert got == cases.msm_expected(scalars, ab), (name, n, c, m, L)
    if name == "equal" and L < 64 and n >= 300:
        assert cut > 0 and (big > 0 or smax == 64)


def test_equal_scalars_take_the_block_parallel_fixup(lib):
    scalars, ab = cases.build_set("equal", 4000)
    got, _, (cut, big) = _msm(lib, scalars, cases.points(ab), 12, 16, 4, 64)
    assert big > 0                                     # 4000 entries / 4 per slice: ~1000 partials in one bucket per window
    assert got == cases.msm_expected(scalars, ab)


def test_undecodable_point_counts_as_identity(lib):
    scalars, ab = cases.build_set("uniform", 50)
    pts = bytearray(cases.points(ab))
    pts[32 * 7:32 * 8] = (2).to_bytes(32, "little")      # y = 2 is not on the curve
    got, bad, _ = _msm(lib, scalars, bytes(pts), 8, 4, 8)
    assert bad == 1
    ab[7] = (0, 0)
    assert got == cases.msm_expected(scalars, ab)


def test_lagrange_weights_mod_l(lib):
    rng = random.Random(5)
    for t in (1, 2, 3, 17, 100):
        idx = rng.sample(range(1 << 20), t - 1) + [0xffffffff]
        out = ctypes.create_string_buffer(32 * t)
        assert lib.emul_ed_lagrange(t, struct.pack("<%dI" % t, *idx), out) == 1
        want = share_poly.lagrange_at_zero(idx, ed.L)
        assert [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(t)] == want
    out = ctypes.create_string_buffer(96)
    assert lib.emul_ed_lagrange(3, struct.pack("<3I", 4, 9, 4), out) == 0


def test_pubpoly_eval_and_check(lib):
    rng = random.Random(9)
    t = 5
    coeffs = [rng.randrange(ed.L) for _ in range(t)]
    commits = b"".join(ed.encode(ed.scalar_mult(a)) for a in coeffs)
    for index in (0, 1, 6, 1000, 0xffffffff):
        x = index + 1
        fx = sum(a * pow(x, j, ed.L) for j, a in enumerate(coeffs)) % ed.L
        out = ctypes.create_string_buffer(32)
        assert lib.emul_ed_pubpoly_eval(t, commits, index, out) == 0
        assert out.raw == ed.encode(ed.scalar_mult(fx))
        assert lib.emul_ed_pubpoly_check(t, commits, index, fx.to_bytes(32, "little")) == 1
        assert lib.emul_ed_pubpoly_check(t, commits, index, ((fx + 1) % ed.L).to_bytes(32, "little")) == 0
        assert lib.emul_ed_pubpoly_check(t, commits, index, (fx + ed.L).to_bytes(32, "little")) == 1   # same point, prime order
    # shares at or above 2^255 are read like geScalarMult reads them
    for k in cases.crafted_high_scalars(rng):
        out = ctypes.create_string_buffer(32)
        lib.emul_ed_ge_scalar_mult_base(k.to_bytes(32, "little"), out)
        assert out.raw == ed.encode(cases.ge_scalar_mult(k.to_bytes(32, "little"), ed.BASE)), hex(k)
