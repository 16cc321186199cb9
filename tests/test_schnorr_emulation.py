"""CPU: the sign/schnorr verification device code (kyber_b200/csrc/schnorr.cuh) compiled for the host and checked against the
oracle (tests/schnorr_oracle.py) -- the same bodies k_schnorr_verify runs, for keys on G1 and on G2.  First the reduction of
the 512-bit big-endian digest mod r on its own, then the whole body on every shared case."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import bls12381 as bls
import schnorr_cases as cases
import schnorr_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_schnorr.cpp")
R = bls.R


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so_path = str(tmp_path_factory.mktemp("emul_schnorr") / "libemul_schnorr.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so_path],
                   check=True)
    lib = ctypes.CDLL(so_path)
    lib.emul_fr_from_be512.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
    lib.emul_schnorr_verify.argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    return lib


def _reduce(lib, x: int) -> int:
    out = ctypes.create_string_buffer(32)
    lib.emul_fr_from_be512(x.to_bytes(64, "big"), out)
    return int.from_bytes(out.raw, "big")


def reduction_inputs() -> list:
    """edge values of hi 2^256 + lo, then random ones with each half below r, in [r, 2r) and in [2r, 2^256)"""
    t = 1 << 256
    xs = [0, 1, (1 << 512) - 1, t - 1, t, t + 1, R - 1, R, R + 1, 2 * R, 3 * R - 1, 3 * R, R * t, (R - 1) * t + R - 1,
          (t - 1) * t + R - 1, (R * t) // R * R, ((1 << 512) - 1) // R * R, ((1 << 512) - 1) // R * R - 1]
    rng = random.Random(5)
    bands = [(0, R), (R, 2 * R), (2 * R, t)]
    for lo_band in bands:
        for hi_band in bands:
            for _ in range(20):
                xs.append(rng.randrange(*hi_band) * t + rng.randrange(*lo_band))
    return xs


def test_reduction_mod_r_against_python_integers(lib):
    for x in reduction_inputs():
        assert _reduce(lib, x) == x % R, hex(x)
    for x in reduction_inputs():
        assert _reduce(lib, x) == so.reduce_be(x.to_bytes(64, "big"))


@pytest.mark.parametrize("group", cases.BLS_GROUPS)
def test_verify_matches_the_oracle_on_every_case(lib, group):
    g2 = int(group == "bls12381_g2")
    got = {}
    for name, pk, msg, sig in cases.cases(group):
        want = so.verify_with_checks(group, pk, msg, sig)
        got[name] = lib.emul_schnorr_verify(g2, pk, msg, len(msg), sig)
        assert got[name] == want, (group, name)
    assert set(got.values()) == {so.OK, so.R_BAD, so.S_BAD, so.PK_BAD, so.INVALID}     # every status 0..4 occurs
