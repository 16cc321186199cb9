"""CPU: the Ed25519 verification device code (kyber_b200/csrc/eddsa.cuh) compiled for the host and checked against the oracle
on every fixture and crafted case -- the same bodies k_ed25519_verify runs.  SHA-512 and the reduction mod l are checked on
their own by the byte harness (test_bytes_emulation.py, test_gpu_bytes.py)."""
import ctypes
import os
import subprocess

import pytest

from oracle import ed25519 as ed
from oracle import eddsa as oe
import eddsa_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_eddsa.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_eddsa") / "libemul_eddsa.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    lib.emul_ed25519_verify.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p]
    return lib


def test_generated_base_table_matches_the_oracle(lib):
    out = ctypes.create_string_buffer(8 * 96)
    lib.emul_base_table(out)
    for k in range(1, 9):
        x, y = ed.scalar_mult(k)
        want = b"".join(v.to_bytes(32, "little") for v in ((y + x) % ed.P, (y - x) % ed.P, 2 * ed.D * x * y % ed.P))
        assert out.raw[96 * (k - 1):96 * k] == want, k


def _check(lib, items):
    n = 0
    for name, pk, msg, sig in items:
        want = oe.verify_with_checks(pk, msg, sig)
        assert lib.emul_ed25519_verify(pk, msg, len(msg), sig) == want, name
        n += 1
    return n


def test_verify_matches_the_oracle_on_the_fixtures(lib):
    items = [("rfc%d" % i, pk, m, s) for i, (_, pk, m, s) in enumerate(cases.rfc8032())]
    items += [("sign.input %d" % i, pk, m, s) for i, (_, pk, m, s) in enumerate(cases.sign_input())]
    items += [("wycheproof %d" % tc, pk, m, s) for tc, pk, m, s, _ in cases.wycheproof() if len(s) == 64 and len(pk) == 32]
    items += [c[:4] for c in cases.inline()]
    assert _check(lib, items) > 1150


def test_verify_matches_the_oracle_on_crafted_cases(lib):
    got = {name: lib.emul_ed25519_verify(pk, msg, len(msg), sig) for name, pk, msg, sig in cases.crafted()}
    assert set(got.values()) == set(range(9))          # every status, 0..8, occurs
    assert _check(lib, cases.crafted() + cases.lengths_cases()) > 60
