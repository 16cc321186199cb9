"""CPU: the DLEQ / PVSS device code (kyber_b200/csrc/pvss.cuh) compiled for the host and checked against the restatement in
tests/pvss_cases.py -- the joint multiplication over two variable bases on both sides of the top-digit rule, the per-share and
per-deal challenges.  BLAKE2b, the keyed XOF and sc_pick are checked on their own by the byte harness (test_bytes_emulation.py,
test_gpu_bytes.py)."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import ed25519 as ed
import ed25519_msm_cases as mc
import pvss_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_emul", "emul_pvss.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_pvss") / "libemul_pvss.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", SRC, "-o", so],
                   check=True)
    lib = ctypes.CDLL(so)
    u32, cp = ctypes.c_uint32, ctypes.c_char_p
    lib.emul_double_mul_var.argtypes = [cp] * 5
    lib.emul_dleq_verify.argtypes = [cp] * 5
    lib.emul_dec_share.argtypes = [cp] * 5
    lib.emul_enc_shares.argtypes = [u32, u32] + [cp] * 8
    return lib


def test_double_mul_var_is_the_sum_of_two_reference_multiplications(lib):
    rng = random.Random(5)
    highs = mc.crafted_high_scalars(rng)
    scalars = highs + [0, 1, mc.L - 1, mc.L, mc.L + 1, (1 << 255) - 1] + [rng.getrandbits(256) for _ in range(6)]
    for k, r in enumerate(scalars):
        c = scalars[(k * 7 + 3) % len(scalars)]
        p = mc.point(rng.randrange(mc.L), rng.randrange(8))            # torsion parts
        p2 = mc.point(rng.randrange(mc.L), rng.randrange(8))
        out = ctypes.create_string_buffer(32)
        assert lib.emul_double_mul_var(r.to_bytes(32, "little"), p, c.to_bytes(32, "little"), p2, out) == 1
        want = ed.add(mc.ge_scalar_mult(r.to_bytes(32, "little"), ed.decode(p)), mc.ge_scalar_mult(c.to_bytes(32, "little"), ed.decode(p2)))
        assert out.raw == ed.encode(want), (hex(r), hex(c))


def test_dleq_and_dec_share_bodies(lib):
    rng = random.Random(6)
    g, h = pc.random_point(rng), pc.random_point(rng, torsion=True)
    proof, xg, xh = pc.new_dleq_proof(g, h, rng.randrange(mc.L), rng.randrange(mc.L))
    cases = [(g, h, xg, xh, proof), (h, g, xg, xh, proof), (g, h, pc.undecodable(), xh, proof),
             (g, h, xg, xh, proof[:64] + pc.add(proof[64:96], pc.T8) + proof[96:])]
    for cs in cases:
        assert lib.emul_dleq_verify(*cs) == pc.dleq_verify(*cs)
    priv = rng.randrange(1, mc.L)
    x = pc.base_mul(priv)
    enc_v = pc.mul(priv, pc.random_point(rng))
    dec_v, p = pc.dec_share(priv, enc_v, rng.randrange(mc.L))
    c_plus_l = (int.from_bytes(p[:32], "little") + mc.L).to_bytes(32, "little") + p[32:]
    for cs in [(pc.G, x, enc_v, dec_v, p), (pc.G, x, enc_v, pc.base_mul(3), p), (pc.G, x, enc_v, dec_v, c_plus_l),
               (pc.G, x, enc_v, dec_v, p[:64] + pc.base_mul(5) + p[96:])]:
        want = pc.verify_dec_share(*cs)
        assert lib.emul_dec_share(*cs) == want
    assert [lib.emul_dec_share(pc.G, x, enc_v, dec_v, q) for q in (p, c_plus_l)] == [pc.OK, pc.CHALLENGE]


@pytest.mark.parametrize("n", [1, 2, 3, 17])
def test_global_challenge_and_enc_shares(lib, n):
    rng = random.Random(10 + n)
    t = n // 2 + 1
    h = pc.random_point(rng)
    xs = [pc.base_mul(rng.randrange(1, mc.L)) for _ in range(n)]
    commits, shares, _ = pc.enc_shares(h, xs, rng.randrange(mc.L), t, pc.RandomStream("emul %d" % n))
    shs = [pc.eval_commits(commits, i + 1) for i in range(n)]
    vs = [v for _, v, _ in shares]
    proofs = [p for _, _, p in shares]

    def run(h_, commits_, xs_, shs_, vs_, proofs_):
        st, ch = ctypes.create_string_buffer(n), ctypes.create_string_buffer(32)
        lib.emul_enc_shares(len(commits_), n, h_, b"".join(commits_), b"".join(xs_), b"".join(shs_), b"".join(vs_),
                            b"".join(proofs_), st, ch)
        return list(st.raw), ch.raw

    st, ch = run(h, commits, xs, shs, vs, proofs)
    assert ch == pc.global_challenge(commits, vs, proofs)
    assert st == [pc.OK] * n
    bad = proofs[:]
    bad[0] = bad[0][:32] + ((int.from_bytes(bad[0][32:64], "little") + 1) % mc.L).to_bytes(32, "little") + bad[0][64:]
    st, _ = run(h, commits, xs, shs, vs, bad)
    assert st == pc.verify_enc_share_batch(h, commits, xs, shs, vs, bad) == [pc.INVALID] + [pc.OK] * (n - 1)
    st, _ = run(h, commits[:-1] + [pc.add(commits[-1], pc.G)], xs, shs, vs, proofs)
    assert st == [pc.CHALLENGE] * n
    st, _ = run(h, [pc.undecodable()] + commits[1:], xs, shs, vs, proofs)
    assert st == [pc.POINT] * n
