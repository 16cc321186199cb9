"""CPU tests: the DEVICE code of every kernel family compiled for the host (tests/host_emul/*.cpp, PTX carry
primitives emulated in ptx.cuh) and checked against the oracle and the reference's fixtures -- the same bodies the
sm_90a kernels run, exercised without a GPU.  (tests/test_abi_and_host.py covers the field and MSM bodies.)"""
import ctypes
import hashlib
import json
import os
import random
import subprocess

import pytest

from oracle import bls12381 as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "host_emul")
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")
GOLD = os.path.join(ROOT, "tests", "golden")


def _lib(name):
    src = os.path.join(EMU, name + ".cpp")
    so = os.path.join(EMU, "lib" + name + ".so")
    newest = max([os.path.getmtime(src)] + [os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith(".cuh")])
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", src, "-o", so],
                       check=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def emul():
    return _lib("emul")


def test_bls12381_pairing_bodies(emul):
    rng = random.Random(4)
    a, b = rng.randrange(o.R), rng.randrange(o.R)
    P, Q = o.g1_mul(a), o.g2_mul(b)
    out = ctypes.create_string_buffer(576)
    emul.emul_bls12381_pair(o.g1_to_affine_bytes(P), o.g2_to_affine_bytes(Q), out)
    assert out.raw == o.gt_to_bytes(o.pairing_reference(P, Q))
    emul.emul_bls12381_pair(bytes(96), o.g2_to_affine_bytes(Q), out)
    assert out.raw == o.gt_to_bytes(o.F12_ONE)
    assert emul.emul_bls12381_final_exp_is_exact_cubed(o.g1_to_affine_bytes(P), o.g2_to_affine_bytes(Q)) == 1
    args = [o.g1_to_affine_bytes(P), o.g2_to_affine_bytes(Q), o.g1_to_affine_bytes(o.g1_mul(a * b % o.R)), o.g2_to_affine_bytes(o.G2)]
    assert emul.emul_bls12381_pairing_check(*args) == 1
    args[2] = o.g1_to_affine_bytes(o.g1_mul(a * b + 1))
    assert emul.emul_bls12381_pairing_check(*args) == 0


def test_decompress_bodies_on_the_zcash_fixtures(emul):
    d = json.load(open(os.path.join(GOLD, "bls12381_deserialization.json")))
    for grp, fn, n_in, n_out, dec, toaff in (("G1", "emul_bls12381_g1_decompress", 48, 96, o.g1_decompress, o.g1_to_affine_bytes),
                                             ("G2", "emul_bls12381_g2_decompress", 96, 192, o.g2_decompress, o.g2_to_affine_bytes)):
        seen = 0
        for v in d[grp]:
            try:
                raw = bytes.fromhex(v["input"])
            except ValueError:
                continue
            if len(raw) != n_in:
                continue
            out = ctypes.create_string_buffer(n_out)
            ok = getattr(emul, fn)(raw, out)
            assert bool(ok) == v["valid"], (grp, v["name"])
            if ok:
                assert out.raw == toaff(dec(raw))
            seen += 1
        assert seen >= 13


def test_g2_mul_and_msm_bodies(emul):
    rng = random.Random(3)
    n = 8
    ks = [0, 1, o.R - 1] + [rng.randrange(o.R) for _ in range(n - 3)]
    pts = [o.g2_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[4] = None
    sb = b"".join(o.scalar_to_bytes(k) for k in ks)
    pb = b"".join(o.g2_to_affine_bytes(p) for p in pts)
    out = ctypes.create_string_buffer(96 * n)
    emul.emul_bls12381_g2_mul_batch(ctypes.c_size_t(n), sb, pb, out)
    acc = None
    for i in range(n):
        r = o.g2_mul(ks[i], pts[i])
        assert out.raw[96 * i:96 * i + 96] == o.g2_compress(r)
        acc = o.g2_add(acc, r)
    o96 = ctypes.create_string_buffer(96)
    assert emul.emul_bls12381_g2_msm(ctypes.c_size_t(n), sb, pb, 8, 8, 3, o96) == 0 and o96.raw == o.g2_compress(acc)


def test_balanced_slice_accumulate_bodies(emul):
    rng = random.Random(9)
    n = 40
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    for ks in ([rng.randrange(o.R) for _ in range(n)], [0x123456789ABCDEF] * n, [rng.randrange(1 << 20) for _ in range(n)]):
        sb = b"".join(o.scalar_to_bytes(k) for k in ks)
        want = o.g1_compress(o.g1_msm(ks, pts))
        for c, m, L in ((4, 2, 1), (8, 1, 7), (13, 32, 5), (16, 32, 2)):
            o48 = ctypes.create_string_buffer(48)
            assert emul.emul_bls12381_g1_msm_v2(ctypes.c_size_t(n), sb, pb, c, m, L, o48) == 0 and o48.raw == want, (c, m, L)


def test_glv_windowed_scalar_mul_body(emul):
    """scalar_mul_glv_bls381 (k_mul_batch's BLS12-381 G1 path): endomorphism split + signed radix-16 digits over one
    affine table -- edge scalars of the split and of the digit recoding, infinity operand."""
    rng = random.Random(21)
    x2 = o.X_ABS ** 2
    ks = [0, 1, 2, 7, 8, 9, 15, 16, 17, x2 - 1, x2, x2 + 1, x2 // 2, x2 // 2 + 1, 8 * x2 + 8, (o.R - 1) // 2, (o.R + 1) // 2,
          o.R - 1, o.R - 2, o.R - x2, int("8" * 32, 16), int("7" * 32, 16), int("f" * 31, 16), (1 << 127) - 1, 1 << 127]
    ks += [rng.randrange(o.R) for _ in range(40)]
    n = len(ks)
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[3] = None
    sb = b"".join(o.scalar_to_bytes(k) for k in ks)
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    out = ctypes.create_string_buffer(48 * n)
    emul.emul_bls12381_g1_mul_batch_glv(ctypes.c_size_t(n), sb, pb, out)
    for i in range(n):
        assert out.raw[48 * i:48 * i + 48] == o.g1_compress(o.g1_mul(ks[i], pts[i])), (i, hex(ks[i]))


def test_fixed_window_scalar_mul_bodies(emul):
    """scalar_mul_w4 (k_mul_batch on every curve): signed radix-16 digits of the whole 256-bit scalar over one affine
    table -- BLS12-381 G1 and G2, bn254 G1; edge scalars of the recoding (runs of 8s, 7s, fs, top nibble), infinity."""
    from oracle import bn254 as o4
    rng = random.Random(22)
    edge = [0, 1, 2, 7, 8, 9, 15, 16, 17, int("8" * 60, 16), int("7" * 63, 16), int("f" * 62, 16), (1 << 254) + 8]
    ks = [k % o.R for k in edge] + [o.R - 1, o.R - 8] + [rng.randrange(o.R) for _ in range(12)]
    n = len(ks)
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[4] = None
    sb = b"".join(o.scalar_to_bytes(k) for k in ks)
    out = ctypes.create_string_buffer(48 * n)
    emul.emul_bls12381_g1_mul_batch_w4(ctypes.c_size_t(n), sb, b"".join(o.g1_to_affine_bytes(p) for p in pts), out)
    for i in range(n):
        assert out.raw[48 * i:48 * i + 48] == o.g1_compress(o.g1_mul(ks[i], pts[i])), (i, hex(ks[i]))
    m = 6
    p2 = [o.g2_mul(rng.randrange(1, o.R)) for _ in range(m)]
    out2 = ctypes.create_string_buffer(96 * m)
    emul.emul_bls12381_g2_mul_batch_w4(ctypes.c_size_t(m), b"".join(o.scalar_to_bytes(k) for k in ks[-m:]),
                                       b"".join(o.g2_to_affine_bytes(p) for p in p2), out2)
    for i in range(m):
        assert out2.raw[96 * i:96 * i + 96] == o.g2_compress(o.g2_mul(ks[-m:][i], p2[i])), i
    k4 = [k % o4.ORDER for k in edge] + [o4.ORDER - 1] + [rng.randrange(o4.ORDER) for _ in range(6)]
    p4 = [o4.g1_mul(rng.randrange(1, o4.ORDER)) for _ in range(len(k4))]
    out4 = ctypes.create_string_buffer(64 * len(k4))
    emul.emul_bn254_g1_mul_batch_w4(ctypes.c_size_t(len(k4)), b"".join(k.to_bytes(32, "big") for k in k4),
                                    b"".join(o4.g1_marshal(p) for p in p4), out4)
    for i in range(len(k4)):
        assert out4.raw[64 * i:64 * i + 64] == o4.g1_marshal(o4.g1_mul(k4[i], p4[i])), i


def test_affine_pair_tree_round_bodies(emul):
    """msm_affine.cuh: R pair-tree rounds (batched affine additions, one inversion per thread) followed by the balanced
    XYZZ slices give the oracle's MSM, including the exceptional cases of the affine group law: repeated points in one
    bucket (P + P), P and -P in one bucket, operands at infinity, all-equal scalars (one bucket per window)."""
    rng = random.Random(11)
    n = 48
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[5] = None
    pts[6] = pts[7] = pts[8] = pts[9]                     # the same point four times
    pts[10] = o.g1_neg(pts[11])                           # P and -P
    pts[13] = (0, 2)                                      # on the curve with x = 0 (outside G1: only the group law matters here)
    pts[14] = (0, o.P - 2)
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    sets = ([rng.randrange(o.R) for _ in range(n)], [0x123456789ABCDEF] * n, [rng.randrange(1 << 9) for _ in range(n)])
    for ks in sets:
        sb = b"".join(o.scalar_to_bytes(k) for k in ks)
        want = o.g1_compress(o.g1_msm(ks, pts))
        for c, m, L, rounds, pbatch in ((4, 2, 3, 1, 1), (4, 2, 2, 2, 3), (5, 4, 4, 3, 8), (8, 8, 5, 6, 64), (3, 2, 1, 9, 5)):
            o48 = ctypes.create_string_buffer(48)
            rc = emul.emul_bls12381_g1_msm_affine(ctypes.c_size_t(n), sb, pb, c, m, L, rounds, pbatch, o48)
            assert rc == 0 and o48.raw == want, (c, m, L, rounds, pbatch)
            o48 = ctypes.create_string_buffer(48)        # the round as three kernels (forward x-only / invert / backward)
            rc = emul.emul_bls12381_g1_msm_affine_split(ctypes.c_size_t(n), sb, pb, c, m, L, rounds, 3 * pbatch, o48)
            assert rc == 0 and o48.raw == want, ("split", c, m, L, rounds, pbatch)
            o48 = ctypes.create_string_buffer(48)        # ... with the backward pass's operands staged by (deferred) cp.async
            emul.emul_set_pt_stage(1)
            try:
                rc = emul.emul_bls12381_g1_msm_affine_split(ctypes.c_size_t(n), sb, pb, c, m, L, rounds, 3 * pbatch, o48)
            finally:
                emul.emul_set_pt_stage(0)
            assert rc == 0 and o48.raw == want, ("split + staged", c, m, L, rounds, pbatch)
    # bn254 (8-limb field) through the same template
    from oracle import bn254 as o4
    pts4 = [o4.g1_mul(rng.randrange(1, o4.ORDER)) for _ in range(12)]
    pts4[3] = pts4[4]
    ks4 = [7] * 6 + [rng.randrange(o4.ORDER) for _ in range(6)]
    sb4 = b"".join(k.to_bytes(32, "big") for k in ks4)
    pb4 = b"".join(o4.g1_marshal(p) for p in pts4)
    acc = None
    for k, p4 in zip(ks4, pts4):
        acc = o4.g1_add(acc, o4.g1_mul(k, p4))
    o64 = ctypes.create_string_buffer(64)
    assert emul.emul_bn254_g1_msm_affine(ctypes.c_size_t(12), sb4, pb4, 4, 2, 3, 2, 4, o64) == 0
    assert o64.raw == o4.g1_marshal(acc)


def test_bucket_exchange_bodies(emul):
    """Multi-GPU shape 1 (msm_host.cuh: msm_buckets_dev -> all-to-all -> msm_reduce_windows_dev -> all-gather ->
    msm_finish_dev) with 1, 2, 4 and 8 virtual ranks: the partial buckets of the ranks, summed inside the chunk
    reduction (msm_reduce_chunk_parts), give the oracle's MSM -- including the same point (and P, -P) landing in the
    same bucket on different ranks, a rank without pairs, and all-equal scalars."""
    rng = random.Random(23)
    n = 36
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[20] = pts[2]                                      # same point, different ranks for world >= 2
    pts[30] = o.g1_neg(pts[3])
    pts[7] = None
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    base = [rng.randrange(o.R) for _ in range(n)]
    base[20] = base[2]
    base[30] = base[3]
    for ks in (base, [0x0FEDCBA987654321] * n, [rng.randrange(1 << 11) for _ in range(n)]):
        sb = b"".join(o.scalar_to_bytes(k) for k in ks)
        want = o.g1_compress(o.g1_msm(ks, pts))
        for c, m, L, rounds, pbatch, world in ((4, 2, 3, 0, 1, 1), (4, 1, 2, 1, 3, 2), (8, 8, 5, 2, 4, 4), (16, 64, 2, 0, 1, 8),
                                               (4, 4, 0, 0, 1, 64)):
            o48 = ctypes.create_string_buffer(48)
            rc = emul.emul_bls12381_g1_msm_exchange(ctypes.c_size_t(n), sb, pb, c, m, L, rounds, pbatch, world, o48)
            assert rc == 0 and o48.raw == want, (c, m, L, rounds, pbatch, world)
    o48 = ctypes.create_string_buffer(48)                 # window count not a multiple of the world size: refused
    assert emul.emul_bls12381_g1_msm_exchange(ctypes.c_size_t(n), sb, pb, 13, 2, 3, 0, 1, 8, o48) == -2


def test_two_level_bucket_reduction_bodies(emul):
    """msm.cuh: msm_reduce_l1 / msm_reduce_l2 (window sum = sum of the level-1 running sums + m1 * sum_t t * run_t, the second
    term reduced again in chunks of m2 with one small scalar multiplication per chunk) against the oracle, for several chunk
    shapes incl. m2 = 1 and a whole window in one level-2 chunk, skewed scalars, and combined with the bucket exchange."""
    rng = random.Random(29)
    n = 30
    pts = [o.g1_mul(rng.randrange(1, o.R)) for _ in range(n)]
    pts[4] = pts[5]
    pts[9] = None
    pb = b"".join(o.g1_to_affine_bytes(p) for p in pts)
    for ks in ([rng.randrange(o.R) for _ in range(n)], [o.R - 1] * n, [rng.randrange(1 << 13) for _ in range(n)]):
        sb = b"".join(o.scalar_to_bytes(k) for k in ks)
        want = o.g1_compress(o.g1_msm(ks, pts))
        for c, m1, m2, L, world in ((4, 2, 2, 0, 1), (4, 1, 8, 2, 1), (8, 4, 4, 3, 1), (8, 8, 16, 0, 1), (8, 2, 1, 5, 1),
                                    (16, 4, 4, 2, 1), (8, 4, 4, 3, 4), (16, 4, 8, 2, 8)):
            o48 = ctypes.create_string_buffer(48)
            rc = emul.emul_bls12381_g1_msm_reduce2(ctypes.c_size_t(n), sb, pb, c, m1, m2, L, world, o48)
            assert rc == 0 and o48.raw == want, (c, m1, m2, L, world)
    from oracle import bn254 as o4
    pts4 = [o4.g1_mul(rng.randrange(1, o4.ORDER)) for _ in range(10)]
    ks4 = [rng.randrange(o4.ORDER) for _ in range(10)]
    acc = None
    for k, p4 in zip(ks4, pts4):
        acc = o4.g1_add(acc, o4.g1_mul(k, p4))
    o64 = ctypes.create_string_buffer(64)
    assert emul.emul_bn254_g1_msm_reduce2(ctypes.c_size_t(10), b"".join(k.to_bytes(32, "big") for k in ks4),
                                          b"".join(o4.g1_marshal(p) for p in pts4), 8, 4, 4, 3, o64) == 0
    assert o64.raw == o4.g1_marshal(acc)


def test_hash_to_curve_bodies():
    from oracle import h2c_bls12381 as h, h2c_bls12381_g2 as h2
    l1, l2 = _lib("emul_h2c"), _lib("emul_h2c_g2")
    rng = random.Random(5)
    for msg, dst in ((b"", h.DST_G1), (b"abc", h.DST_G2), (rng.randbytes(119), b"X"), (rng.randbytes(56), h.DST_G1)):
        o128 = ctypes.create_string_buffer(128)
        l1.emul_expand_xmd_128(msg, len(msg), dst, len(dst), o128)
        assert o128.raw == h.expand_message_xmd(msg, dst, 128)
        out = ctypes.create_string_buffer(96)
        l1.emul_bls12381_hash_to_g1(msg, len(msg), dst, len(dst), out)
        assert out.raw == o.g1_to_affine_bytes(h.hash_to_g1(msg, dst))
    for msg, dst in ((b"", h.DST_G2), (rng.randbytes(77), b"Y")):
        out = ctypes.create_string_buffer(192)
        l2.emul_bls12381_hash_to_g2(msg, len(msg), dst, len(dst), out)
        assert out.raw == o.g2_to_affine_bytes(h2.hash_to_g2(msg, dst))


def test_isogeny_tool_and_oracle_derivations_agree():
    """tools/derive_isogeny.py (standalone, feeds the device constants) and oracle/h2c_bls12381.py derive the same map."""
    import importlib.util
    from oracle import h2c_bls12381 as h, h2c_bls12381_g2 as h2
    spec = importlib.util.spec_from_file_location("derive_isogeny", os.path.join(ROOT, "tools", "derive_isogeny.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    xn, xd, yn, yd = mod.derive()
    assert (xn, xd, yn, yd) == (h.ISO_XNUM, h.ISO_XDEN, h.ISO_YNUM, h.ISO_YDEN)
    x0, v, u = mod.derive_g2()
    assert x0 == h2.X0 and v == h2._VQ and u == h2._UQ


def test_bn254_pairing_bodies():
    from oracle import bn254 as c, bn254_pairing as b
    lib = _lib("emul_bn")
    rng = random.Random(8)
    for x, y in ((1, 1), (rng.randrange(c.ORDER), rng.randrange(c.ORDER))):
        P, Q = c.g1_mul(x), b.g2_mul(y)
        out = ctypes.create_string_buffer(384)
        lib.emul_bn254_pair(c.g1_marshal(P), b.g2_marshal(Q), out)
        assert out.raw == b.gt_to_bytes(b.pairing(P, Q))
    x, y = rng.randrange(c.ORDER), rng.randrange(c.ORDER)
    args = [c.g1_marshal(c.g1_mul(x)), b.g2_marshal(b.g2_mul(y)), c.g1_marshal(c.g1_mul(x * y % c.ORDER)), b.g2_marshal(b.G2)]
    assert lib.emul_bn254_pairing_check(*args) == 1
    # bn256 twin (pairing/bn256/optate.go): same templates, xi = i+3, 10-limb field, its own digit table
    from oracle import bn256 as c6, bn256_pairing as b6
    for x, y in ((1, 1), (rng.randrange(c6.ORDER), rng.randrange(c6.ORDER))):
        P, Q = c6.g1_mul(x), b6.g2_mul(y)
        out = ctypes.create_string_buffer(384)
        lib.emul_bn256_pair(c6.g1_marshal(P), c6.g2_marshal(Q), out)
        assert out.raw == b6.gt_to_bytes(b6.pairing(P, Q))


def test_ed25519_and_inversion_bodies():
    from oracle import ed25519 as ed
    import ed25519_msm_cases as mc
    lib = _lib("emul_ed")
    t8 = bytes.fromhex("c7176a703d4dd84fba3c0b760d10670f2a2053fa2c39ccc64ec7fd7792ac037a")
    high = mc.crafted_high_scalars(random.Random(5))            # geScalarMult's rule: e63 = 8 kept, 9 and 16 dropped
    assert {mc.top_digit(k) for k in high} >= {8, 9, 16}
    for pt in (ed.encode(ed.BASE), t8, ed.encode(ed.add(ed.scalar_mult(77), ed.decode(t8)))):
        for k in [0, 1, ed.L, ed.L + 5, (1 << 255) - 1, 0x1234567890ABCDEF] + high:
            out = ctypes.create_string_buffer(32)
            assert lib.emul_ed25519_mul(k.to_bytes(32, "little"), pt, out) == 1
            assert out.raw == ed.point_mul(k.to_bytes(32, "little"), pt)
    assert lib.emul_ed25519_mul((1).to_bytes(32, "little"), (2).to_bytes(32, "little"), ctypes.create_string_buffer(32)) == 0
    inv = _lib("emul_inv")
    rng = random.Random(3)
    for name, p, n in (("fp381", o.P, 12), ("fp254", 21888242871839275222246405745257275088696311157297823662689037894645226208583, 8),
                       ("fp256", 65000549695646603732796438742359905742825358107623003571877145026864184071783, 10)):
        R = 1 << (32 * n)
        for a in [0, 1, p - 1] + [rng.randrange(p) for _ in range(40)]:
            am = a * R % p
            inp = (ctypes.c_uint32 * n)(*[(am >> (32 * i)) & 0xFFFFFFFF for i in range(n)])
            out = (ctypes.c_uint32 * n)()
            getattr(inv, f"emul_{name}_inv_vartime")(inp, out)
            assert sum(int(x) << (32 * i) for i, x in enumerate(out)) == (pow(a, -1, p) * R % p if a else 0)
    # branch-free binary GCD on 64-bit approximations (fp_inv_bingcd): edge values, short operands, many random ones
    for name, p, n in (("fp381", o.P, 12), ("fp254", 21888242871839275222246405745257275088696311157297823662689037894645226208583, 8),
                       ("fp256", 65000549695646603732796438742359905742825358107623003571877145026864184071783, 10),
                       ("fp25519", 2 ** 255 - 19, 8)):
        R = 1 << (32 * n)
        Ri = pow(R, -1, p)
        cases = [0, 1, 2, 3, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, 1 << (p.bit_length() - 1), (1 << (p.bit_length() - 1)) - 1]
        cases += [rng.randrange(1, 1 << k) for k in range(1, p.bit_length(), 5) for _ in range(2)]
        cases += [rng.randrange(p) for _ in range(1500)]
        fn = getattr(inv, f"emul_{name}_inv_bingcd")
        for am in cases:                       # am = the Montgomery representative itself (so short VALUES reach the loop)
            a = am * Ri % p
            inp = (ctypes.c_uint32 * n)(*[(am >> (32 * i)) & 0xFFFFFFFF for i in range(n)])
            out = (ctypes.c_uint32 * n)()
            fn(inp, out)
            assert sum(int(x) << (32 * i) for i, x in enumerate(out)) == (pow(a, -1, p) * R % p if a else 0), (name, am)


def test_bn_hash_to_g1_bodies_against_reference_vectors():
    """bn_hash.cuh on the host: Keccak-256, expand_message_xmd, hashToField, the SvdW map and the full bn254 hash against
    the reference's vectors (pairing/bn254/point_test.go:14-124, test_vectors_test.go); bn256 try-and-increment against
    the oracle, which the byte-exact BDN signature fixtures pin (tests/test_oracle_bdn_bn256.py)."""
    from oracle import bn254_hash as bh, bn256 as o6
    lib = _lib("emul_bn_hash")
    fx = json.load(open(os.path.join(GOLD, "bn254_hash_vectors.json")))
    out32, out64, out96 = (ctypes.create_string_buffer(k) for k in (32, 64, 96))
    for m in (b"", b"abc", bytes(135), bytes(136), bytes(137), bytes(range(256)) * 3):
        lib.emul_keccak256(m, len(m), out32)
        assert out32.raw == bh.keccak256(m)
    e = fx["expand_msg"]
    lib.emul_bn254_expand_96(bytes.fromhex(e["msg_hex"]), len(e["msg_hex"]) // 2, e["dst"].encode(), len(e["dst"]), out96)
    assert out96.raw.hex() == e["out"]
    dst = fx["hash_to_field"]["dst"].encode()
    for c in fx["hash_to_field"]["cases"]:
        m = bytes.fromhex(c["msg"])
        lib.emul_bn254_hash_to_field(m, len(m), dst, len(dst), out64)
        assert out64.raw.hex() == c["x"] + c["y"]
    for c in fx["map_to_point"]["cases"]:
        lib.emul_bn254_map_to_point(int(c["u"]).to_bytes(32, "big"), out64)
        assert out64.raw == int(c["x"]).to_bytes(32, "big") + int(c["y"]).to_bytes(32, "big")
    dst = fx["hash_to_point"]["dst"].encode()
    for c in fx["hash_to_point"]["cases"]:
        m = bytes.fromhex(c["msg_hex"])
        lib.emul_bn254_hash_to_g1(m, len(m), dst, len(dst), out64)
        assert out64.raw.hex() == c["point"]
    # bn256 HashG1 (pairing/bn256/hash.go:10-110): HMAC-SHA256 vs hashlib, then the reference's 11 KATs (hash_test.go:11-57)
    import hmac
    for key, m in ((b"", b""), (bytes(32), b"abc"), (b"k" * 64, bytes(100)), (b"long key " * 20, bytes(range(200)))):
        lib.emul_hmac_sha256(key, len(key), m, len(m), out32)
        assert out32.raw == hmac.new(key, m, hashlib.sha256).digest()
    for c in json.load(open(os.path.join(GOLD, "bn256_hashg1_vectors.json")))["cases"]:
        m = bytes.fromhex(c["msg_hex"])
        lib.emul_bn256_hash_g1(m, len(m), None, 0, out64)
        assert out64.raw.hex() == c["point"]
    rng = random.Random(77)
    for _ in range(40):                                                                # non-nil dst, ragged lengths: vs the oracle
        m = bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 150)))
        d = bytes(rng.getrandbits(8) for _ in range(rng.choice((1, 16, 64, 65, 200))))
        lib.emul_bn256_hash_g1(m, len(m), d, len(d), out64)
        assert out64.raw == o6.g1_marshal(o6.hash_g1(m, d))
    bdn_msg = json.load(open(os.path.join(GOLD, "bdn_bn256_fixtures.json")))["fixtures"]["msg"].encode()
    for m in (bdn_msg, b"", b"x" * 200, bytes(range(64))):
        lib.emul_bn256_hash_to_g1(m, len(m), out64)
        assert out64.raw == o6.g1_marshal(o6.hash_to_g1(m))



@pytest.mark.parametrize("group", ["bls12381_g1", "bls12381_g2", "bn254_g1", "bn254_g2", "bn256_g1", "bn256_g2"])
def test_msm_bodies_every_group_and_input_set(emul, group):
    """emul_msm (msm.cuh: digits, counting sort, slices or one thread per bucket, fix-up, chunk reduction, Horner) for each
    group the device instantiates, on the input sets of tests/test_gpu_msm_curves.py (equal points in one bucket, P and -P,
    infinities, empty upper windows, scalar edges, digit patterns that fill the largest bucket) through the forced (c, m, L)
    shapes of its plans.  The operands repeat a few multipliers so that the oracle side stays cheap."""
    import msm_cases as mc
    g = mc.GROUPS[group]
    fn = {"bls12381_g1": "emul_bls12381_g1_msm_v2", "bls12381_g2": "emul_bls12381_g2_msm", "bn254_g1": None,
          "bn254_g2": "emul_bn254_g2_msm", "bn256_g1": "emul_bn256_g1_msm", "bn256_g2": "emul_bn256_g2_msm"}[group]
    n = 96
    A = mc.multipliers(g, 5)
    operand = {0: bytes(g.in_bytes)}
    for x in A + [g.r - A[0]]:
        operand[x] = g.operand(g.mul(x))
    assert operand[0] == g.operand(None)
    for name in mc.SETS:
        a, s = mc.build_set(g, name, n, A)
        sb, pb = mc.scalars_to_bytes(s), b"".join(operand[x] for x in a)
        want = g.expected(a, s)
        for c, m, L in mc.EMUL_PLANS:
            out = ctypes.create_string_buffer(g.out_bytes)
            if fn is None:       # bn254 G1 enters through the affine-rounds wrapper with no rounds
                rc = emul.emul_bn254_g1_msm_affine(ctypes.c_size_t(n), sb, pb, c, m, L, 0, 1, out)
            else:
                rc = getattr(emul, fn)(ctypes.c_size_t(n), sb, pb, c, m, L, out)
            assert rc == 0 and out.raw == want, (group, name, c, m, L)
    bad = mc.scalars_to_bytes([g.r] + s[1:])
    out = ctypes.create_string_buffer(g.out_bytes)
    rc = emul.emul_bn254_g1_msm_affine(ctypes.c_size_t(n), bad, pb, 4, 2, 3, 0, 1, out) if fn is None else \
        getattr(emul, fn)(ctypes.c_size_t(n), bad, pb, 4, 2, 3, out)
    assert rc == -3, group
