"""GPU parity: edwards25519 batch Point.Mul through the C ABI vs the oracle, which is pinned by the reference's
seeded KAT (examples/dh_test.go:17-49).  BASELINE configs[0]: batch of 1024 Point.Mul (seed b2k/c1)."""
import random

import pytest

from kyber_b200 import B2KError, workload as wl
from oracle import ed25519 as ed
import ed25519_msm_cases as mc

pytestmark = pytest.mark.gpu


def test_reference_dh_kat_on_device(engine):
    rng = ed.Blake2Xb(b"")
    a, b = ed.pick_scalar(rng), ed.pick_scalar(rng)
    base = ed.encode(ed.BASE)
    pubs = engine.ed25519_mul_batch(a + b, base * 2)                 # A = a*B, B = b*B
    shared = engine.ed25519_mul_batch(a + b, pubs[32:] + pubs[:32])   # a*B', b*A
    assert shared[:32] == shared[32:]
    assert shared[:32].hex() == "80ea238cacfdab279626970bba18c69083c7751865dec4c6434bff4351282847"


def test_batch_1024_matches_oracle(engine):
    n = 1024
    s = wl.prng_scalars("b2k/c1", n, ed.L)
    a = wl.prng_scalars("b2k/c1-a", n, ed.L)
    base = ed.encode(ed.BASE)
    pts = engine.ed25519_mul_batch(b"".join(x.to_bytes(32, "little") for x in a), base * n)
    out = engine.ed25519_mul_batch(b"".join(x.to_bytes(32, "little") for x in s), pts)
    for i in range(0, n, 8):
        want = ed.encode(ed.scalar_mult(s[i] * a[i] % ed.L))
        assert out[32 * i:32 * i + 32] == want, i
    nacl = pytest.importorskip("nacl.bindings")
    for i in (1, 500, 1023):
        assert nacl.crypto_scalarmult_ed25519_noclamp(s[i].to_bytes(32, "little"), pts[32 * i:32 * i + 32]) == out[32 * i:32 * i + 32]


def test_raw_scalars_torsion_and_bad_points(engine):
    t8 = bytes.fromhex("c7176a703d4dd84fba3c0b760d10670f2a2053fa2c39ccc64ec7fd7792ac037a")
    mixed = ed.encode(ed.add(ed.scalar_mult(77), ed.decode(t8)))
    ks = [0, 1, ed.L, ed.L + 5, (1 << 255) - 1, 0x123456789]
    pts = [mixed, t8, mixed, mixed, ed.encode(ed.BASE), ((2 ** 255 - 19) + 1).to_bytes(32, "little")]
    out = engine.ed25519_mul_batch(b"".join(k.to_bytes(32, "little") for k in ks), b"".join(pts))
    for i, (k, p) in enumerate(zip(ks, pts)):
        assert out[32 * i:32 * i + 32] == ed.point_mul(k.to_bytes(32, "little"), p), i
    high = mc.crafted_high_scalars(random.Random(6))            # geScalarMult's rule: e63 = 8 kept, 9 and 16 dropped
    assert {mc.top_digit(k) for k in high} >= {8, 9, 16}
    ks = high * 2
    pts = [ed.encode(ed.BASE)] * len(high) + [mixed] * len(high)
    out = engine.ed25519_mul_batch(b"".join(k.to_bytes(32, "little") for k in ks), b"".join(pts))
    for i, (k, p) in enumerate(zip(ks, pts)):
        assert out[32 * i:32 * i + 32] == ed.point_mul(k.to_bytes(32, "little"), p), (i, hex(k))
    with pytest.raises(B2KError) as e:
        engine.ed25519_mul_batch((1).to_bytes(32, "little"), (2).to_bytes(32, "little"))     # y = 2 is not on the curve
    assert e.value.code == -5
