"""CPU tests: pin hash-to-G1 (derived isogeny, SSWU, XMD) on the reference's signature KATs
(tests/golden/bls12381_signature_kats.json, extracted from kilic/suite_test.go and bls12381_test.go)."""
import hashlib
import json
import os

import pytest

from oracle import bls12381 as o
from oracle import h2c_bls12381 as h

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bls12381_signature_kats.json")))


def test_expand_message_xmd_shape():
    out = h.expand_message_xmd(b"abc", b"QUUX-V01-CS02-with-expander-SHA256-128", 128)
    assert len(out) == 128 and out != bytes(128)


XMD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "xmd_sha256_vectors.json")))["vectors"]


@pytest.mark.parametrize("dst_kind", ["short", "oversize"])
def test_expand_message_xmd_rfc9380_vectors(dst_kind):
    """RFC 9380 appendix K.1 (tests/golden/make_golden_xmd.py): five messages, 32 and 128 output bytes; the 256-byte DST takes
    the H2C-OVERSIZE-DST- pre-hash of section 5.3.3 (the device refuses DSTs over 255 bytes, so only the oracle sees it)"""
    vs = [v for v in XMD if (len(v["dst"]) > 255) == (dst_kind == "oversize")]
    assert len(vs) == 10
    for v in vs:
        got = h.expand_message_xmd(v["msg"].encode(), v["dst"].encode(), v["len_in_bytes"])
        assert got.hex() == v["uniform_bytes"], (len(v["msg"]), len(v["dst"]), v["len_in_bytes"])


def test_isogeny_is_a_homomorphism_onto_the_curve():
    import random
    rng = random.Random(3)
    pts = []
    while len(pts) < 3:
        x = rng.randrange(o.P)
        y = o.fp_sqrt((x ** 3 + h.ISO_A * x + h.ISO_B) % o.P)
        if y is not None:
            pts.append((x, y))
    for p in pts:
        assert o.g1_is_on_curve(h.iso_map(p))
    assert h.iso_map(h._add(pts[0], pts[1])) == o.g1_add(h.iso_map(pts[0]), h.iso_map(pts[1]))
    # monic denominators, leading coefficients 1/121 and 1/1331
    assert h.ISO_XDEN[-1] == 1 and h.ISO_YDEN[-1] == 1
    assert h.ISO_XNUM[-1] * 121 % o.P == 1 and h.ISO_YNUM[-1] * 1331 % o.P == 1


def test_signature_edge_case_default_dst():
    k = KAT["edge_case_g1"]                       # bls12381_test.go:877-904
    pk = o.g2_decompress(bytes.fromhex(k["pk_g2"]))
    sig = o.g1_decompress(bytes.fromhex(k["sig_g1"]))
    hm = h.hash_to_g1(bytes.fromhex(k["msg"]))
    assert o.g1_in_subgroup(hm)
    assert o.validate_pairing(hm, pk, sig, o.G2)  # bls.Verify on G1: sign/bls/bls.go:36-38,82-96


def test_sig_on_g1_verifies_only_with_g2_domain():
    k = KAT["sig_on_g1_g2domain"]                 # kilic/suite_test.go:17-46 and :84-106
    pk = o.g2_decompress(bytes.fromhex(k["pk_g2"]))
    sig = o.g1_decompress(bytes.fromhex(k["sig_g1"]))
    msg = hashlib.sha256((k["round"]).to_bytes(8, "big")).digest()
    assert not o.validate_pairing(h.hash_to_g1(msg, h.DST_G1), pk, sig, o.G2)
    assert o.validate_pairing(h.hash_to_g1(msg, h.DST_G2), pk, sig, o.G2)


def test_hash_to_g2_isogeny_cofactor_and_drand_kat():
    from oracle import h2c_bls12381_g2 as h2
    import random
    rng = random.Random(4)
    # isogeny lands on E2 and is a homomorphism
    pts = []
    while len(pts) < 2:
        x = (rng.randrange(o.P), rng.randrange(o.P))
        y = o.f2_sqrt(o.f2_add(o.f2_add(o.f2_mul(o.f2_sqr(x), x), o.f2_mul(h2.A2, x)), h2.B2))
        if y is not None:
            pts.append((x, y))
    for p in pts:
        assert o.g2_is_on_curve(h2.iso_map(p))
    # cofactor clearing: endomorphism form == multiplication by h_eff, result in G2
    q = h2.iso_map(pts[0])
    c = h2.clear_cofactor(q)
    assert c == h2._g2_mul_any(h2.H_EFF_G2, q) and o.g2_in_subgroup(c)
    # drand KAT, signatures on G2 (kilic/suite_test.go:48-72): e(G1 base, sig) == e(pk, H(msg))
    k = KAT["sig_on_g2"]
    pk = o.g1_decompress(bytes.fromhex(k["pk_g1"]))
    sig = o.g2_decompress(bytes.fromhex(k["sig_g2"]))
    msg = hashlib.sha256(bytes.fromhex(k["prev_sig"]) + (k["round"]).to_bytes(8, "big")).digest()
    hm = h2.hash_to_g2(msg)
    assert o.g2_in_subgroup(hm)
    assert o.validate_pairing(o.G1, sig, pk, hm)
