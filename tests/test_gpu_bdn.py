"""GPU: sign/bdn's verifier batch -- a roster's terms once (NewMask), then aggregate keys (AggregatePublicKeys) and bls.Verify
for many masks in one call, on BLS12-381 (both schemes) and bn256.

The expected aggregate key of every mask is (sum over enabled i of (c_i + 1) x_i) B from one fixed-base multiplication, so the
device's masked sums are checked against a path that never adds terms; a sample also equals today's per-mask G2/G1 MSM byte for
byte, and the bn256 aggregate equals the reference's byte-exact fixture."""
import json
import os
import random

import pytest

import bdn_cases as bc
from kyber_b200.capi import B2KError, ERR_ARG, ERR_POINT
from oracle import bdn, bls12381 as o, bn256 as ob

pytestmark = pytest.mark.gpu
FX = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bdn_bn256_fixtures.json")))["fixtures"]
DST_G1 = b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_"
DST_G2 = b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_"
OK, SIG, INVALID = 0, 1, 2

# key group -> (key wire bytes, operand bytes, signature wire bytes, dst)
SCHEMES = {"bls12381_g2": (96, 192, 48, DST_G1), "bls12381_g1": (48, 96, 96, DST_G2)}


class Roster:
    """n seeded keys of one scheme, their terms and (c_i + 1) factors"""

    def __init__(self, eng, group: str, n: int, seed: int):
        wire, operand, _, _ = SCHEMES[group]
        self.group, self.n, self.operand = group, n, operand
        rng = random.Random(seed)
        self.xs = [rng.randrange(1, o.R) for _ in range(n)]
        base = o.g2_to_affine_bytes(o.G2) if group == "bls12381_g2" else o.g1_to_affine_bytes(o.G1)
        mul = eng.bls12381_g2_mul_batch if group == "bls12381_g2" else eng.bls12381_g1_mul_batch
        self.pubs = mul(bc.scalars_be(self.xs, o.R), base * n)
        fac = eng.bdn_coefficients(self.pubs, wire, add_one=True)
        self.factors = [int.from_bytes(fac[32 * i:32 * i + 32], "big") for i in range(n)]
        self.terms = eng.bdn_terms(group, self.pubs)

    def expected_keys(self, eng, masks):
        return eng.commit_batch(self.group, bc.scalars_be([bc.mask_scalar(self.factors, self.xs, k, self.n, o.R) for k in masks], o.R))

    def signatures(self, eng, masks, msgs):
        """valid aggregate signatures: the mask's scalar times H(m), compressed"""
        _, _, _, dst = SCHEMES[self.group]
        scal = bc.scalars_be([bc.mask_scalar(self.factors, self.xs, k, self.n, o.R) for k in masks], o.R)
        if self.group == "bls12381_g2":
            return eng.bls12381_g1_mul_batch(scal, eng.bls12381_hash_to_g1(msgs, dst))
        return eng.bls12381_g2_mul_batch(scal, eng.bls12381_hash_to_g2(msgs, dst))


def _rows(blob: bytes, width: int):
    return [blob[width * i:width * i + width] for i in range(len(blob) // width)]


@pytest.mark.parametrize("group", ["bls12381_g2", "bls12381_g1"])
def test_aggregate_keys_match_scalar_sum_and_per_mask_msm(engine, group):
    n, m = 1001, 2048
    rng = random.Random(7 if group == "bls12381_g2" else 8)
    r = Roster(engine, group, n, seed=11)
    # the coefficients the library hashed are the reference's (oracle restatement of hashPointToR)
    wire = SCHEMES[group][0]
    coefs = bdn.hash_point_to_r(_rows(r.pubs, wire), o.R)
    assert [c + 1 for c in coefs] == r.factors
    masks = bc.edge_masks(n, rng)
    masks += bc.random_masks(n, m - len(masks), rng)
    got = engine.bdn_aggregate_keys(group, r.terms, masks)
    assert _rows(got, r.operand) == _rows(r.expected_keys(engine, masks), r.operand)
    assert got[:r.operand] == bytes(r.operand)                     # the empty mask: infinity, all zeros
    # today's path, one MSM per mask over (c_i + 1, PK_i), gives the same bytes
    dec, ok = (engine.bls12381_g2_decompress if group == "bls12381_g2" else engine.bls12381_g1_decompress)(r.pubs)
    assert set(ok) == {1}
    keys = _rows(dec, r.operand)
    fac = bc.scalars_be(r.factors, o.R)
    for k in list(range(1, len(bc.edge_masks(n, random.Random(0))))) + rng.sample(range(8, m), 24):
        en = [i for i in range(n) if bc.bit(masks[k], i)]
        want = engine._call(f"b2k_{group}_msm_affine", len(en), b"".join(fac[32 * i:32 * i + 32] for i in en),
                            b"".join(keys[i] for i in en), out=r.operand)
        assert got[r.operand * k:r.operand * (k + 1)] == want, k


def test_oracle_masked_sum_on_a_sample(engine):
    """the oracle's plain masked sum of the device's terms equals the device's aggregate (duplicates and a negated term too)"""
    rng = random.Random(9)
    r = Roster(engine, "bls12381_g1", 21, seed=12)
    pts = [None if t == bytes(96) else (int.from_bytes(t[:48], "big"), int.from_bytes(t[48:], "big")) for t in _rows(r.terms, 96)]
    # duplicate term 3 into slot 4, the negation of term 5 into slot 6, infinity into slot 7
    pts[4] = pts[3]
    pts[6] = o.g1_neg(pts[5])
    pts[7] = None
    enc = [bytes(96) if p is None else p[0].to_bytes(48, "big") + p[1].to_bytes(48, "big") for p in pts]
    masks = bc.edge_masks(21, rng) + bc.random_masks(21, 16, rng) + [bc.mask_of(21, [3, 4]), bc.mask_of(21, [5, 6, 7])]
    got = _rows(engine.bdn_aggregate_keys("bls12381_g1", b"".join(enc), masks), 96)
    for k, mk in enumerate(masks):
        want = bc.aggregate_public_keys(pts, mk, 21, o.g1_add)
        assert got[k] == (bytes(96) if want is None else want[0].to_bytes(48, "big") + want[1].to_bytes(48, "big")), k


def _non_subgroup_sig(group, rng):
    while True:
        if group == "bls12381_g2":                       # signatures on G1
            x = rng.randrange(o.P)
            y = o.fp_sqrt((x ** 3 + 4) % o.P)
            if y is not None:
                return o.g1_compress((x, y))
        else:
            x = (rng.randrange(o.P), rng.randrange(o.P))
            y = o.f2_sqrt(o.f2_add(o.f2_mul(o.f2_sqr(x), x), o.B2))
            if y is not None:
                return o.g2_compress((x, y))


@pytest.mark.parametrize("group", ["bls12381_g2", "bls12381_g1"])
def test_verify_statuses_in_a_mixed_batch(engine, group):
    n, m = 300, 64
    rng = random.Random(21)
    r = Roster(engine, group, n, seed=13)
    _, _, sig_bytes, dst = SCHEMES[group]
    masks = bc.edge_masks(n, rng) + bc.random_masks(n, m - 6, rng)
    masks = masks[:m]
    msgs = [b"block %d" % k for k in range(m)]
    sigs = _rows(r.signatures(engine, masks, msgs), sig_bytes)
    want = [OK] * m
    msgs[7] = b"another block"; want[7] = INVALID                           # wrong message
    sigs[8] = sigs[9]; want[8] = INVALID                                    # a signature made for a different mask
    sigs[10] = b"\xff" * sig_bytes; want[10] = SIG                          # does not decode
    sigs[11] = _non_subgroup_sig(group, rng); want[11] = SIG                # on the curve, outside the subgroup
    assert masks[0] == bc.mask_of(n, [])
    sigs[0] = b"\xc0" + bytes(sig_bytes - 1)                                # empty mask, infinity signature: OK
    masks[12] = bc.mask_of(n, []); sigs[12] = sigs[13]; want[12] = INVALID  # empty mask, a real signature
    st = engine.bdn_verify(group, r.terms, masks, msgs, b"".join(sigs), dst)
    assert list(st) == want
    # the same statuses as today's path: one MSM per mask, then bls.Verify under the compressed aggregate
    fac = bc.scalars_be(r.factors, o.R)
    dec, _ = (engine.bls12381_g2_decompress if group == "bls12381_g2" else engine.bls12381_g1_decompress)(r.pubs)
    keys = _rows(dec, r.operand)
    sample = [k for k in range(1, 16) if any(masks[k])]
    aggs = [engine._call(f"b2k_{group}_msm", sum(bc.bit(masks[k], i) for i in range(n)),
                         b"".join(fac[32 * i:32 * i + 32] for i in range(n) if bc.bit(masks[k], i)),
                         b"".join(keys[i] for i in range(n) if bc.bit(masks[k], i)), out=r.operand // 2) for k in sample]
    verify = engine.bls12381_verify_g1sig if group == "bls12381_g2" else engine.bls12381_verify_g2sig
    ok = verify(b"".join(aggs), [msgs[k] for k in sample], dst, b"".join(sigs[k] for k in sample))
    assert [OK if v else (SIG if want[k] == SIG else INVALID) for k, v in zip(sample, ok)] == [want[k] for k in sample]


def test_single_mask_over_a_large_roster(engine):
    """m = 1 with n = 2^16: the slices, not the masks, fill the GPU"""
    n = 1 << 16
    rng = random.Random(5)
    r = Roster(engine, "bls12381_g2", n, seed=14)
    masks = [bc.mask_of(n, range(n)), bc.mask_of(n, [i for i in range(n) if rng.random() < 2 / 3]),
             bc.mask_of(n, [i for i in range(n) if rng.random() < 0.1])]
    want = _rows(r.expected_keys(engine, masks), 192)
    for k in range(3):
        assert engine.bdn_aggregate_keys("bls12381_g2", r.terms, masks[k:k + 1]) == want[k]
    msgs = [b"checkpoint"] * 3
    st = engine.bdn_verify("bls12381_g2", r.terms, masks, msgs, r.signatures(engine, masks, msgs), DST_G1)
    assert list(st) == [OK] * 3


def test_dev_forms_equal_host_forms(engine):
    import torch
    n, m = 77, 40
    rng = random.Random(33)
    for group in ("bls12381_g2", "bls12381_g1"):
        r = Roster(engine, group, n, seed=15)
        _, operand, sig_bytes, dst = SCHEMES[group]
        masks = bc.edge_masks(n, rng) + bc.random_masks(n, m - 7, rng)
        msgs = [b"m%d" % k for k in range(m)]
        sigs = r.signatures(engine, masks, msgs)
        sigs = sigs[:sig_bytes] + b"\xff" * sig_bytes + sigs[2 * sig_bytes:]
        host_keys = engine.bdn_aggregate_keys(group, r.terms, masks)
        host_st = engine.bdn_verify(group, r.terms, masks, msgs, sigs, dst)
        blob, offs = engine._pack_msgs(msgs)
        dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
        d_terms, d_masks, d_msgs, d_offs, d_dst, d_sigs = (dev(x) for x in (r.terms, b"".join(masks), blob, offs, dst, sigs))
        d_keys = torch.zeros(m * operand, dtype=torch.uint8, device="cuda")
        d_st = torch.full((m,), 255, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        engine.bdn_aggregate_keys_dev(group, n, d_terms.data_ptr(), m, d_masks.data_ptr(), d_keys.data_ptr())
        engine.bdn_verify_dev(group, n, d_terms.data_ptr(), m, d_masks.data_ptr(), d_msgs.data_ptr(), d_offs.data_ptr(),
                              d_dst.data_ptr(), len(dst), d_sigs.data_ptr(), d_st.data_ptr())
        engine.wait()
        assert bytes(d_keys.cpu().numpy()) == host_keys
        assert bytes(d_st.cpu().numpy()) == host_st
        assert host_st[1] == SIG


def test_call_errors_and_bad_roster_keys(engine):
    r = Roster(engine, "bls12381_g2", 10, seed=16)
    mask = [bc.mask_of(10, [1, 2])]
    with pytest.raises(B2KError) as e:
        engine.bdn_terms("bls12381_g2", r.pubs[:96] + b"\xff" * 96 + r.pubs[192:])
    assert e.value.code == ERR_POINT
    bad_term = bytearray(r.terms)
    bad_term[192 + 100] ^= 1                                               # off the curve
    with pytest.raises(B2KError) as e:
        engine.bdn_aggregate_keys("bls12381_g2", bytes(bad_term), mask)
    assert e.value.code == ERR_POINT
    with pytest.raises(B2KError) as e:
        engine.bdn_verify("bls12381_g2", bytes(bad_term), mask, [b"x"], b"\xc0" + bytes(47), DST_G1)
    assert e.value.code == ERR_POINT
    lib, h = engine.lib, engine.h
    out, st = bytearray(192), bytearray(1)
    assert lib.b2k_bls12381_g2_bdn_aggregate_keys(h, 0, r.terms, 1, mask[0], bytes(out)) == ERR_ARG
    assert lib.b2k_bls12381_g2_bdn_aggregate_keys(h, 10, r.terms, 0, mask[0], bytes(out)) == ERR_ARG
    assert lib.b2k_bls12381_g2_bdn_aggregate_keys(h, 10, None, 1, mask[0], bytes(out)) == ERR_ARG
    assert lib.b2k_bls12381_g2_bdn_aggregate_keys(h, (1 << 20) + 1, r.terms, 1, mask[0], bytes(out)) == ERR_ARG
    sig = b"\xc0" + bytes(47)
    offs = b"".join(x.to_bytes(4, "little") for x in (0, 1))
    assert lib.b2k_bls12381_bdn_verify_g1sig(h, 10, r.terms, 1, mask[0], b"x", offs, DST_G1, 0, sig, bytes(st)) == ERR_ARG
    assert lib.b2k_bls12381_bdn_verify_g1sig(h, 10, r.terms, 1, mask[0], b"x", offs, DST_G1, 256, sig, bytes(st)) == ERR_ARG
    dec = b"".join(x.to_bytes(4, "little") for x in (1, 0))
    assert lib.b2k_bls12381_bdn_verify_g1sig(h, 10, r.terms, 1, mask[0], b"x", dec, DST_G1, len(DST_G1), sig, bytes(st)) == ERR_ARG
    assert lib.b2k_bn256_bdn_verify_g1sig(h, 10, r.terms, 0, mask[0], b"x", offs, sig, bytes(st)) == ERR_ARG
    # the context still works after every refusal
    assert engine.bdn_aggregate_keys("bls12381_g2", r.terms, mask) == r.expected_keys(engine, mask)


def test_bn256_fixture_aggregate_key_and_verification(engine):
    pubs = b"".join(bytes.fromhex(x) for x in FX["public"])
    terms = engine.bdn_terms("bn256_g2", pubs)
    assert bytes([0x05]) == bc.mask_of(3, FX["mask_enabled"])
    assert engine.bdn_aggregate_keys("bn256_g2", terms, [bytes([0x05])]).hex() == FX["agg_key"]
    msg = FX["msg"].encode()
    st = engine.bdn_verify("bn256_g2", terms, [bytes([0x05]), bytes([0x03]), bytes([0x05]), bytes([0x00])], [msg] * 4,
                           bytes.fromhex(FX["agg_sig"]) * 2 + b"\x01" * 64 + bytes(64))
    assert list(st) == [OK, INVALID, SIG, OK]
    # a key with unreduced coordinates is the same point: its coefficient hashes the canonical re-encoding
    raw = bytearray(pubs)
    x = int.from_bytes(raw[0:32], "big")
    if x + ob.P < 1 << 256:
        raw[0:32] = (x + ob.P).to_bytes(32, "big")
        assert engine.bdn_terms("bn256_g2", bytes(raw)) == terms
