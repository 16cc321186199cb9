"""GPU timing of sign/bdn's verifier batch on BLS12-381, both schemes: b2k_bls12381_g{2,1}_bdn_aggregate_keys (AggregatePublicKeys
for m masks) and b2k_bls12381_bdn_verify_g{1,2}sig (bls.Verify under every aggregate), for rosters n in {128, 1024, 8192},
m in {1, 64, 1024, 16384} and masks full / 90 % / 2/3 / 50 %.  In the same process, alternating with them, today's path: one
b2k_bls12381_g{2,1}_msm per mask over (c_i + 1, PK_i), then b2k_bls12381_verify_g{1,2}sig under the aggregates -- at m <= 64
for every density and at m = 1024 for 2/3 masks (one blocking MSM call per mask makes the rest minutes long).  Its per-mask
MSM inputs are selected before the timed region.  Masks and
signatures are tiled from 64 distinct masks with valid signatures; both paths must give the same statuses (all OK).  Every
row is the median of ROUNDS rounds with the lowest and highest beside it.  The card's name and power limit are read in the same run.
Usage: python tools/perf_bdn.py --out DIR   (writes DIR/h100_perf_bdn.txt and DIR/h100_perf_bdn.jsonl; the committed records
are profiles/h100_perf_bdn.*, so --out profiles regenerates them on an H100)"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import bdn_cases as bc  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
from oracle import bls12381 as o  # noqa: E402

ROSTERS = [128, 1024, 8192]
MASKS = [1, 64, 1024, 16384]
DENSITIES = [("full", 1.0), ("90%", 0.9), ("2/3", 2 / 3), ("50%", 0.5)]
TILE = 64
ROUNDS = 3
DST = {"bls12381_g2": b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_", "bls12381_g1": b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def ms(call):
    t0 = time.perf_counter()
    out = call()
    return (time.perf_counter() - t0) * 1e3, out


def roster(eng, group, n, rng):
    xs = [rng.randrange(1, o.R) for _ in range(n)]
    g2 = group == "bls12381_g2"
    base = o.g2_to_affine_bytes(o.G2) if g2 else o.g1_to_affine_bytes(o.G1)
    pubs = (eng.bls12381_g2_mul_batch if g2 else eng.bls12381_g1_mul_batch)(bc.scalars_be(xs, o.R), base * n)
    wire = 96 if g2 else 48
    fac = eng.bdn_coefficients(pubs, wire, add_one=True)
    factors = [int.from_bytes(fac[32 * i:32 * i + 32], "big") for i in range(n)]
    dec, ok = (eng.bls12381_g2_decompress if g2 else eng.bls12381_g1_decompress)(pubs)
    assert set(ok) == {1}
    return xs, factors, fac, dec, eng.bdn_terms(group, pubs)


def tile(eng, group, n, density, xs, factors, rng):
    """TILE masks of the density (exact popcount), their messages and valid signatures"""
    k = max(1, round(density * n))
    masks = [bc.mask_of(n, rng.sample(range(n), k)) for _ in range(TILE)]
    msgs = [b"block %d" % i for i in range(TILE)]
    scal = bc.scalars_be([bc.mask_scalar(factors, xs, mk, n, o.R) for mk in masks], o.R)
    if group == "bls12381_g2":
        sigs = eng.bls12381_g1_mul_batch(scal, eng.bls12381_hash_to_g1(msgs, DST[group]))
    else:
        sigs = eng.bls12381_g2_mul_batch(scal, eng.bls12381_hash_to_g2(msgs, DST[group]))
    return masks, msgs, sigs


def selections(group, n, fac, dec, masks):
    """per mask, the MSM inputs of today's path: (count, factors, decoded keys) of the enabled members -- built before timing"""
    op = 192 if group == "bls12381_g2" else 96
    out = []
    for mk in masks:
        en = [i for i in range(n) if bc.bit(mk, i)]
        out.append((len(en), b"".join(fac[32 * i:32 * i + 32] for i in en), b"".join(dec[op * i:op * i + op] for i in en)))
    return out


def today(eng, group, sel, msgs, sigs):
    """one MSM per mask (inputs selected beforehand), then bls.Verify under the compressed aggregates
    -> (statuses (0 ok, 2 invalid), ms of the MSM calls alone)"""
    op = 192 if group == "bls12381_g2" else 96
    t_msm, aggs = ms(lambda: [eng._call(f"b2k_{group}_msm", cnt, scal, pts, out=op // 2) for cnt, scal, pts in sel])
    verify = eng.bls12381_verify_g1sig if group == "bls12381_g2" else eng.bls12381_verify_g2sig
    ok = verify(b"".join(aggs), msgs, DST[group], sigs)
    return bytes(0 if v else 2 for v in ok), t_msm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    info = card()
    print("card:", info, flush=True)
    rng = random.Random("perf/bdn")
    rows = []
    for group in ("bls12381_g2", "bls12381_g1"):
        sig_bytes = 48 if group == "bls12381_g2" else 96
        for n in ROSTERS:
            xs, factors, fac, dec, terms = roster(eng, group, n, rng)
            for dname, dens in DENSITIES:
                masks_t, msgs_t, sigs_t = tile(eng, group, n, dens, xs, factors, rng)
                sel_t = selections(group, n, fac, dec, masks_t)
                for m in MASKS:
                    masks = [masks_t[i % TILE] for i in range(m)]
                    msgs = [msgs_t[i % TILE] for i in range(m)]
                    sigs = b"".join(sigs_t[sig_bytes * (i % TILE):sig_bytes * (i % TILE + 1)] for i in range(m))
                    base = m <= 64 or (m == 1024 and dname == "2/3")
                    agg_t, ver_t, old_t, msm_t = [], [], [], []
                    for _ in range(ROUNDS):
                        t, _keys = ms(lambda: eng.bdn_aggregate_keys(group, terms, masks))
                        agg_t.append(t)
                        t, st = ms(lambda: eng.bdn_verify(group, terms, masks, msgs, sigs, DST[group]))
                        ver_t.append(t)
                        assert set(st) == {0}, (group, n, dname, m)
                        if base:
                            sel = [sel_t[i % TILE] for i in range(m)]
                            t, (st_old, t_msm) = ms(lambda: today(eng, group, sel, msgs, sigs))
                            old_t.append(t)
                            msm_t.append(t_msm)
                            assert st_old == st
                    row = {"scheme": "keys G2 / sigs G1" if group == "bls12381_g2" else "keys G1 / sigs G2", "n": n, "m": m,
                           "masks": dname, "aggregate_ms": [statistics.median(agg_t), min(agg_t), max(agg_t)],
                           "verify_ms": [statistics.median(ver_t), min(ver_t), max(ver_t)],
                           "per_mask_msm_then_verify_ms": [statistics.median(old_t), min(old_t), max(old_t)] if old_t else None,
                           "of_which_msm_calls_ms": [statistics.median(msm_t), min(msm_t), max(msm_t)] if msm_t else None,
                           "card": info}
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    with open(os.path.join(args.out, "h100_perf_bdn.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    with open(os.path.join(args.out, "h100_perf_bdn.txt"), "w") as f:
        f.write(f"sign/bdn verifier batch, BLS12-381 -- {info}\n")
        f.write(f"median of {ROUNDS} rounds [min, max], ms per call; today = one MSM per mask + verify (blocking calls)\n")
        f.write(f"{'scheme':20s} {'n':>5s} {'m':>6s} {'masks':>5s} {'aggregate':>26s} {'bdn verify':>26s} {'today':>26s}\n")
        fmt = lambda v: "-" if v is None else f"{v[0]:9.3f} [{v[1]:.3f}, {v[2]:.3f}]"
        for r in rows:
            f.write(f"{r['scheme']:20s} {r['n']:5d} {r['m']:6d} {r['masks']:>5s} {fmt(r['aggregate_ms']):>26s} "
                    f"{fmt(r['verify_ms']):>26s} {fmt(r['per_mask_msm_then_verify_ms']):>26s}\n")
    eng.close()


if __name__ == "__main__":
    main()
