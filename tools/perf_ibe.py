"""GPU timing of Boneh-Franklin IBE (CCA) on BLS12-381: decrypts/s of b2k_bls12381_ibe_decrypt_cca_g1 / _g2 and encrypts/s of
b2k_bls12381_ibe_encrypt_cca_g1 / _g2 at n = 2^10 .. 2^18 messages of 16 bytes (one key, one identity: the timelock case), and the
alternating A/B of the fixed-G2 Miller loop (b2k_bls12381_pair_fixed_g2) against the pairing launcher (b2k_bls12381_pair with the
G2 operand repeated n times) on the same inputs at n >= 2^14, outputs compared byte for byte.  Host-buffer calls, times from a host
clock around the blocking call (each call ends in a stream synchronise); B's input copy carries 192 n more bytes than A's.
Usage: python tools/perf_ibe.py --out DIR   (writes DIR/perf_ibe.txt and DIR/perf_ibe.jsonl)"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
from oracle import bls12381 as o  # noqa: E402
from oracle import ibe  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()                                                  # warm-up of this shape
    best = []
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        best.append(time.perf_counter() - t)
    return min(best), sorted(best)[len(best) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--max-log2", type=int, default=18)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_ibe needs a GPU")
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    lines, rows = [], []

    def emit(rec):
        rows.append(rec)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    emit({"card": card(), "coop_max_n": 10240})
    rng = random.Random(1)
    ident = b"round 4242"
    for on in (1, 2):
        master, priv = ibe.keypair(on, rng.randrange(1, o.R), ident)
        for lg in range(10, args.max_log2 + 1, 2):
            n = 1 << lg
            msgs = [rng.randbytes(16) for _ in range(n)]
            sigmas = [rng.randbytes(16) for _ in range(n)]
            te, tem, (u, v, w) = timed(lambda: eng.bls12381_ibe_encrypt(on, master, ident, msgs, sigmas), args.reps)
            td, tdm, (got, st) = timed(lambda: eng.bls12381_ibe_decrypt(on, priv, u, v, w), args.reps)
            assert st == bytes(n) and got == msgs, "round trip failed"
            emit({"op": f"ibe_on_g{on}", "n": n, "encrypt_s": te, "encrypt_median_s": tem, "encrypts_per_s": n / te,
                  "decrypt_s": td, "decrypt_median_s": tdm, "decrypts_per_s": n / td})

    # A/B: fixed-G2 Miller loop vs the pairing launcher, alternating, same inputs
    q = o.g2_to_affine_bytes(o.g2_mul(rng.randrange(1, o.R)))
    base = [o.g1_to_affine_bytes(o.g1_mul(rng.randrange(1, o.R))) for _ in range(64)]
    for lg in range(14, args.max_log2 + 1, 2):
        n = 1 << lg
        g1 = b"".join(base[i % 64] for i in range(n))
        g2n = q * n
        a_out = eng.bls12381_pair_fixed_g2(g1, q)
        b_out = eng.bls12381_pair(g1, g2n)
        assert a_out == b_out, "fixed-G2 pairing differs from the launcher"
        ta, tb = [], []
        for _ in range(2 * args.reps):
            t = time.perf_counter(); eng.bls12381_pair_fixed_g2(g1, q); ta.append(time.perf_counter() - t)
            t = time.perf_counter(); eng.bls12381_pair(g1, g2n); tb.append(time.perf_counter() - t)
        emit({"op": "ab_pair_fixed_g2_vs_launcher", "n": n, "outputs_equal": True, "fixed_g2_s": sorted(ta), "launcher_s": sorted(tb),
              "fixed_g2_pairs_per_s": n / min(ta), "launcher_pairs_per_s": n / min(tb), "speedup_min": min(tb) / min(ta)})
    eng.close()
    with open(os.path.join(args.out, "perf_ibe.jsonl"), "w") as f:
        f.write("\n".join(lines) + "\n")
    with open(os.path.join(args.out, "perf_ibe.txt"), "w") as f:
        f.write(f"card: {rows[0]['card']}\n")
        f.write(f"{'op':<30}{'n':>8}{'enc/s':>12}{'dec/s':>12}\n")
        for r in rows[1:]:
            if r["op"].startswith("ibe"):
                f.write(f"{r['op']:<30}{r['n']:>8}{r['encrypts_per_s']:>12.0f}{r['decrypts_per_s']:>12.0f}\n")
        f.write(f"\n{'A/B (best of runs)':<30}{'n':>8}{'fixed/s':>12}{'launch/s':>12}{'speedup':>9}\n")
        for r in rows[1:]:
            if r["op"].startswith("ab"):
                f.write(f"{'fixed-G2 vs launcher':<30}{r['n']:>8}{r['fixed_g2_pairs_per_s']:>12.0f}{r['launcher_pairs_per_s']:>12.0f}"
                        f"{r['speedup_min']:>9.3f}\n")


if __name__ == "__main__":
    main()
