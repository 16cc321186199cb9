"""GPU timing of ECIES on edwards25519 (b2k_ed25519_ecies_encrypt / _decrypt), or on BLS12-381 with keys on G1 or G2
(b2k_bls12381_g{1,2}_ecies_encrypt / _decrypt, --group): whole calls for n = 2^10 .. 2^20 ciphertexts with 32-byte messages
(one DKG share) and 1 KiB messages.  Inputs are tiled from 1024 distinct (r, message) pairs to one
public key; the decryption times the ciphertexts the encryption produced, and every status and every decrypted message is
checked before timing.  Every size is timed in ROUNDS separate rounds (encryption and decryption alternating, the inputs
kept), and the table gives the median rate with the lowest and highest round beside it.  For information, beside them: the
decryption of an empty body (one constant-time variable-base multiplication, the Fermat inversion, HKDF and the GCM set-up)
against b2k_ed25519_mul_batch (variable-time double-and-add and binary-GCD inversion) at the same n (edwards25519 only).  The
card's name, power limit and maximum SM clock are read in the same run.
Usage: python tools/perf_ecies.py --out DIR [--group ed25519 | --group bls12381_g1 bls12381_g2]
  (edwards25519, the default: writes DIR/h100_perf_ecies.{txt,jsonl}; BLS12-381: DIR/h100_perf_ecies_bls12381.{txt,jsonl}, one
  table per group; the committed records are profiles/h100_perf_ecies*, so --out profiles regenerates them on an H100)"""
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
from oracle import bls12381 as bls  # noqa: E402
from oracle import ecies as ec  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ecies_bls12381_oracle as eb  # noqa: E402

SIZES = [1 << k for k in (10, 12, 14, 16, 18, 20)]
LENGTHS = [32, 1024]
TILE = 1024
ROUNDS = 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(call, min_s=1.0, min_reps=3):
    call()
    torch.cuda.synchronize()
    reps, t0 = 0, time.perf_counter()
    while True:
        call()
        reps += 1
        if time.perf_counter() - t0 >= min_s and reps >= min_reps:
            break
    return (time.perf_counter() - t0) / reps * 1e3, reps


class Ed25519:
    """the calls and keys of one group"""
    name, lengths = "ed25519", LENGTHS + [0]

    def __init__(self, eng, rng):
        self.eng = eng
        self.priv = rng.randbytes(32)
        self.pub = ec.mul(self.priv)

    def scalar(self, rng):
        return rng.randbytes(32)

    def encrypt(self, P, R, M):
        return self.eng.ed25519_ecies_encrypt(P, R, M)

    def decrypt(self, cts, length):
        return self.eng.ed25519_ecies_decrypt(self.priv, cts, length)

    def oracle(self, r, m):
        return ec.encrypt(self.pub, r, m)[1]


class Bls12381(Ed25519):
    lengths = LENGTHS

    def __init__(self, eng, rng, group):
        self.eng, self.group, self.name = eng, group, f"bls12381_g{group}"
        self.priv = self.scalar(rng)
        self.pub = eb.public(group, self.priv)

    def scalar(self, rng):
        return rng.randrange(bls.R).to_bytes(32, "big")

    def encrypt(self, P, R, M):
        return self.eng.bls12381_ecies_encrypt(self.group, P, R, M)

    def decrypt(self, cts, length):
        return self.eng.bls12381_ecies_decrypt(self.group, self.priv, cts, length)

    def oracle(self, r, m):
        return eb.encrypt(self.group, self.pub, r, m)[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--group", nargs="+", choices=["ed25519", "bls12381_g1", "bls12381_g2"], default=["ed25519"])
    args = ap.parse_args()
    if "ed25519" in args.group and len(args.group) > 1:
        ap.error("ed25519 and the BLS12-381 groups go to different records: run them separately")
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    info = card()
    print("card:", info, flush=True)
    rows = []
    for gname in args.group:
        if gname == "ed25519":
            rng = random.Random("perf/ecies")
            g = Ed25519(eng, rng)
        else:
            rng = random.Random("perf/ecies/" + gname)
            g = Bls12381(eng, rng, int(gname[-1]))
        rows += run_group(eng, g, rng)
    write(args.out, "h100_perf_ecies" if args.group == ["ed25519"] else "h100_perf_ecies_bls12381", info, rows,
          bls_groups=args.group != ["ed25519"])
    eng.close()


def run_group(eng, g, rng):
    rows = []
    pub = g.pub
    for length in g.lengths:
        rs = [g.scalar(rng) for _ in range(TILE)]
        msgs = [rng.randbytes(length) for _ in range(TILE)]
        for n in SIZES:
            R, M = [rs[i % TILE] for i in range(n)], [msgs[i % TILE] for i in range(n)]
            P = [pub] * n
            cts, st = g.encrypt(P, R, M)
            assert st == bytes(n) and cts[1] == g.oracle(R[1], M[1])
            back, st = g.decrypt(cts, length + 16)
            assert st == bytes(n) and back == M, "a valid ciphertext did not decrypt"
            few = 2 if n >= 1 << 18 else 3
            calls = []
            if length:
                calls.append(("encrypt", length, lambda: g.encrypt(P, R, M)))
            calls.append(("decrypt", length, lambda: g.decrypt(cts, length + 16)))
            if length == 0:                                      # the variable-time batch multiplication at the same n
                ks, pts = b"".join(R), pub * n
                calls.append(("mul_batch (variable time)", None, lambda: eng.ed25519_mul_batch(ks, pts)))
            runs = {name: [] for name, _, _ in calls}
            for _ in range(ROUNDS):
                for name, _, call in calls:
                    runs[name].append(timed(call, min_s=0.5, min_reps=few))
            for name, ln, _ in calls:
                rates = sorted(n / ms * 1e3 for ms, _ in runs[name])
                rows.append({"group": g.name, "call": name, "len": ln, "n": n, "per_s": rates[len(rates) // 2], "per_s_min": rates[0],
                             "per_s_max": rates[-1], "ms_rounds": [ms for ms, _ in runs[name]],
                             "reps_rounds": [r for _, r in runs[name]]})
                print(json.dumps(rows[-1]), flush=True)
            del cts, back
    return rows


def write(out, stem, info, rows, bls_groups):
    lines = ["card: " + info,
             "whole host calls (inputs staged, outputs copied back, staged bytes cleared, synchronised), after one warm-up call; "
             "every status OK and every message round-tripped before timing; %d rounds per size, median rate with the lowest "
             "and highest round" % ROUNDS]
    if not bls_groups:
        lines.append("len 0 rows: decryption of an empty body = one constant-time variable-base multiplication + Fermat inversion + "
                     "HKDF + GCM set-up, beside b2k_ed25519_mul_batch at the same n (for information)")
    lines.append("")
    lines.append("%-26s %6s %9s %13s %13s %13s  %s" % ("call", "len", "n", "median /s", "lowest /s", "highest /s", "reps per round"))
    for r in rows:
        call = r["call"] if not bls_groups else r["group"] + " " + r["call"]
        lines.append("%-26s %6s %9d %13.4g %13.4g %13.4g  %s" % (call, "-" if r["len"] is None else r["len"], r["n"],
                                                               r["per_s"], r["per_s_min"], r["per_s_max"],
                                                               " ".join(str(x) for x in r["reps_rounds"])))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(out, stem + ".txt"), "w") as f:
        f.write(text)
    with open(os.path.join(out, stem + ".jsonl"), "w") as f:
        for r in rows:
            if not bls_groups:
                r = {k: v for k, v in r.items() if k != "group"}
            f.write(json.dumps(dict(r, card=info)) + "\n")


if __name__ == "__main__":
    main()
