"""GPU timing of Neff shuffle verification on edwards25519 (b2k_ed25519_shuffle_verify): whole calls for m = 1 shuffle of
k = 2^10, 2^14 and 2^17 pairs and for m = 100 shuffles of k = 1000, with honest proofs (every status checked OK), and the split
between the host transcript and the device kernels from torch.profiler.  Beside each row: the variable-base Point.Mul count of
one reference verification (10k + 4: B, 2k thver, Phi1 / Phi2, (33), U, W, (34), (35)).
Usage: python tools/perf_shuffle.py --out DIR   (writes DIR/perf_shuffle.txt and DIR/perf_shuffle.jsonl)"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
import shuffle_cases as sc  # noqa: E402

L = sc.L
STAGES = ("k_shuffle_decode", "k_shuffle_uw", "k_shuffle_thver", "k_shuffle_pair_terms", "k_shuffle_resolve")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def honest(eng, k, seed):
    """one honest shuffle of k pairs, built on discrete logs (shuffle_cases.DlogOps) and encoded by b2k_ed25519_mul_batch"""
    def mul_base(ks):
        out = eng.ed25519_mul_batch(b"".join(sc.le(v) for v in ks), sc.G * len(ks))
        return [out[i:i + 32] for i in range(0, len(out), 32)]
    ops = sc.DlogOps(mul_base)
    rng = random.Random(seed)
    hd = rng.randrange(1, L)
    X, Y = sc.elgamal_pairs(k, rng, hd, ops)
    Xb, Yb, prf = sc.shuffle(None, hd, X, Y, b"PairShuffle", seed, ops)
    enc = ops.enc(X + Y + Xb + Yb + [hd])
    return [b"".join(enc[q * k:(q + 1) * k]) for q in range(4)], prf, enc[-1]


def timed(call, min_s=1.0):
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    reps, t0 = 0, time.perf_counter()
    while True:
        call()
        reps += 1
        if time.perf_counter() - t0 >= min_s and reps >= 3:
            break
    return (time.perf_counter() - t0) / reps * 1e3, reps


def split(calls):
    """per call: kernel ms per stage, and the host window, from the call's first device operation to the start of the Zrho / t, c
    copies (the two host-to-device copies right before k_shuffle_uw), which wait for the transcript; the staging copies and the
    decode overlap it.  The calls run once each in one profiler session (a second session records no CUDA events here) and
    are told apart by their k_shuffle_resolve."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in calls:
            call()
            torch.cuda.synchronize()
    evs = sorted((e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA)
    out, seg = [], []
    for ev in evs:
        seg.append(ev)
        if "k_shuffle_resolve" in ev[2]:
            stage = {k: sum((e - s) / 1e3 for s, e, n in seg if k in n) for k in STAGES}
            uw = [s for s, _, n in seg if "k_shuffle_uw" in n]
            h2d = [s for s, _, n in seg if "HtoD" in n and uw and s < uw[0]]
            out.append((stage, (h2d[-2] - seg[0][0]) / 1e3 if len(h2d) >= 2 else None))
            seg = []
    assert len(out) == len(calls), "the profiler trace does not hold one k_shuffle_resolve per call"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    info = card()
    rows = []
    calls = []
    for m, k in ((1, 1 << 10), (1, 1 << 14), (1, 1 << 17), (100, 1000)):
        t0 = time.perf_counter()
        (x, y, xb, yb), prf, h = honest(eng, k, "perf %d %d" % (m, k))
        build_s = time.perf_counter() - t0
        call = (lambda k, a: lambda: eng.ed25519_shuffle_verify(k, *a))(k, (x * m, y * m, xb * m, yb * m, prf * m, b"PairShuffle",
                                                                            None, h * m))
        assert call() == bytes(m), "an honest shuffle was rejected"
        ms, reps = timed(call)
        calls.append(call)
        rows.append({"call": "shuffle_verify", "m": m, "k": k, "ms": ms, "pairs_per_s": m * k / ms * 1e3, "reps": reps,
                     "ref_point_mul_per_shuffle": 10 * k + 4, "input_build_s": build_s})
        print(json.dumps(rows[-1]), flush=True)
    for r, (stage, host) in zip(rows, split(calls)):
        r.update(stage_ms=stage, kernel_ms=sum(stage.values()), host_window_ms=host)
        print(json.dumps(r), flush=True)

    lines = ["card: " + info, "whole host calls (inputs staged, transcript on host threads, status copied back), after two "
             "warm-up calls; honest proofs, every status OK", ""]
    lines.append("%-14s %10s %10s %10s %12s %12s %10s  %s" % ("size", "ms/call", "pairs/s", "kernel ms", "host window", "ref Mul/shuf",
                                                              "", "kernel ms (decode, uw, thver, pair_terms, resolve)"))
    for r in rows:
        lines.append("%-14s %10.3f %10.4g %10.3f %12.3f %12d %10s  %s" % (
            "m=%d k=%d" % (r["m"], r["k"]), r["ms"], r["pairs_per_s"], r["kernel_ms"], r["host_window_ms"] or float("nan"),
            r["ref_point_mul_per_shuffle"], "", " ".join("%.3f" % r["stage_ms"][s] for s in STAGES)))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_shuffle.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_shuffle.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
