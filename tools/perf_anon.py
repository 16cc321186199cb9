"""GPU timing of ring signature verification on edwards25519 (b2k_ed25519_anon_verify): whole calls for m = 1, 2^10, 2^14 and
2^16 signatures over rings of n = 10 and 100 keys, and m = 2^10 over n = 1000, unlinkable and linkable.  The batches are tiled
from 4 distinct signatures per (n, mode), signed with b2k_ed25519_mul_batch doing the signer's multiplications; every status is
checked OK before timing.  The kernel split of each size comes from one torch.profiler run of its own.  Beside each row: the
Point.Mul count of one reference verification (2n unlinkable, 4n linkable).
Usage: python tools/perf_anon.py --out DIR   (writes DIR/perf_anon.txt and DIR/perf_anon.jsonl)"""
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
import anon_cases as ac  # noqa: E402
import pvss_cases as pc  # noqa: E402

STAGES = ("k_anon_setup", "k_anon_link_base", "k_anon_tables", "k_anon_ring_step", "k_anon_finish")
SIZES = [(m, n) for n in (10, 100) for m in (1, 1 << 10, 1 << 14, 1 << 16)] + [(1 << 10, 1000)]
SCOPE = b"perf scope"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def signatures(eng, n, scope, count=4):
    """(ring, msgs, sigs): count signatures by random members of a random ring of n keys"""
    def mul(k, p):
        return eng.ed25519_mul_batch(k.to_bytes(32, "little"), p if p is not None else pc.G)
    rng = random.Random(f"perf/{n}/{scope}")
    keys = [rng.randrange(1, ac.L) for _ in range(n)]
    ring_blob = eng.ed25519_mul_batch(b"".join(k.to_bytes(32, "little") for k in keys), pc.G * n)
    ring = [ring_blob[32 * i:32 * i + 32] for i in range(n)]
    rand = pc.Xof(b"perf")
    msgs, sigs = [], []
    for j in range(count):
        mine = rng.randrange(n)
        msgs.append(rng.randbytes(32))
        sigs.append(ac.sign(msgs[-1], ring, scope, mine, keys[mine], rand, mul=mul))
    return ring, msgs, sigs


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


def split(call):
    """kernel ms per stage of one call, in a profiler run of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    evs = [(e.time_range.start, e.time_range.end, e.name) for e in prof.events()
           if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k: sum((e - s) / 1e3 for s, e, nm in evs if k in nm) for k in STAGES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    info = card()
    print("card:", info, flush=True)
    rows, calls = [], []
    for scope in (None, SCOPE):
        base = {}
        for m, n in SIZES:
            if n not in base:
                base[n] = signatures(eng, n, scope)
            ring, msgs, sigs = base[n]
            rb, ms_, ss = b"".join(ring), [msgs[j % 4] for j in range(m)], [sigs[j % 4] for j in range(m)]
            call = (lambda rb, ms_, ss, scope: lambda: eng.ed25519_anon_verify(rb, ms_, ss, scope))(rb, ms_, ss, scope)
            assert call()[0] == bytes(m), "a valid signature was rejected"
            ms, reps = timed(call)
            calls.append(call)
            rows.append({"call": "anon_verify", "linkable": scope is not None, "m": m, "n": n, "ms": ms,
                         "sigs_per_s": m / ms * 1e3, "positions_per_s": m * n / ms * 1e3, "reps": reps,
                         "ref_point_mul_per_sig": (4 if scope is not None else 2) * n})
            print(json.dumps(rows[-1]), flush=True)
    for r, call in zip(rows, calls):
        stage = split(call)
        r.update(stage_ms=stage, kernel_ms=sum(stage.values()))
        print(json.dumps(r), flush=True)

    lines = ["card: " + info, "whole host calls (inputs staged, statuses and tags copied back, synchronised), after two warm-up "
             "calls; every status OK; kernel split from one torch.profiler run per size", ""]
    lines.append("%-10s %-22s %10s %12s %14s %10s %12s  %s" % ("mode", "size", "ms/call", "sigs/s", "positions/s", "kernel ms",
                                                              "ref Mul/sig", "kernel ms (" + ", ".join(s[7:] for s in STAGES) + ")"))
    for r in rows:
        lines.append("%-10s %-22s %10.3f %12.4g %14.4g %10.3f %12d  %s" % (
            "linkable" if r["linkable"] else "unlinkable", "m=%d n=%d" % (r["m"], r["n"]), r["ms"], r["sigs_per_s"],
            r["positions_per_s"], r["kernel_ms"], r["ref_point_mul_per_sig"], " ".join("%.3f" % r["stage_ms"][s] for s in STAGES)))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_anon.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_anon.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
