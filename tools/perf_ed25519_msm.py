"""GPU timing of the edwards25519 MSM (b2k_ed25519_msm_dev) with its stage split, next to the per-term alternative,
b2k_ed25519_mul_batch_dev (one bit-serial Point.Mul per thread) on the same inputs, at n = 2^10, 2^16 and 2^20.
Both are timed with CUDA events on the device-pointer forms after a warm-up; the card, its power limit and its maximum SM
clock are read in the same run.
Usage: python tools/perf_ed25519_msm.py --out DIR   (writes DIR/perf_ed25519_msm.txt and DIR/perf_ed25519_msm.jsonl)"""
import argparse
import json
import os
import random
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
import ed25519_msm_cases as cases  # noqa: E402

STAGES = {0: "load+decode", 2: "scan", 3: "sort", 4: "slices", 9: "fixup", 5: "chunks", 6: "window sums", 7: "horner+encode"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--check", action="store_true", help="also compare the MSM with the oracle at every n")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    info = card()
    rows, lines = [], ["card: " + info, ""]
    rng = random.Random(1)
    pool_a = [rng.randrange(1, cases.L) for _ in range(256)]
    pool = [cases.point(a) for a in pool_a]

    def timed(call, reps):
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    for n in (1 << 10, 1 << 16, 1 << 20):
        scalars = [rng.getrandbits(253) for _ in range(n)]        # Pick-style scalars below l
        s = torch.frombuffer(bytearray(cases.le(scalars)), dtype=torch.uint8).cuda()
        p = torch.frombuffer(bytearray(b"".join(pool[i % len(pool)] for i in range(n))), dtype=torch.uint8).cuda()
        o = torch.zeros(32, dtype=torch.uint8, device="cuda")
        om = torch.zeros(32 * n, dtype=torch.uint8, device="cuda")
        msm = lambda: eng.ed25519_msm_dev(n, s.data_ptr(), p.data_ptr(), o.data_ptr())
        mul = lambda: eng.call_dev("b2k_ed25519_mul_batch_dev", n, s.data_ptr(), p.data_ptr(), om.data_ptr())
        reps = max(5, min(200, int(2e7 // n)))
        ms_msm = timed(msm, reps)
        msm()
        eng.wait()
        stages = eng.last_timings()
        plan = eng.last_msm_plan()
        if args.check:
            want = cases.msm_expected(scalars, [(pool_a[i % len(pool_a)], 0) for i in range(n)])
            assert bytes(o.cpu().numpy().tobytes()) == want, n
        ms_mul = timed(mul, max(3, reps // 20))
        eng.wait()
        row = {"n": n, "msm_ms": ms_msm, "mul_batch_ms": ms_mul, "speedup": ms_mul / ms_msm, "reps": reps,
               "c": plan["c"], "W": plan["W"], "slice_len": plan["slice_len"],
               "stages_ms": {name: stages[i] for i, name in STAGES.items()}, "pipeline_ms": stages[8]}
        rows.append(row)
    lines.append("%9s %11s %15s %8s  %s" % ("n", "MSM ms", "mul_batch ms", "ratio", "MSM stages (ms, one call)"))
    for r in rows:
        st = "  ".join("%s %.3f" % (k, v) for k, v in r["stages_ms"].items())
        lines.append("%9d %11.4f %15.4f %8.1f  c=%d W=%d L=%d  %s" % (r["n"], r["msm_ms"], r["mul_batch_ms"], r["speedup"], r["c"],
                                                                   r["W"], r["slice_len"], st))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_ed25519_msm.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_ed25519_msm.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
