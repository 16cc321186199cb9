"""Per-kernel time of one BLS12-381 G1 MSM over 2^20 distinct pairs resident on the device (the shape bench.py measures),
taken with torch.profiler (CUDA activities) in a run of its own.  Usage:

    python tools/perf_kernels.py OUTDIR [--rounds R] [--batch B] [--split 0|1] [--msms K] [--set uniform|equal|bdn128]

The MSM is warmed up outside the profiler, then K MSMs (default 1) run back to back on one stream under it.  Written to OUTDIR:
kernels.txt (table: kernel, launches per MSM, total / mean microseconds per MSM, share of the MSM's device span) and kernels.json
(the same rows plus the GPU's name, power limit and the plan the MSMs ran with).  Every MSM's output is checked against the oracle.
--set picks the input: uniform scalars and distinct points (default), one (s, P) repeated 2^20 times (every window's entries in one
bucket), or 128-bit BDN-style factors (s mod 2^128 + 1) over the distinct points."""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def short_name(name: str) -> str:
    """'void b2k::k_pt_forward<b2k::Bls381G1, true>(unsigned int, ...)' -> 'k_pt_forward<Bls381G1, true>'"""
    name = re.sub(r"^void\s+", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return re.sub(r"\b(b2k|b2k_host)::", "", name[:cut]).strip()


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, plim = [x.strip() for x in q.split(",")]
        return name, plim
    except Exception:   # noqa: BLE001 -- the table is still worth writing without them
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--rounds", type=int, default=-1, help="affine pair-tree rounds (-1 = the library's automatic plan)")
    ap.add_argument("--batch", type=int, default=0, help="outputs per thread of a round (0 = automatic)")
    ap.add_argument("--split", type=int, default=1, help="1 = split round kernels (library default), 0 = fused")
    ap.add_argument("--msms", type=int, default=1, help="MSMs inside the profiled region")
    ap.add_argument("--set", default="uniform", choices=("uniform", "equal", "bdn128"), help="input set (skewed scalars: equal, bdn128)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from kyber_b200 import workload as wl
    from kyber_b200.capi import Engine
    from oracle import bls12381 as o

    n = 1 << 20
    eng = Engine(0)
    eng.set_msm_affine_split(bool(args.split))
    eng.set_msm_affine(args.rounds, args.batch)
    a = wl.prng_scalars("b2k/c2-a", n, o.R)
    s = wl.prng_scalars("b2k/c2", n, o.R)
    if args.set == "equal":
        a, s = [a[0]] * n, [s[0]] * n
    elif args.set == "bdn128":
        s = [x % (1 << 128) + 1 for x in s]
    base = eng.bls12381_g1_mul_batch_affine(wl.scalars_to_bytes(a), wl.G1_BLS12381_AFFINE * n)
    want = o.g1_compress(o.g1_mul(wl.dot_mod(s, a, o.R)))
    pts = torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()
    sc = torch.frombuffer(bytearray(wl.scalars_to_bytes(s)), dtype=torch.uint8).cuda()
    out = torch.zeros(256, dtype=torch.uint8, device="cuda")

    def msm():
        eng.call_dev("b2k_bls12381_g1_msm_dev", n, sc.data_ptr(), pts.data_ptr(), out.data_ptr())

    for _ in range(3):
        msm()
    eng.synchronize()
    l0 = eng.launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.msms):
            msm()
        eng.synchronize()
    launches = (eng.launch_count() - l0) / args.msms
    got = bytes(out[:48].cpu().numpy())
    assert got == want, "MSM differs from the oracle"

    rows, t_lo, t_hi = {}, None, None
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.time_range.elapsed_us()
        t_lo = e.time_range.start if t_lo is None else min(t_lo, e.time_range.start)
        t_hi = e.time_range.end if t_hi is None else max(t_hi, e.time_range.end)
        k = short_name(e.name)
        c, t = rows.get(k, (0, 0.0))
        rows[k] = (c + 1, t + us)
    span = (t_hi - t_lo) / args.msms
    K = args.msms
    table = sorted(((k, c / K, t / K, t / c, t / K / span) for k, (c, t) in rows.items()), key=lambda r: -r[2])
    busy = sum(r[2] for r in table)
    gname, plim = gpu_info()
    plan = eng.last_msm_plan()
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "kernels.txt"), "w") as f:
        f.write(f"# BLS12-381 G1 MSM, 2^20 pairs ({args.set} set), one stream, {K} MSM(s) under torch.profiler (CUDA activities); per MSM\n")
        f.write(f"# GPU: {gname}, power limit {plim}; plan: {json.dumps(plan)}\n")
        f.write(f"# device span {span / 1e3:.3f} ms per MSM, kernels + memsets busy {busy / 1e3:.3f} ms, {launches:.0f} library launches\n")
        f.write(f"{'kernel':72s} {'count':>6s} {'total_us':>10s} {'mean_us':>9s} {'share':>6s}\n")
        for k, c, t, m, sh in table:
            f.write(f"{k[:72]:72s} {c:6.1f} {t:10.1f} {m:9.1f} {100 * sh:5.1f}%\n")
    with open(os.path.join(args.outdir, "kernels.json"), "w") as f:
        json.dump({"set": args.set, "gpu": gname, "power_limit": plim, "msms": K, "span_us_per_msm": span, "busy_us_per_msm": busy,
                   "launches_per_msm": launches, "plan": plan,
                   "kernels": [{"name": k, "count": c, "total_us": t, "mean_us": m, "share": sh} for k, c, t, m, sh in table]}, f, indent=1)
    print(open(os.path.join(args.outdir, "kernels.txt")).read())
    eng.close()


if __name__ == "__main__":
    main()
