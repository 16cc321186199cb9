"""A/B: BLS12-381 G1 MSM, 2^20 distinct pairs resident on the device, with 0..R affine pair-tree rounds in front of the
XYZZ slices, fused or split rounds, several batch widths.  Per variant: the stage timings of single MSMs (the library's CUDA
events) and the throughput with 4 MSMs in flight on 4 contexts (bench.py's shape), ms per MSM; every variant must give the
oracle's bytes.  `--profile`: run exactly one fused and one split single-round MSM (for a profiler).  `--out FILE`: also write
the rows as JSON lines."""
import json
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from kyber_b200 import workload as wl
from kyber_b200.capi import Engine
from oracle import bls12381 as o

profile = "--profile" in sys.argv
out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
n = 1 << 20
NC = 4
eng = Engine(0)
a = wl.prng_scalars("b2k/c2-a", n, o.R)
s = wl.prng_scalars("b2k/c2", n, o.R)
base = eng.bls12381_g1_mul_batch_affine(wl.scalars_to_bytes(a), wl.G1_BLS12381_AFFINE * n)
want = o.g1_compress(o.g1_mul(wl.dot_mod(s, a, o.R))).hex()
pts = torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()
sc = torch.frombuffer(bytearray(wl.scalars_to_bytes(s)), dtype=torch.uint8).cuda()
streams = [torch.cuda.Stream() for _ in range(NC)]
engines = [eng] + [Engine(0) for _ in range(NC - 1)]
for e, st in zip(engines, streams):
    e.set_stream(st.cuda_stream)
outs = [torch.zeros(256, dtype=torch.uint8, device="cuda") for _ in range(NC)]
names = ["load", "digits_hist", "scan", "scatter", "accumulate", "reduce_chunks", "window_sum", "final", "pipeline", "fixup", "rounds"]
rows = []


def msm(j):
    engines[j].call_dev("b2k_bls12381_g1_msm_dev", n, sc.data_ptr(), pts.data_ptr(), outs[j].data_ptr())


def run(split, rounds, batch, K, steps=24):
    for e in engines:
        e.set_msm_affine_split(bool(split))
        e.set_msm_affine(rounds, batch)
    acc = None
    for k in range(K + (0 if profile else 3)):
        msm(0); eng.synchronize()
        if profile or k >= 3:
            t = eng.last_timings()
            acc = t if acc is None else [x + y for x, y in zip(acc, t)]
    ok = bytes(outs[0][:48].cpu().numpy()).hex() == want
    inflight = None
    if not profile:                       # NC MSMs in flight, round robin on NC contexts (device time, max over the streams)
        for k in range(2 * NC):
            msm(k % NC)
        torch.cuda.synchronize()
        ev0, ends = torch.cuda.Event(enable_timing=True), [torch.cuda.Event(enable_timing=True) for _ in range(NC)]
        ev0.record(streams[0])
        for st in streams[1:]:
            st.wait_event(ev0)
        for k in range(steps):
            msm(k % NC)
        for st, ev in zip(streams, ends):
            ev.record(st)
        torch.cuda.synchronize()
        inflight = max(ev0.elapsed_time(ev) for ev in ends) / steps
        ok = ok and all(bytes(x[:48].cpu().numpy()).hex() == want for x in outs)
    plan = eng.last_msm_plan()
    row = {"split": split, "rounds": rounds, "batch": batch, "ok": ok, "plan_rounds": plan["affine_rounds"],
           "plan_batch": plan["affine_batch"], "ms_per_msm_4_in_flight": None if inflight is None else round(inflight, 4),
           "stages_ms": dict(zip(names, [round(v / K, 3) for v in acc]))}
    rows.append(row)
    print(json.dumps(row), flush=True)


if profile:
    run(0, 1, 64, 1)
    run(1, 1, 64, 1)
    sys.exit(0)
run(1, -1, 0, 8)
for split, rounds, batch in [(1, 0, 0), (0, 2, 64),
                             (1, 1, 0), (1, 2, 0), (1, 3, 0), (1, 4, 0),
                             (1, 1, 64), (1, 1, 128), (1, 1, 256),
                             (1, 2, 32), (1, 2, 64), (1, 2, 128), (1, 2, 256),
                             (1, 3, 16), (1, 3, 32), (1, 3, 64), (1, 3, 128),
                             (1, 4, 32), (1, 4, 64), (1, 4, 128),
                             (1, -1, 0)]:
    run(split, rounds, batch, 8)
if out_path:
    with open(out_path, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
