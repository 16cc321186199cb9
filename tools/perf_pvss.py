"""GPU timing of DLEQ proof verification and the PVSS share checks on edwards25519: b2k_ed25519_dleq_verify_dev at 2^16 and
2^20 proofs, b2k_ed25519_pvss_verify_enc_shares at (m, n, t) = (1, 1000, 501), (100, 100, 51), (1000, 1000, 501) with the
split between its kernels (commitments, Horner coms + canonical points, per-deal SHA-256 + Pick, per-share verify) from
torch.profiler, and b2k_ed25519_pvss_verify_dec_shares at 2^16.  Inputs are honest, so every share runs the whole check.
Usage: python tools/perf_pvss.py --out DIR   (writes DIR/perf_pvss.txt and DIR/perf_pvss.jsonl)"""
import argparse
import hashlib
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
import pvss_cases as pc  # noqa: E402

L = pc.L
STAGES = ("k_pvss_load_commits", "k_pvss_hashed_points", "k_pvss_deal_challenge", "k_pvss_enc_verify")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def le(k):
    return (k % (1 << 256)).to_bytes(32, "little")


def chunks(b, w=32):
    return [b[i:i + w] for i in range(0, len(b), w)]


def muls(eng, ks, pts):
    if isinstance(pts, bytes):
        pts = [pts] * len(ks)
    return chunks(eng.ed25519_mul_batch(b"".join(le(k) for k in ks), b"".join(pts)))


def dleq_inputs(eng, n, rng):
    a = [rng.randrange(1, L) for _ in range(2 * n)]
    gh = muls(eng, a, pc.G)
    g, h = gh[:n], gh[n:]
    x, v, c = ([rng.randrange(L) for _ in range(n)] for _ in range(3))
    out = muls(eng, x + x + v + v, g + h + g + h)
    proofs = [le(ci) + le((vi - xi * ci) % L) + a_ + b_ for ci, vi, xi, a_, b_ in zip(c, v, x, out[2 * n:3 * n], out[3 * n:])]
    return [b"".join(z) for z in (g, h, out[:n], out[n:2 * n], proofs)]


def enc_inputs(eng, m, n, t, rng):
    """m honest deals sharing one polynomial and the n keys; a base H per deal"""
    coeffs = [rng.randrange(L) for _ in range(t)]
    s = [sum(a * pow(i + 1, j, L) for j, a in enumerate(coeffs)) % L for i in range(n)]
    hs = muls(eng, [rng.randrange(1, L) for _ in range(m)], pc.G)
    xs = muls(eng, [rng.randrange(1, L) for _ in range(n)], pc.G)
    vs = muls(eng, s, xs)
    commits, sh_all, proofs = [], [], []
    for d in range(m):
        cm = muls(eng, coeffs, hs[d])
        commits += cm
        coms = chunks(eng.ed25519_pubpoly_eval(b"".join(cm), list(range(n))))
        v = [rng.randrange(L) for _ in range(n)]
        out = muls(eng, v + v, [hs[d]] * n + xs)
        c = pc.pick(pc.Xof(hashlib.sha256(b"".join(coms + vs + out)).digest()))
        ci = int.from_bytes(c, "little")
        sh_all += coms
        proofs += [c + le((vi - si * ci) % L) + a + b for vi, si, a, b in zip(v, s, out[:n], out[n:])]
    return b"".join(hs), b"".join(commits), b"".join(xs) * m, b"".join(sh_all), b"".join(vs) * m, b"".join(proofs)


def dec_inputs(eng, n, rng, distinct=4096):
    k = min(n, distinct)
    priv = [rng.randrange(1, L) for _ in range(k)]
    xs = muls(eng, priv, pc.G)
    enc = muls(eng, [rng.randrange(1, L) for _ in range(k)], pc.G)
    dec = muls(eng, [pow(p, -1, L) for p in priv], enc)
    v = [rng.randrange(L) for _ in range(k)]
    out = muls(eng, v + v, [pc.G] * k + dec)
    proofs = []
    for i in range(k):
        c = pc.challenge(xs[i], enc[i], out[i], out[k + i])
        proofs.append(c + le((v[i] - priv[i] * int.from_bytes(c, "little")) % L) + out[i] + out[k + i])
    reps = n // k
    return pc.G, b"".join(xs) * reps, b"".join(enc) * reps, b"".join(dec) * reps, b"".join(proofs) * reps


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


def stage_split(call):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in STAGES}
    for e in prof.key_averages():
        for k in STAGES:
            if k in e.key:
                out[k] += e.device_time_total / 1e3          # us -> ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    info = card()
    rng = random.Random(2026)
    rows = []

    for n in (1 << 16, 1 << 20):
        base = dleq_inputs(eng, 1 << 16, rng)
        reps_in = n >> 16
        d = [torch.frombuffer(bytearray(b * reps_in), dtype=torch.uint8).cuda() for b in base]
        st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()

        def call():
            eng.ed25519_dleq_verify_dev(n, *[x.data_ptr() for x in d], st.data_ptr())
            eng.synchronize()
        ms, reps = timed(call)
        assert int(st.sum()) == 0, "an honest proof was rejected"
        rows.append({"call": "dleq_verify_dev", "n": n, "ms": ms, "proofs_per_s": n / ms * 1e3, "reps": reps})
        print(json.dumps(rows[-1]), flush=True)

    for m, n, t in ((1, 1000, 501), (100, 100, 51), (1000, 1000, 501)):
        ins = enc_inputs(eng, m, n, t, rng)
        call = lambda: eng.ed25519_pvss_verify_enc_shares(ins[0], ins[1], t, *ins[2:])
        assert call() == bytes(m * n), "an honest share was rejected"
        ms, reps = timed(call)
        split = stage_split(call)
        rows.append({"call": "pvss_verify_enc_shares", "m": m, "n": n, "t": t, "ms": ms, "proofs_per_s": m * n / ms * 1e3,
                     "reps": reps, "stage_ms": split})
        print(json.dumps(rows[-1]), flush=True)

    n = 1 << 16
    ins = dec_inputs(eng, n, rng)
    call = lambda: eng.ed25519_pvss_verify_dec_shares(*ins)
    assert call() == bytes(n), "an honest decrypted share was rejected"
    ms, reps = timed(call)
    rows.append({"call": "pvss_verify_dec_shares", "n": n, "ms": ms, "proofs_per_s": n / ms * 1e3, "reps": reps})

    lines = ["card: " + info, "whole calls ended by a synchronise, after two warm-up calls; host forms stage their inputs", ""]
    lines.append("%-24s %18s %12s %14s  %s" % ("call", "size", "ms / call", "proofs/s", "kernel ms (commits, Horner+points, hash+Pick, verify)"))
    for r in rows:
        size = "m=%d n=%d t=%d" % (r["m"], r["n"], r["t"]) if "m" in r else "n=%d" % r["n"]
        split = " ".join("%.3f" % r["stage_ms"][k] for k in STAGES) if "stage_ms" in r else ""
        lines.append("%-24s %18s %12.3f %14.4g  %s" % (r["call"], size, r["ms"], r["proofs_per_s"], split))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_pvss.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_pvss.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
