"""GPU timing of batched sign/schnorr verification over BLS12-381 keys on G1 and G2 (b2k_bls12381_g{1,2}_schnorr_verify and
_dev, one thread per signature), with 32-byte messages (the DKG's bundle-hash size), next to today's path: decompress R and the
keys (b2k_bls12381_g{1,2}_decompress), SHA-512 and the reduction mod r on the host, two *_mul_batch_affine calls, one
*_add_batch and a comparison on the host, timed alternating with the new call in the same process.  Statuses must agree on
every call.  Median of 3 rounds with min and max; the card's name and power limit are read in the same run.
Usage: python tools/perf_schnorr.py --out DIR   (writes DIR/perf_schnorr.txt and DIR/perf_schnorr.jsonl)"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
from kyber_b200.capi import _buf  # noqa: E402
from oracle import bls12381 as bls  # noqa: E402
import schnorr_oracle as so  # noqa: E402

DISTINCT = 64
SIZES = (1, 1 << 10, 1 << 14, 1 << 16, 1 << 20)
GEN = {"bls12381_g1": bls.g1_to_affine_bytes(bls.G1), "bls12381_g2": bls.g2_to_affine_bytes(bls.G2)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def signatures(group):
    """DISTINCT valid (pk, 32-byte msg, sig) over 8 keys; the last one has its message changed (status INVALID)"""
    out = []
    for i in range(DISTINCT):
        x = int.from_bytes(hashlib.sha256(b"perf key %d" % (i % 8)).digest(), "big") % bls.R
        m = hashlib.sha256(b"perf bundle %d" % i).digest()
        k = int.from_bytes(hashlib.sha256(b"perf nonce %d" % i).digest(), "big") % bls.R
        out.append((so.public_key(group, x), m, so.sign(group, x, m, k)))
    pk, m, s = out[-1]
    out[-1] = (pk, bytes([m[0] ^ 1]) + m[1:], s)
    return out


def todays_path(eng, group, pks, msgs, sigs, n):
    """statuses from the entry points a caller has without this change (every input here decodes)"""
    pl = so.POINT_LEN[group]
    gi = 1 if group == "bls12381_g1" else 2
    rs = b"".join(sigs[(pl + 32) * i:(pl + 32) * i + pl] for i in range(n))
    ss = b"".join(sigs[(pl + 32) * i + pl:(pl + 32) * (i + 1)] for i in range(n))
    dec = eng.bls12381_g1_decompress if gi == 1 else eng.bls12381_g2_decompress
    ops, ok = dec(rs + pks)
    assert all(ok)
    ol = 2 * pl
    r_ops, k_ops = ops[:ol * n], ops[ol * n:]
    hs = b"".join(so.reduce_be(hashlib.sha512(rs[pl * i:pl * (i + 1)] + pks[pl * i:pl * (i + 1)] + msgs[i]).digest()).to_bytes(32, "big")
                  for i in range(n))
    assert all(int.from_bytes(ss[32 * i:32 * (i + 1)], "big") < bls.R for i in range(n))
    mul = eng.bls12381_g1_mul_batch_affine if gi == 1 else eng.bls12381_g2_mul_batch_affine
    sb = mul(ss, GEN[group] * n)
    hk = mul(hs, k_ops)
    rhk = eng.bls12381_add_batch(gi, r_ops, hk)
    return bytes(0 if sb[ol * i:ol * (i + 1)] == rhk[ol * i:ol * (i + 1)] else 4 for i in range(n))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    info = card()
    rows, lines = [], ["card: " + info, ""]

    for group in ("bls12381_g1", "bls12381_g2"):
        pl = so.POINT_LEN[group]
        base = signatures(group)
        for n in SIZES:
            reps = (n + DISTINCT - 1) // DISTINCT
            pks = (b"".join(c[0] for c in base) * reps)[:pl * n]
            msgs = ([c[1] for c in base] * reps)[:n]
            sigs = (b"".join(c[2] for c in base) * reps)[:(pl + 32) * n]
            want = bytes(0 if (i % DISTINCT) != DISTINCT - 1 else 4 for i in range(n))
            blob, offs = eng._pack_msgs(msgs)
            t = [torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in (pks, blob, offs, sigs)]
            d_st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
            st = bytearray(n)
            bufs = [_buf(x) for x in (pks, blob, offs, sigs, st)]
            host_fn = getattr(eng.lib, f"b2k_{group}_schnorr_verify")
            host = lambda: eng._check(host_fn(eng.h, n, *[b[0] for b in bufs]))
            dev = lambda: eng.schnorr_verify_dev(group, n, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(),
                                                 d_st.data_ptr())
            calls = max(1, min(50, int(2 ** 16 // n)))
            for _ in range(2):
                host(); dev()
            torch.cuda.synchronize()
            res = {"host": [], "dev": [], "today": []}
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                for _ in range(calls):
                    host()
                res["host"].append((time.perf_counter() - t0) / calls * 1e3)
                assert bytes(st) == want, "host form: statuses differ"
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(calls):
                    dev()
                e1.record()
                torch.cuda.synchronize()
                res["dev"].append(e0.elapsed_time(e1) / calls)
                assert bytes(d_st.cpu().numpy()) == want, "dev form: statuses differ"
                t0 = time.perf_counter()
                got = todays_path(eng, group, pks, msgs, sigs, n)
                torch.cuda.synchronize()
                res["today"].append((time.perf_counter() - t0) * 1e3)
                assert got == want, "today's path: statuses differ"
            for form, ts in res.items():
                ts = sorted(ts)
                rows.append({"group": group, "form": form, "n": n, "msg_bytes": 32, "ms_median": ts[len(ts) // 2], "ms_min": ts[0],
                             "ms_max": ts[-1], "verifications_per_s": n / ts[len(ts) // 2] * 1e3, "calls_per_round": calls if form != "today" else 1})
            print(group, n, {k: sorted(v)[len(v) // 2] for k, v in res.items()}, flush=True)

    lines.append("%-12s %-6s %8s %12s %12s %12s %16s" % ("group", "form", "n", "ms median", "ms min", "ms max", "verifications/s"))
    for r in rows:
        lines.append("%-12s %-6s %8d %12.4f %12.4f %12.4f %16.4g" % (r["group"], r["form"], r["n"], r["ms_median"], r["ms_min"],
                                                                    r["ms_max"], r["verifications_per_s"]))
    lines += ["", "host = blocking host-buffer call (staging and synchronise included), dev = _dev call timed with CUDA events,",
              "today = decompress R and keys, host SHA-512 and mod r, two mul_batch_affine, add_batch, host comparison (one call)"]
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_schnorr.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_schnorr.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
