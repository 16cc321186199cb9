"""GPU timing of batched Ed25519 verification (b2k_ed25519_verify_dev, one thread per signature) next to a host baseline,
libsodium's crypto_sign_open through PyNaCl on one CPU thread, on the same signatures.
Usage: python tools/perf_eddsa.py --out DIR   (writes DIR/perf_eddsa.txt and DIR/perf_eddsa.jsonl)"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import nacl.bindings  # noqa: E402
import nacl.signing  # noqa: E402
from kyber_b200 import Engine  # noqa: E402
from kyber_b200.capi import _buf  # noqa: E402

DISTINCT = 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def signatures(msg_len):
    """DISTINCT (pk, msg, sig) signed by libsodium: 64 keys, msg_len-byte messages"""
    out = []
    for i in range(DISTINCT):
        k = nacl.signing.SigningKey(hashlib.sha256(b"perf key %d" % (i % 64)).digest())
        msg = b"".join(hashlib.sha512(b"perf msg %d %d" % (i, j)).digest() for j in range((msg_len + 63) // 64))[:msg_len]
        out.append((bytes(k.verify_key), msg, k.sign(msg).signature))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    eng = Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    info = card()
    rows, lines = [], ["card: " + info, ""]
    sets = {32: signatures(32), 1024: signatures(1024)}

    def inputs(n, msg_len):
        base = sets[msg_len]
        reps = (n + DISTINCT - 1) // DISTINCT
        pks = b"".join(c[0] for c in base) * reps
        sigs = b"".join(c[2] for c in base) * reps
        msgs = [c[1] for c in base] * reps
        blob, offs = eng._pack_msgs(msgs[:n])
        return pks[:32 * n], blob, offs, sigs[:64 * n]

    def dev_time(n, msg_len):
        pks, blob, offs, sigs = inputs(n, msg_len)
        t = [torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in (pks, blob, offs, sigs)]
        st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
        call = lambda: eng.ed25519_verify_dev(n, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), st.data_ptr())
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        reps = max(3, min(200, int(2e6 // max(n, 1))))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        assert int(st.sum()) == 0, "a valid signature was rejected"
        return ms, reps

    for n, msg_len in ((1, 32), (1024, 32), (1 << 16, 32), (1 << 20, 32), (1 << 16, 1024)):
        ms, reps = dev_time(n, msg_len)
        rows.append({"form": "dev", "n": n, "msg_bytes": msg_len, "ms": ms, "verifications_per_s": n / ms * 1e3, "reps": reps})

    # host-buffer form: pageable host inputs staged by the call, which synchronises; prepacked outside the timed window
    n = 1 << 16
    pks, blob, offs, sigs = inputs(n, 32)
    st = bytearray(n)
    bufs = [_buf(x) for x in (pks, blob, offs, sigs, st)]
    call = lambda: eng._check(eng.lib.b2k_ed25519_verify(eng.h, n, *[b[0] for b in bufs]))
    for _ in range(3):
        call()
    t0 = time.perf_counter()
    for _ in range(10):
        call()
    ms = (time.perf_counter() - t0) / 10 * 1e3
    assert st == bytearray(n)
    rows.append({"form": "host", "n": n, "msg_bytes": 32, "ms": ms, "verifications_per_s": n / ms * 1e3, "reps": 10})

    # libsodium baseline: crypto_sign_open (verification of signed message R || s || M), one thread, same signatures
    for msg_len in (32, 1024):
        sm = [(c[2] + c[1], c[0]) for c in sets[msg_len]]
        for s, pk in sm[:64]:
            nacl.bindings.crypto_sign_open(s, pk)
        t0 = time.perf_counter()
        for s, pk in sm:
            nacl.bindings.crypto_sign_open(s, pk)
        ms = (time.perf_counter() - t0) * 1e3
        rows.append({"form": "libsodium crypto_sign_open (PyNaCl), 1 CPU thread", "n": DISTINCT, "msg_bytes": msg_len, "ms": ms,
                     "verifications_per_s": DISTINCT / ms * 1e3, "reps": 1})

    lines.append("%-52s %9s %6s %12s %16s" % ("form", "n", "msg B", "ms / call", "verifications/s"))
    for r in rows:
        lines.append("%-52s %9d %6d %12.4f %16.4g" % (r["form"], r["n"], r["msg_bytes"], r["ms"], r["verifications_per_s"]))
    text = "\n".join(lines) + "\n"
    print(text)
    with open(os.path.join(args.out, "perf_eddsa.txt"), "w") as f:
        f.write(text)
    with open(os.path.join(args.out, "perf_eddsa.jsonl"), "w") as f:
        for r in rows:
            f.write(json.dumps(dict(r, card=info)) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
