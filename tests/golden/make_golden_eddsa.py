#!/usr/bin/env python3
"""Extract the reference's Ed25519 signature fixtures into tests/golden/eddsa_*.

Run where the reference tree is available (like make_golden.py, which extracts the other curves' fixtures); the files are
committed so that tests can use them without it.  Only DATA (hex strings, expected errors, valid/invalid flags) is
extracted -- no reference code.
Sources:
  sign/eddsa/eddsa_test.go:24-245       (RFC 8032 7.1 vectors; the byte vectors of each rejection test)
  sign/eddsa/testdata/sign.input.gz     (1024 golden lines -> eddsa_sign_input.json.gz)
  sign/eddsa/testdata/ed25519_test.json (Wycheproof, Apache-2.0 -> eddsa_wycheproof.json + WYCHEPROOF_LICENSE)
  group/edwards25519/const.go           (weakKeys: the five small-order encodings)
"""
import gzip
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def go_bytes_list(src, var):
    m = re.search(var + r"\s*:?=\s*\[\]u?i?n?t?\d*(?:byte)?\{([^}]*)\}", src)
    return bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]+)", m.group(1))).hex()


def eddsa_vectors():
    """sign/eddsa: eddsa_test.go (RFC 8032 7.1 vectors, the byte vectors of each rejection test), testdata/sign.input.gz
    (1024 golden lines: seed || pk, pk, msg, sig || msg), testdata/ed25519_test.json (Wycheproof), and the small-order
    encodings of group/edwards25519/const.go (weakKeys)."""
    src = open(f"{REF}/sign/eddsa/eddsa_test.go").read()
    rfc = [{"seed": s, "pk": p, "msg": m, "sig": g} for s, p, m, g in
           re.findall(r'\{"([0-9a-f]{64})",\s*"([0-9a-f]{64})",\s*"([0-9a-f]*)",\s*"([0-9a-f]{128})"\}', src)]
    assert len(rfc) == 5
    inline = {
        "_how": "replace_r: the vector replaces R of a valid signature; replace_pk: it replaces the key; add_to_s: it is "
                "added to s (little-endian); full: a complete (pk, msg, sig) case",
        "cases": [
            {"test": "TestEdDSAVerifyMalleability", "kind": "add_to_s", "bytes": go_bytes_list(src, "L"),
             "expect": "ErrSignatureNotCanonical"},
            {"test": "TestEdDSAVerifyMalleability", "kind": "full", "pk": go_bytes_list(src, "publicKey"),
             "msg": go_bytes_list(src, "msg2"), "sig": go_bytes_list(src, "sig2"), "expect": "ErrSignatureNotCanonical"},
            {"test": "TestEdDSAVerifyNonCanonicalR", "kind": "replace_r", "bytes": go_bytes_list(src, "nonCanonicalR"),
             "expect": "ErrPointRNotCanonical"},
            {"test": "TestEdDSAVerifyNonCanonicalPK", "kind": "replace_pk", "bytes": go_bytes_list(src, "nonCanonicalPk"),
             "expect": "ErrPKNotCanonical"},
            {"test": "TestEdDSAVerifySmallOrderR", "kind": "replace_r", "bytes": go_bytes_list(src, "smallOrderR"),
             "expect": "ErrPointRSmallOrder"},
            {"test": "TestEdDSAVerifySmallOrderPK", "kind": "replace_pk", "bytes": go_bytes_list(src, "smallOrderPk"),
             "expect": "ErrPKSmallOrder"},
        ]}
    for c in inline["cases"]:
        assert all(len(c.get(k, "")) % 2 == 0 for k in ("bytes", "pk", "msg", "sig"))
    const = open(f"{REF}/group/edwards25519/const.go").read()
    body = const[const.index("var weakKeys"):]
    weak = [bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", blk)).hex() for blk in re.findall(r"\{(0x[^}]*)\}", body)[:5]]
    assert len(weak) == 5 and all(len(w) == 64 for w in weak)
    json.dump({"_source": "sign/eddsa/eddsa_test.go:24-245, group/edwards25519/const.go weakKeys (data only)",
               "rfc8032": rfc, "inline": inline, "weak_keys": weak},
              open(os.path.join(HERE, "eddsa_vectors.json"), "w"), indent=1)
    wp = json.load(open(f"{REF}/sign/eddsa/testdata/ed25519_test.json"))
    cases = [{"tcId": t["tcId"], "pk": g["publicKey"]["pk"], "msg": t["msg"], "sig": t["sig"], "result": t["result"]}
             for g in wp["testGroups"] for t in g["tests"]]
    assert len(cases) == 150
    json.dump({"_source": "sign/eddsa/testdata/ed25519_test.json (Wycheproof, Apache-2.0: see WYCHEPROOF_LICENSE)",
               "cases": cases}, open(os.path.join(HERE, "eddsa_wycheproof.json"), "w"), indent=1)
    with open(f"{REF}/sign/eddsa/testdata/LICENSE") as f, open(os.path.join(HERE, "WYCHEPROOF_LICENSE"), "w") as g:
        g.write(f.read())
    lines = []
    with gzip.open(f"{REF}/sign/eddsa/testdata/sign.input.gz", "rt") as f:
        for line in f:
            parts = line.strip().split(":")
            assert len(parts) == 5
            lines.append({"seed": parts[0][:64], "pk": parts[1], "msg": parts[2], "sig": parts[3][:128]})
    assert len(lines) == 1024
    with gzip.GzipFile(os.path.join(HERE, "eddsa_sign_input.json.gz"), "wb", mtime=0) as f:
        f.write(json.dumps({"_source": "sign/eddsa/testdata/sign.input.gz (seed, pk, msg, R || s)", "cases": lines}).encode())


if __name__ == "__main__":
    eddsa_vectors()
    print("wrote Ed25519 fixtures")
