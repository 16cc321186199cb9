#!/usr/bin/env python3
"""Extract the RFC 9380 expand_message_xmd(SHA-256) vectors from the reference into tests/golden/xmd_sha256_vectors.json.

Run where the reference tree is available (like make_golden_anon.py); the file is committed so that tests can use it without
it.  Only DATA is extracted -- the five messages of inputsTestVectRFC9380, the two DSTs and the expected hex outputs of 32 and
128 bytes -- no reference code.
Source: group/edwards25519/point_test.go, TestExpandMessageXMDSHA256ShortDST and TestExpandMessageXMDSHA256LongDST.  The long DST
is 255 bytes longer than the limit of RFC 9380 5.3.3, so its vectors exercise the H2C-OVERSIZE-DST- pre-hash.
"""
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def go_string(expr: str) -> str:
    """a Go string expression made of "..." literals joined by +"""
    return "".join(re.findall(r'"([^"]*)"', expr))


def block(src: str, start: str) -> str:
    i = src.index(start)
    return src[i:src.index("\n}\n", i)]


def main():
    src = open(os.path.join(REF, "group", "edwards25519", "point_test.go")).read()
    inputs_expr = src[src.index("inputsTestVectRFC9380 = []string{"):]
    inputs_expr = inputs_expr[inputs_expr.index("{") + 1:inputs_expr.index("\n\t}")]
    msgs = [go_string(part + '"') for part in re.split(r'",\n', inputs_expr.rstrip().rstrip(","))]
    out = []
    for test in ("TestExpandMessageXMDSHA256ShortDST", "TestExpandMessageXMDSHA256LongDST"):
        body = block(src, f"func {test}(")
        dst = re.search(r'dst := "([^"]*)"', body).group(1)
        for length, name in ((32, "expectedHex32byte"), (128, "expectedHex128byte")):
            arr = body[body.index(name):]
            arr = arr[arr.index("{") + 1:arr.index("}")]
            hexes = re.findall(r'"([0-9a-f]+)"', arr)
            assert len(hexes) == len(msgs) == 5, (test, len(hexes), len(msgs))
            for m, hx in zip(msgs, hexes):
                out.append({"msg": m, "dst": dst, "len_in_bytes": length, "uniform_bytes": hx})
    path = os.path.join(HERE, "xmd_sha256_vectors.json")
    with open(path, "w") as f:
        json.dump({"source": "RFC 9380 appendix K.1 (expand_message_xmd, SHA-256), as pinned by the reference's "
                             "group/edwards25519/point_test.go", "vectors": out}, f, indent=1)
        f.write("\n")
    print(f"{len(out)} vectors -> {path}")


if __name__ == "__main__":
    main()
