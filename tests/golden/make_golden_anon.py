#!/usr/bin/env python3
"""Extract the reference's ring signature fixtures into tests/golden/anon_examples.json.

Run where the reference tree is available (like make_golden_eddsa.py); the file is committed so that tests can use it without
it.  Only DATA is extracted -- the messages, the scope, the signers' positions and the printed hex dumps and tags -- no
reference code.
Source: sign/anon/sig_test.go, the `// Output:` blocks of ExampleSign_one, ExampleSign_anonSet and ExampleSign_linkable.  All
three seed their suite with blake2xb.New(nil) as the random stream.
"""
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def example(src: str, name: str) -> str:
    start = src.index(f"func {name}()")
    return src[start:src.index("\n}\n", start)]


def dumps(body: str):
    """the hex dumps of the Output block, one bytes string per `Signature...:` header"""
    out, cur = [], None
    for line in body[body.index("// Output:"):].splitlines():
        line = line.strip().removeprefix("//").strip()
        if line.startswith("Signature") and line.endswith(":"):
            cur = bytearray()
            out.append(cur)
        elif cur is not None and re.match(r"^[0-9a-f]{8}  ", line):
            cur += bytes.fromhex(line[10:58].replace(" ", ""))
    return [bytes(b).hex() for b in out]


def main():
    src = open(f"{REF}/sign/anon/sig_test.go").read()
    bad = re.search(r'BAD := \[\]byte\("([^"]*)"\)', src).group(1)
    out = {"_source": "sign/anon/sig_test.go: ExampleSign_one, ExampleSign_anonSet, ExampleSign_linkable (Output blocks); "
                      "suite = edwards25519.NewBlakeSHA256Ed25519WithRand(blake2xb.New(nil))",
           "examples": []}
    for name, n in (("ExampleSign_one", 1), ("ExampleSign_anonSet", 3), ("ExampleSign_linkable", 3)):
        body = example(src, name)
        msg = re.search(r'M := \[\]byte\("([^"]*)"\)', body).group(1)
        scope = re.search(r'S := \[\]byte\("([^"]*)"\)', body)
        mine = [int(v) for v in re.findall(r"mine\d? := (\d+)", body)]
        tags = re.findall(r"// Sig\d tag: ([0-9a-f]{64})", body)
        out["examples"].append({"name": name, "n": n, "message": msg, "bad_message": bad,
                                "scope": scope.group(1) if scope else None, "mine": mine, "sigs": dumps(body), "tags": tags})
    with open(os.path.join(HERE, "anon_examples.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
