#!/usr/bin/env python3
"""Extract the reference's Example_schnorr output into tests/golden/pvss_schnorr_example.json.

Run where the reference tree is available (like make_golden.py and make_golden_eddsa.py); the file is committed so that tests
can use it without it.  Only DATA is extracted: the 64 signature bytes C || R of the example's hex dump.
Source: examples/sig_test.go:93-120 (suite edwards25519.NewBlakeSHA256Ed25519, XOF seeded with "example", message
"Hello World!").
"""
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def schnorr_example():
    src = open(f"{REF}/examples/sig_test.go").read()
    body = src[src.index("func Example_schnorr"):]
    rows = re.findall(r"//\s+[0-9a-f]{8}\s+((?:[0-9a-f]{2}\s+){16})", body)
    sig = bytes(int(x, 16) for row in rows for x in row.split())
    assert len(sig) == 64
    json.dump({"_source": "examples/sig_test.go:93-120 (Example_schnorr output, data only)", "seed": "example",
               "message": "Hello World!", "c": sig[:32].hex(), "r": sig[32:].hex()},
              open(os.path.join(HERE, "pvss_schnorr_example.json"), "w"), indent=1)


if __name__ == "__main__":
    schnorr_example()
    print("wrote the Example_schnorr fixture")
