#!/usr/bin/env python3
"""Static check of the field-product code the compiler generated (no GPU needed).

Every kernel of a translation unit carries its own copies of the out-of-line field products (fp.cuh, B2K_COMPACT_FIELD).  ptxas
allocates registers across the whole call graph of a kernel, so ONE caller that holds many field elements by value degrades the
products of that kernel: a 12-limb Montgomery product is 276 IMAD.WIDE + ~100 other instructions when it is compiled well and
~500 instructions (moves + callee-save spills) when it is not -- a 25 % slowdown of a pairing kernel that nothing else reveals.
Usage:  python tools/codegen_check.py kyber_b200/csrc/b2k_pairing.o [more .o / .cubin ...]
Prints, per kernel, the product-like functions (>= 100 IMAD.WIDE) with their instruction / move / local-memory counts, and
exits 1 if a product of a kernel listed in WATCH exceeds its budget.
"""
import collections
import re
import subprocess
import sys

WATCH = {  # kernel name fragment -> max instructions of its largest 12-limb product function (385 when compiled well)
    "k_bls_pairing_checkILi64ELi4": 420, "k_bls_pairILi64ELi4": 420,                 # the default pairing kernels (b2k_pairing.o)
    "k_coop_pairing_check": 420, "k_coop_pairE": 420,                                # the cooperative ones
    "k_msm_accumulate_slicesINS_8Bls381G2": 420, "k_msm_reduce_l1INS_8Bls381G2": 420, "k_msm_accumulateINS_8Bls381G2": 420,   # b2k_g2.o
    "k_msm_accumulate_slices_directINS_8Bls381G1": 420, "k_pt_backwardINS_8Bls381G1": 420,                                  # b2k_api.o
    "k_msm_accumulate_slicesINS_8Bls381G1ELi3": 420,                                 # the slice kernel the automatic plan runs
    "k_bdn_masked_sumINS_8Bls381G2": 420, "k_bdn_masked_sumINS_8Bls381G1": 420,      # sign/bdn's masked sums (b2k_bdn.o)
    "k_bdn_finishINS_8Bls381G2": 420, "k_bdn_totalINS_8Bls381G2": 420,
}


def functions(sass_lines):
    """split one kernel's SASS into (start, instructions) at RET / EXIT"""
    out, cur = [], []
    for ln in sass_lines:
        cur.append(ln)
        if ln.startswith(("RET", "EXIT")):
            out.append(cur)
            cur = []
    return out


def report(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    kernels, name, cur = [], None, []
    for ln in txt.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            if name:
                kernels.append((name, cur))
            name, cur = m.group(1), []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(.*?)\s*;", ln)
        if m and name:
            ins = m.group(1)
            cur.append(ins.split(None, 1)[1] if ins.startswith("@") and " " in ins else ins)
    if name:
        kernels.append((name, cur))
    bad = 0
    for name, ins in kernels:
        rows = []
        for f in functions(ins):
            c = collections.Counter()
            for i in f:
                op = i.split()[0]
                c["wide" if "WIDE" in op else "mov" if "MOV" in op else "local" if op.startswith(("LDL", "STL")) else "other"] += 1
            if c["wide"] >= 100:
                rows.append((len(f), c["wide"], c["mov"], c["local"]))
        if not rows:
            continue
        worst = max([r[0] for r in rows if 270 <= r[1] <= 290] or [0])    # the 12-limb product (276 IMAD.WIDE); other rows are inversions etc.
        flag = ""
        for frag, budget in WATCH.items():
            if frag in name and worst > budget:
                flag = f"   <-- over budget ({budget})"
                bad = 1
        print(f"{name[:70]:70s} " + "  ".join(f"[{n} instr: {w} wide, {m} mov, {l} ldl/stl]" for n, w, m, l in rows) + flag)
    return bad


if __name__ == "__main__":
    rc = 0
    for p in sys.argv[1:]:
        print("==", p)
        rc |= report(p)
    sys.exit(rc)
