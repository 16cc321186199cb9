"""CPU check of the field products in sign/bdn's masked-sum kernels (b2k_bdn.o), with the budgets tools/codegen_check.py holds the
MSM and pairing kernels to: the G2 sums keep their Fp2 points in memory and add them out of line (bdn_add / bdn_madd in bdn.cuh), so
that the products underneath are compiled without moves or callee-save spills.  Skipped when the library has not been built here."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "kyber_b200", "csrc", "b2k_bdn.o")


def test_bdn_kernels_field_products_are_compiled_clean():
    if not os.path.exists(OBJ) or shutil.which("cuobjdump") is None:
        pytest.skip("object not built here / cuobjdump not available")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "codegen_check.py"), OBJ], capture_output=True, text=True)
    assert r.returncode == 0 and "over budget" not in r.stdout, r.stdout[-2000:]
    for kernel in ("k_bdn_masked_sumINS_8Bls381G2", "k_bdn_masked_sumINS_8Bls381G1", "k_bdn_finishINS_8Bls381G2"):
        line = next((ln for ln in r.stdout.splitlines() if kernel in ln), None)
        assert line is not None and "276 wide" in line, f"no 12-limb product found in {kernel}: the parser no longer understands the SASS"
