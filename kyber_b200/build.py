"""Build the sm_90a (H100) shared library in-tree (nvcc cross-compiles without a GPU)."""
from __future__ import annotations
import os, subprocess, sys, hashlib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb2kyber.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
              "-Xfatbin", "-compress-all",   # the library is ~85 MB of SASS + line tables uncompressed, ~26 MB compressed
              "-DB2K_COMPACT_FIELD=1"]     # field products as out-of-line by-value calls (fp.cuh); *_inlined.cu units undo it for A/B
UNITS = ["b2k_api.cu", "b2k_msm_inlined.cu", "b2k_g1_mul.cu", "b2k_bn254.cu", "b2k_g2.cu", "b2k_pairing.cu", "b2k_pairing_inlined.cu", "b2k_h2c.cu", "b2k_share.cu", "b2k_share2.cu", "b2k_ed25519.cu", "b2k_eddsa.cu", "b2k_ed25519_msm.cu", "b2k_pvss.cu", "b2k_shuffle.cu", "b2k_anon.cu", "b2k_bn256.cu", "b2k_bn254_pairing.cu", "b2k_bdn.cu", "b2k_bn_hash.cu", "b2k_bn_codec.cu", "b2k_multi.cu", "b2k_gt.cu", "b2k_ibe.cu", "b2k_ecies.cu", "b2k_schnorr.cu", "b2k_ecies_bls.cu"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _hash_files(paths) -> str:
    import re
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            data = f.read()
        if p.endswith("b2kyber.h"):            # the public header is mostly documentation: comment edits do not recompile
            data = re.sub(rb"/\*.*?\*/", b"", data, flags=re.S)
        h.update(os.path.basename(p).encode()); h.update(data)
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _closure(src: str) -> list:
    """The source plus every project header it reaches through #include "..." (transitively), in a stable order."""
    import re
    seen, todo = [], [os.path.abspath(src)]
    while todo:
        f = todo.pop()
        if f in seen or not os.path.exists(f):
            continue
        seen.append(f)
        with open(f, "r", errors="replace") as fh:
            for inc in re.findall(r'^\s*#\s*include\s+"([^"]+)"', fh.read(), flags=re.M):
                todo.append(os.path.abspath(os.path.join(os.path.dirname(f), inc)))
    return [seen[0]] + sorted(seen[1:])


def generate_tables() -> None:
    """Write the generated tables the device headers include, when missing or older than their generator."""
    # the program tables of the warp-cooperative pairing are generated (1 s, pure Python, the curve's public parameters only): tools/gen_coop_pairing.py
    gen = os.path.join(HERE, "..", "tools", "gen_coop_pairing.py")
    incs = [os.path.join(CSRC, f"coop_program_{c}.inc") for c in ("bls", "bn254", "bn256")]
    if any(not os.path.exists(i) or os.path.getmtime(i) < os.path.getmtime(gen) for i in incs):
        subprocess.run([sys.executable, gen], check=True, stdout=subprocess.DEVNULL)
    # the comb of the edwards25519 base point that ECIES's fixed-base multiplication reads (tools/gen_ecies_table.py, < 1 s)
    gen_ecies = os.path.join(HERE, "..", "tools", "gen_ecies_table.py")
    inc = os.path.join(CSRC, "ecies_base_comb.inc")
    if not os.path.exists(inc) or os.path.getmtime(inc) < os.path.getmtime(gen_ecies):
        subprocess.run([sys.executable, gen_ecies], check=True, stdout=subprocess.DEVNULL)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile kyber_b200/libb2kyber.so.  Incremental per translation unit: a unit is recompiled when its own source or a
    header it includes (transitively) changed (stamp next to the object), the library is relinked when an object changed.  Returns the library path."""
    generate_tables()
    objs, procs = [], []
    for u in UNITS:
        src = os.path.join(CSRC, u)
        obj = os.path.join(CSRC, u.replace(".cu", ".o"))
        objs.append(obj)
        stamp = _hash_files(_closure(src))
        sf = obj + ".stamp"
        if not force and os.path.exists(obj) and os.path.exists(sf) and open(sf).read() == stamp:
            continue
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas"); cmd.insert(2, "-v")
        if os.path.exists(sf):
            os.remove(sf)
        procs.append((u, sf, stamp, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = None
    for u, sf, stamp, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            failed = failed or u
        else:
            with open(sf, "w") as f:
                f.write(stamp)
    if failed:
        raise RuntimeError(f"nvcc failed on {failed}")
    link_stamp = _hash_files([o + ".stamp" for o in objs])
    lf = LIB + ".stamp"
    if not procs and not force and os.path.exists(LIB) and os.path.exists(lf) and open(lf).read() == link_stamp:
        return LIB
    cmd = [_nvcc(), "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB + ".tmp", *objs, "-lcudart", "-ldl"]
    subprocess.run(cmd, check=True)
    os.replace(LIB + ".tmp", LIB)          # atomic: a reader (or a snapshot of the tree) never sees a half-written library
    with open(lf, "w") as f:
        f.write(link_stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
