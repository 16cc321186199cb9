"""CPU tests: the byte and scalar harness (tests/device/bytes_harness.cu) compiled by g++ -- SHA-256 and HMAC, SHA-512 and the
EdDSA challenge, BLAKE2b, BLAKE2Xb and Scalar.Pick, the arithmetic mod l and the recodings, ECIES's AES-256, GHASH and GCM, the
constant-time selections and multiplications -- on the case list of tests/bytes_cases.py against hashlib, hmac, Python integers
and the oracles.  test_gpu_bytes.py runs the same list on the device build, so a case that passes here and fails there is a
code-generation difference, not an algorithm one."""
import ctypes
import hashlib
import os
import subprocess
import sys

import pytest

import bytes_cases as bc
import pvss_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "device", "bytes_harness.cu")


@pytest.fixture(scope="module")
def twin(tmp_path_factory):
    d = tmp_path_factory.mktemp("bytes_harness")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_ecies_table
    gen_ecies_table.main(str(d / "ecies_base_comb.inc"))       # the table build() generates, for a tree not built yet
    so = str(d / "libemul_bytes_harness.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DB2K_HOST_EMUL", "-Wno-unknown-pragmas", "-I", str(d), "-x",
                    "c++", SRC, "-o", so], check=True)
    return ctypes.CDLL(so)


@pytest.mark.parametrize("op", bc.OPS)
def test_bytes_ops_on_the_twin(twin, op):
    failures = bc.run_all(twin, "host", [op])
    assert not failures, "\n".join(failures)


# the case classes every operation must have (besides "uniform")
REQUIRED = {
    "sha256_update": {"length", "length split3", "boundary 55/56/63/64", "empty fragments"},
    "sha256_zero": {"update_zero", "update_zero 64"},
    "sha256_blocks": {"blocks"},
    "hmac_sha256": {"key <= 64", "key > 64 (hashed)"},
    "ecies_kdf": {"dh"},
    "sha512_3": {"length (0,0,n)", "length (32,32,n-64)", "block edge", "padding edge"},
    "sha512_challenge": {"R || A || M"},
    "blake2b": {"whole", "128-byte chunks", "random chunks", "1 byte after a full block", "1-byte chunks"},
    "xb_root": {"seed", "seed + Write"},
    "xb_block": {"block 0..2", "block 3, 2^31, 2^32-1"},
    "sc_pick": {f"{k} draws rejected" for k in range(5)} | {"fixed seeds", "seed lengths"},
    "sc_canonical": {"l-1, l, l+1, 0, 2^256-1", "l +- 2^32j", "random"},
    "sc_reduce512": {"edges", "(mu-k) l + l-1", "k l +- 1", "low 224 bits ones", "random"},
    "sc_neg": {"multiples of l", "2^255, 2^256-1", "crafted", "random"},
    "sc_recode4": {"all-8, all-F, ripple", "crafted", "random"},
    "sc_rule": {"top<=8", "top>8 carry0", "top>8 carry1"},
    "challenge_is": {"equal", "one byte differs", "c + l"},
    "aes_subbytes": {"all 256 inputs", "random"},
    "aes_expand": {"FIPS-197 key", "zero, ones", "random"},
    "aes_encrypt2": {"FIPS-197 C.3", "random"},
    "ghash": {"length"},
    "gcm_seal": {"length", "len % 32 in 1..16", "len % 32 in 17..31", "zero key and nonce"},
    "gcm_open": {"good tag", "flipped byte", "flipped tag bit", "flipped body byte"},
    "select_cached": {"d in [-8, 8]", "|d| > 8"},
    "select_niels": {"d in [-8, 8]", "|d| > 8"},
    "mul_var": {"scalar x point"},
    "mul_base": {"scalar"},
}


def test_case_counts(capsys):
    """every class of every operation has cases; prints the count per (operation, class)"""
    counts = bc.case_counts()
    assert set(REQUIRED) == set(bc.OPS)
    for op in bc.OPS:
        have = {cls for (o, cls) in counts if o == op}
        assert REQUIRED[op] | {"uniform"} <= have, (op, sorted(REQUIRED[op] - have))
    with capsys.disabled():
        print(f"\n{sum(counts.values())} cases")
        for op in bc.OPS:
            print(f"{op}: " + ", ".join(f"{cls} {n}" for (o, cls), n in counts.items() if o == op))


def batch(op, label="mixed"):
    return next(b for b in bc.batches() if b.op == op and b.label == label)


def test_the_list_reaches_the_edges():
    """Barrett needs 0 and 1 final subtractions (never more than 2), the picks reach XOF block 2, the recodings and rules see every
    top-digit case, the selections every digit, and the lengths of the mixed launches differ within a warp"""
    subs = [bc.barrett_subtractions(int.from_bytes(c.frags[0], "little")) for c in batch("sc_reduce512").cases]
    assert {0, 1} <= set(subs) and max(subs) <= 2
    assert max(pc.pick_draws(c.frags[0]) for c in batch("sc_pick").cases) == 5
    for op in ("sc_recode4", "sc_rule", "mul_var", "mul_base"):
        tops = {bc.rule_class(int.from_bytes(c.frags[0], "little")) for c in batch(op).cases}
        assert tops == {"top<=8", "top>8 carry0", "top>8 carry1"}, op
    for c in batch("sc_recode4").cases:                     # the restatement: digits in range, sum e_i 16^i = k
        e = bc.recode4(int.from_bytes(c.frags[0], "little"))
        assert all(-8 <= x < 8 for x in e[:63]) and 0 <= e[63] <= 16
        assert sum(x << (4 * i) for i, x in enumerate(e)) == int.from_bytes(c.frags[0], "little")
    for op in ("select_cached", "select_niels"):
        assert {bc.to_int(c.args[0]) for c in batch(op).cases} == set(range(-8, 17)), op
    for b in bc.batches():
        shapes = {(tuple(len(f) for f in c.frags), tuple(c.args)) for c in b.cases[:32]}
        if b.label == "uniform":
            assert len({s[0] for s in shapes}) == 1, b.op
        elif b.op in ("sha256_update", "sha512_3", "blake2b", "xb_root", "sc_pick", "hmac_sha256", "ghash", "gcm_seal", "gcm_open"):
            assert len(shapes) > 8, b.op
    assert len({pc.pick_draws(c.frags[0]) for c in batch("sc_pick").cases[:32]}) >= 3


def test_expected_values_hold_the_known_answers():
    """the oracles behind the expectations reproduce FIPS-197 C.3, the zero-key AES-256-GCM vectors, and the keyed BLAKE2Xb root
    of the pvss_cases restatement"""
    fips = [c for c in batch("aes_encrypt2").cases if c.cls == "FIPS-197 C.3"]
    assert fips and all(bc.FIPS_CT in c.want for c in fips)
    zero = [c for c in batch("gcm_seal").cases if c.cls == "zero key and nonce"]
    assert sorted(c.want for c in zero) == sorted(bc.ZERO_KEY_TAGS.values())
    for n in (0, 1, 63, 64, 65, 128, 129, 200):
        seed = hashlib.sha256(b"%d" % n).digest() * 7
        assert bc.xb_root(seed[:n]) == pc.Xof(seed[:n]).root
        assert bc.xb_block(pc.Xof(seed[:n]).root, 2) == pc.Xof(seed[:n]).block_bytes(2)
