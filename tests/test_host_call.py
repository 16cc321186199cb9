"""The staged host-call pattern of kyber_b200/csrc/host_call.cuh.

CPU: every host-buffer entry point stages through host_call / arena_carve (one reservation of the one arena), and the status
bits live in one enum; the stage's count pass, compiled for the host, counts exactly the bytes its take pass walks.
GPU: a host-buffer call clears the device status word in front and fetches and clears it behind, so a bit left by an
enqueued *_dev call surfaces neither in the host call nor in a later b2k_wait."""
import json
import os
import random
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kyber_b200", "csrc")

# where the arena and the status word are handled directly: the helpers themselves, their definitions, the MSM's own
# pipeline (msm_host.cuh) and the sharded MSM, whose async call leaves the status word for b2k_wait on purpose
EXEMPT = {"host_call.cuh", "b2k_api.cu", "b2k_ctx.h", "msm_host.cuh", "b2k_multi.cu"}
FORBIDDEN = [
    ("arena_reserve", re.compile(r"\barena_reserve\(")),
    ("arena_take", re.compile(r"\barena_take<|\bb2k_arena_take\(")),
    ("input arena", re.compile(r"\bb2k_arena_in\b|\barena_in\b")),
    ("h_flags", re.compile(r"\bh_flags\b")),
    ("raw d_flags copy", re.compile(r"cudaMemcpyAsync\([^;]*\bd_flags\b")),
    ("raw d_flags memset", re.compile(r"cudaMemsetAsync\(\s*ctx->d_flags\b")),
]


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_host_calls_stage_through_the_helpers():
    bad = [(name, what) for name, text in _sources() if name not in EXEMPT for what, rx in FORBIDDEN if rx.search(text)]
    assert bad == []


def test_status_bits_only_in_the_enum():
    literal_bit = re.compile(r"atomicOr\([^;]*,\s*(0x[0-9a-fA-F]+|\d+)u?\s*\)")
    flag_def = re.compile(r"\bFLAG_[A-Z0-9_]+\s*=")
    bad = [name for name, text in _sources() if literal_bit.search(text)]
    bad += [name for name, text in _sources() if name != "host_call.cuh" and flag_def.search(text)]
    assert bad == []


STAGE_TEST = r"""
#include "host_call.cuh"
#include <cstdint>
#include <cstdio>
using namespace b2k_host;

static char* g_base;
static size_t g_cap, g_used;
static int g_reserves, g_takes;
int b2k_arena_reserve(b2k_ctx*, size_t bytes) {
  static std::vector<char> buf;
  buf.assign(bytes + 256, 0);
  g_base = (char*)(((uintptr_t)buf.data() + 255) & ~uintptr_t(255));
  g_cap = bytes; g_used = 0; g_reserves++;
  return B2K_OK;
}
void* b2k_arena_take(b2k_ctx*, size_t bytes) {
  g_takes++;
  size_t off = (g_used + 255) & ~size_t(255);
  if (off + bytes > g_cap) return nullptr;
  g_used = off + bytes;
  return g_base + off;
}
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
  b2k_ctx ctx;
  const uint8_t in_a[100] = {}, *none = nullptr;
  uint8_t out_a[300];
  const uint32_t offs[5] = {};
  uint8_t *da = nullptr, *dz = nullptr, *dout = nullptr, *dscr = nullptr;
  uint32_t* doff = nullptr;
  auto layout = [&](Carve& c) {
    da = c.in(in_a, 10, 10);
    dz = c.in(none, 0);
    doff = c.in(offs, 5);
    dscr = c.take<uint8_t>(3, 7);
    dout = c.out(out_a, 3, 100);
  };
  Carve count;
  layout(count);
  CHECK(count.ok && count.ins.empty() && count.outs.empty() && !da);
  Carve take;
  CHECK(arena_carve(&ctx, layout, take) == B2K_OK && g_reserves == 1);
  CHECK(take.bytes == count.bytes && g_used == count.bytes && g_cap == count.bytes);   // counted = walked
  CHECK(take.ins.size() == 2 && take.ins[0].dst == da && take.ins[0].src == in_a && take.ins[0].bytes == 100);
  CHECK(take.ins[1].dst == doff && take.ins[1].src == offs && take.ins[1].bytes == 20);
  CHECK(take.outs.size() == 1 && take.outs[0].dst == out_a && take.outs[0].src == dout && take.outs[0].bytes == 300);
  // a zero-length input: no copy, a pointer inside the arena
  CHECK(dz && (char*)dz >= g_base && (char*)dz <= g_base + g_cap);
  CHECK((char*)dscr >= g_base && (char*)dscr + 21 <= g_base + g_cap);
  // a count whose bytes overflow size_t fails the count pass: nothing reserved, nothing taken
  const int takes = g_takes;
  Carve big;
  auto overflow = [&](Carve& c) { c.in(in_a, 4); c.in(in_a, SIZE_MAX / 2, 3); c.out(out_a, 1); };
  CHECK(arena_carve(&ctx, overflow, big) == B2K_ERR_ARG && g_reserves == 1 && g_takes == takes && big.ins.empty());
  CHECK(ctx.err == "batch too large");
  auto padding = [&](Carve& c) { c.take<uint8_t>(SIZE_MAX - 100); c.take<uint8_t>(1); };   // the 256-byte rounding overflows
  CHECK(arena_carve(&ctx, padding, big) == B2K_ERR_ARG && g_reserves == 1 && g_takes == takes);
  std::printf("OK\n");
  return 0;
}
"""


def _cuda_include():
    from kyber_b200 import build
    nvcc = build._nvcc()
    if not os.path.isabs(nvcc):
        import shutil
        nvcc = shutil.which(nvcc) or "/usr/local/cuda/bin/nvcc"
    return os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")


def test_stage_count_pass_on_the_host(tmp_path):
    src, exe = tmp_path / "stage.cpp", tmp_path / "stage"
    src.write_text(STAGE_TEST)
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", CSRC, "-I", _cuda_include(), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "OK", out.stdout + out.stderr


# ---- GPU: no stale status bit ----------------------------------------------------------------------------------------------

def _cases():
    """name -> callable(engine) returning (got, want) for small valid inputs"""
    from oracle import bls12381 as o
    from oracle import h2c_bls12381 as h
    from oracle import h2c_bls12381_g2 as h2
    from oracle import bn254 as o4
    from oracle import bn254_hash as bh
    from oracle import bn256 as o6
    from oracle import ecies as ec
    import eddsa_cases
    import pvss_cases as pc

    rng = random.Random(7)
    msgs = [b"", b"abc", rng.randbytes(70)]
    kat = json.load(open(os.path.join(ROOT, "tests", "golden", "bls12381_signature_kats.json")))["edge_case_g1"]
    p1, p2 = o.g1_mul(5), o.g2_mul(7)
    priv = rng.randbytes(32)
    cts = [ec.encrypt(ec.mul(priv), rng.randbytes(32), rng.randbytes(32))[1] for _ in range(3)]
    pubs, rs, pts = [ec.mul(rng.randbytes(32)) for _ in range(3)], [rng.randbytes(32) for _ in range(3)], [rng.randbytes(16) for _ in range(3)]
    rfc = [(pk, m, s) for _, pk, m, s in eddsa_cases.rfc8032()]
    g, hh = pc.base_mul(3), pc.base_mul(11)
    proof, xg, xh = pc.new_dleq_proof(g, hh, 5, 9)

    def ecies_decrypt(e):
        got, st = e.ed25519_ecies_decrypt(priv, cts, 48)
        return list(zip(st, got)), [ec.decrypt(priv, c) for c in cts]

    def ecies_encrypt(e):
        got, st = e.ed25519_ecies_encrypt(pubs, rs, pts)
        return list(zip(st, got)), [ec.encrypt(p, r, m) for p, r, m in zip(pubs, rs, pts)]

    return {
        "hash_to_g1": lambda e: (e.bls12381_hash_to_g1(msgs, h.DST_G1), b"".join(o.g1_to_affine_bytes(h.hash_to_g1(m, h.DST_G1)) for m in msgs)),
        "hash_to_g2": lambda e: (e.bls12381_hash_to_g2(msgs, h2.DST_G2), b"".join(o.g2_to_affine_bytes(h2.hash_to_g2(m, h2.DST_G2)) for m in msgs)),
        "bn254_hash": lambda e: (e.bn254_hash_to_g1(msgs), b"".join(o4.g1_marshal(bh.hash_to_g1(b"BN254G1_XMD:KECCAK-256_SVDW_RO_", m)) for m in msgs)),
        "bn256_hash": lambda e: (e.bn256_hash_to_g1(msgs), b"".join(o6.g1_marshal(o6.hash_to_g1(m)) for m in msgs)),
        "g1_decompress": lambda e: (e.bls12381_g1_decompress(o.g1_compress(p1)), (o.g1_to_affine_bytes(p1), b"\x01")),
        "g2_decompress": lambda e: (e.bls12381_g2_decompress(o.g2_compress(p2)), (o.g2_to_affine_bytes(p2), b"\x01")),
        "bn254_unmarshal": lambda e: (e.bn_unmarshal_check("bn254", 1, o4.g1_marshal(o4.G1)), b"\x01"),
        "bn256_unmarshal": lambda e: (e.bn_unmarshal_check("bn256", 1, o6.g1_marshal(o6.G1)), b"\x01"),
        "verify_g1sig": lambda e: (e.bls12381_verify_g1sig(bytes.fromhex(kat["pk_g2"]), [bytes.fromhex(kat["msg"])], h.DST_G1,
                                                           bytes.fromhex(kat["sig_g1"])), b"\x01"),
        "g1_mul_batch": lambda e: (e.bls12381_g1_mul_batch((3).to_bytes(32, "big"), o.g1_to_affine_bytes(p1)), o.g1_compress(o.g1_mul(3, p1))),
        "ed25519_verify": lambda e: (e.ed25519_verify(b"".join(c[0] for c in rfc), [c[1] for c in rfc], b"".join(c[2] for c in rfc)),
                                     bytes(len(rfc))),
        "ecies_decrypt": ecies_decrypt,
        "ecies_encrypt": ecies_encrypt,
        "dleq_verify": lambda e: (e.ed25519_dleq_verify(g, hh, xg, xh, proof), bytes(1)),
    }


CASE_NAMES = ["hash_to_g1", "hash_to_g2", "bn254_hash", "bn256_hash", "g1_decompress", "g2_decompress", "bn254_unmarshal",
              "bn256_unmarshal", "verify_g1sig", "g1_mul_batch", "ed25519_verify", "ecies_decrypt", "ecies_encrypt", "dleq_verify"]


def _leave_point_flag(engine):
    """enqueue one G1 Point.Mul whose point has a non-canonical x (x = p): the kernel sets FLAG_POINT; nothing waits for it"""
    import torch
    from oracle import bls12381 as o
    pt = o.P.to_bytes(48, "big") + bytes(47) + b"\x02"
    d_s = torch.zeros(32, dtype=torch.uint8, device="cuda")
    d_p = torch.tensor(list(pt), dtype=torch.uint8, device="cuda")
    d_o = torch.zeros(144, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.call_dev("b2k_bls12381_g1_mul_batch_dev", 1, d_s.data_ptr(), d_p.data_ptr(), d_o.data_ptr())
    engine.synchronize()
    return d_s, d_p, d_o


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_host_call_leaves_no_stale_status_bit(engine, name):
    from kyber_b200.capi import B2KError
    case = _cases()[name]
    keep = _leave_point_flag(engine)
    got, want = case(engine)
    assert got == want
    engine.wait()                                  # the host call fetched and cleared the bit it found
    # the same sequence with a wait in between still reports the operand error: the bit did reach the status word
    _leave_point_flag(engine)
    with pytest.raises(B2KError):
        engine.wait()
    del keep
