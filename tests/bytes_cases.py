"""The case list of the byte and scalar harness (tests/device/bytes_harness.cu) and its expected values, shared by the host twin
(test_bytes_emulation.py) and the device build (test_gpu_bytes.py).

Expected values come from hashlib, hmac and Python integers; the XOF pick from pvss_cases.pick (blake2xb.New + Scalar.Pick
restated), AES, GCM and the multiplications from oracle/ecies.py over oracle/ed25519.py.

Every operation runs as one launch over its whole list, shuffled so that lengths, chunkings and rejection counts differ from lane
to lane, and once more over 128 cases of one shape (the "uniform" class) with different bytes."""
from __future__ import annotations

import ctypes
import functools
import hashlib
import hmac
import random
from dataclasses import dataclass, field

import numpy as np

import ed25519_msm_cases as mc
import pvss_cases as pc
from oracle import ecies as ec
from oracle import ed25519 as ed

L = ed.L
OPS = ["sha256_update", "sha256_zero", "sha256_blocks", "hmac_sha256", "ecies_kdf", "sha512_3", "sha512_challenge", "blake2b",
       "xb_root", "xb_block", "sc_pick", "sc_canonical", "sc_reduce512", "sc_neg", "sc_recode4", "sc_rule", "challenge_is",
       "aes_subbytes", "aes_expand", "aes_encrypt2", "ghash", "gcm_seal", "gcm_open", "select_cached", "select_niels", "mul_var",
       "mul_base"]                                        # enum Op of bytes_harness.cu, in order
HDR = 16
LANES = 128
MU = (1 << 512) // L                                     # Barrett's mu for b = 2^32, k = 8
XOF_ROOT_NODE = 0xFFFFFFFF << 32                         # blake2xb.New: node offset 0, XOF length 2^32 - 1 (unknown)


@dataclass
class Case:
    cls: str
    frags: list                                          # up to four byte strings
    args: list = field(default_factory=list)             # up to four 32-bit words
    want: bytes = b""
    fill: int = 0                                        # the byte the output is pre-filled with


def le(v: int, n: int = 32) -> bytes:
    return v.to_bytes(n, "little")


def rbytes(rng: random.Random, n: int) -> bytes:
    return rng.randbytes(n)


def split3(rng, data: bytes):
    i, j = sorted(rng.randrange(len(data) + 1) for _ in range(2))
    return [data[:i], data[i:j], data[j:]]


# ---- expectations -------------------------------------------------------------------------------------------------------------
def xb_root(seed: bytes, extra: bytes = b"") -> bytes:
    return hashlib.blake2b(seed[64:] + extra, digest_size=64, key=seed[:64], fanout=1, depth=1, node_offset=XOF_ROOT_NODE).digest()


def xb_block(root: bytes, i: int) -> bytes:
    return ed._blake2b(root, ed._param(64, 0, 0, 64, i, 0xFFFFFFFF, 0, 64), 64)


def recode4(k: int):
    return mc.nibbles(le(k))


def neg_point(pt):
    return ((-pt[0]) % ed.P, pt[1])


def sel_expected(d: int, pt) -> bytes:
    """d T for |d| <= 8, the identity otherwise (a top digit above 8 selects nothing)"""
    if abs(d) > 8:
        return ed.encode(ed.IDENT)
    q = ed.scalar_mult(abs(d), pt)
    return ed.encode(neg_point(q) if d < 0 else q)


def barrett_q3(x: int) -> int:
    return ((x >> 224) * MU) >> 288


def barrett_subtractions(x: int) -> int:
    """how many final subtractions of l sc_reduce512 needs for x (the estimate q3 is below the true quotient by this much)"""
    return x // L - barrett_q3(x)


def rule_class(k: int) -> str:
    carry = ((k & ((1 << 252) - 1)) + ed._K63) >> 252
    e63 = ed.top_digit(k)
    return "top<=8" if e63 <= 8 else f"top>8 carry{carry}"


def expect(op: str, f, a) -> bytes:
    if op == "sha256_update":
        return hashlib.sha256(b"".join(f[:3])).digest()
    if op == "sha256_zero":
        return hashlib.sha256(bytes(a[0]) + b"".join(f[:3])).digest()
    if op == "sha256_blocks":
        return hashlib.sha256(f[0]).digest()
    if op == "hmac_sha256":
        return hmac.new(f[0], b"".join(f[1:4]), hashlib.sha256).digest()
    if op == "ecies_kdf":
        return ec.hkdf_sha256(f[0], 44)
    if op == "sha512_3":
        return hashlib.sha512(b"".join(f[:3])).digest()
    if op == "sha512_challenge":
        return le(int.from_bytes(hashlib.sha512(b"".join(f[:3])).digest(), "little") % L)
    if op == "blake2b":
        return hashlib.blake2b(b"".join(f)).digest()
    if op == "xb_root":
        return xb_root(f[0]) + xb_root(f[0], f[1])
    if op == "xb_block":
        return xb_block(f[0], a[0])
    if op == "sc_pick":
        return pc.pick(pc.Xof(f[0])) * 2
    if op == "sc_canonical":
        return bytes([int.from_bytes(f[0], "little") < L])
    if op == "sc_reduce512":
        return le(int.from_bytes(f[0], "little") % L)
    if op == "sc_neg":
        return le(-int.from_bytes(f[0], "little") % L)
    if op == "sc_recode4":
        return bytes(e & 0xFF for e in recode4(int.from_bytes(f[0], "little")))
    if op == "sc_rule":
        return le(ed.effective_scalar(int.from_bytes(f[0], "little")))
    if op == "challenge_is":
        return bytes([f[0] == f[1]])
    if op == "aes_subbytes":
        return bytes(ec.SBOX[b] for b in f[0])
    if op == "aes_expand":
        return b"".join(ec.aes256_round_keys(f[0]))
    if op == "aes_encrypt2":
        rks = ec.aes256_round_keys(f[0])
        return ec.aes256_encrypt_block(b"", f[1][:16], rks) + ec.aes256_encrypt_block(b"", f[1][16:], rks)
    if op == "ghash":
        return ec._ghash(int.from_bytes(f[0], "big"), f[1]).to_bytes(16, "big")
    if op == "gcm_seal":
        return ec.gcm_seal(f[0][:32], f[0][32:], f[1])
    if op == "gcm_open":
        m = ec.gcm_open(f[0][:32], f[0][32:], f[1])
        return bytes(len(f[1]) - 16) + b"\x00" if m is None else m + b"\x01"
    if op == "select_cached":
        return sel_expected(to_int(a[0]), ed.decode(f[0]))
    if op == "select_niels":
        return sel_expected(to_int(a[0]), ed.scalar_mult(1 << (8 * a[1])))
    if op == "mul_var":
        return ec.mul(f[0], ed.decode(f[1]))
    if op == "mul_base":
        return ec.mul(f[0])
    raise KeyError(op)


def to_int(w: int) -> int:
    return w - (1 << 32) if w >> 31 else w


def u32(d: int) -> int:
    return d & 0xFFFFFFFF


# ---- the case classes of each operation ---------------------------------------------------------------------------------------
def sha256_update(rng):
    out = []
    for n in list(range(0, 201)) + [447, 448, 511, 512]:
        d = rbytes(rng, n)
        out.append(Case("length", [d]))
        out.append(Case("length split3", split3(rng, d)))
    for n in (56, 64, 100, 119, 120, 128, 130, 200):       # a fragment boundary at 55/56/63/64 bytes
        d = rbytes(rng, n)
        for p in (55, 56, 63, 64):
            if p > n:
                continue
            for s in ([d[:p], b"", d[p:]], [b"", d[:p], d[p:]], [d[:p], d[p:], b""], [d[:1], d[1:p], d[p:]],
                      [d[:p - 1], d[p - 1:p], d[p:]]):
                out.append(Case("boundary 55/56/63/64", s))
    out += [Case("empty fragments", [b"", b"", b""]), Case("empty fragments", [b"", b"", rbytes(rng, 64)]),
            Case("empty fragments", [b"", rbytes(rng, 55), b""])]
    return out


def sha256_zero(rng):
    out = []
    for z in (0, 1, 55, 56, 63, 64, 65, 128, 136):
        for n in (0, 1, 7, 37, 64, 100):
            out.append(Case("update_zero 64" if z == 64 else "update_zero", split3(rng, rbytes(rng, n)), [z]))
    return out


def sha256_blocks(rng):
    return [Case("blocks", [rbytes(rng, 64 * k)]) for k in list(range(0, 7)) + [9, 17]]


def hmac_sha256(rng):
    out = []
    for k in list(range(0, 65)) + [65, 100, 128, 200]:
        cls = "key <= 64" if k <= 64 else "key > 64 (hashed)"
        out.append(Case(cls, [rbytes(rng, k)] + split3(rng, rbytes(rng, rng.choice([0, 1, 32, 33, 55, 64, 100, 200])))))
    return out


def ecies_kdf(rng):
    return [Case("dh", [d]) for d in [bytes(32), b"\xff" * 32] + [rbytes(rng, 32) for _ in range(30)]]


def sha512_3(rng):
    out = []
    for n in list(range(0, 301)) + [1023, 100000]:
        d = rbytes(rng, n)
        out.append(Case("length (0,0,n)", [b"", b"", d]))
        if n >= 64:
            out.append(Case("length (32,32,n-64)", [d[:32], d[32:64], d[64:]]))
    for n in (300, 1023):                                  # a or b ending inside, and exactly on, a 128-byte block
        d = rbytes(rng, n)
        for na, nb in ((128, 0), (0, 128), (127, 1), (100, 28), (130, 126), (64, 100), (128, 128), (200, 0), (0, 200), (129, 127),
                       (1, 255), (256, 0)):
            out.append(Case("block edge", [d[:na], d[na:na + nb], d[na + nb:]]))
    for n in (111, 112, 239, 240):                         # the padding's edges, in every split
        d = rbytes(rng, n)
        splits = {(0, 0), (n, 0), (0, n), (32, 32), (n - 1, 1), (1, n - 1), (n // 2, n - n // 2), (n // 3, n // 3)}
        splits |= {tuple(sorted((rng.randrange(n + 1), rng.randrange(n + 1)))) for _ in range(4)}
        for na, nb in sorted(splits):
            out.append(Case("padding edge", [d[:na], d[na:na + nb], d[na + nb:]]))
    return out


def sha512_challenge(rng):
    out = []
    for n in (0, 1, 63, 64, 65, 100, 111, 112, 1000):
        out.append(Case("R || A || M", [rbytes(rng, 32), rbytes(rng, 32), rbytes(rng, n)]))
    return out


def blake2b(rng):
    out = []
    for n in list(range(0, 261)) + [1000, 4096]:
        d = rbytes(rng, n)
        out.append(Case("whole", [d, b"", b"", b""], [0]))
        out.append(Case("128-byte chunks", [d, b"", b"", b""], [128]))
        out.append(Case("random chunks", [d, b"", b"", b""], [rng.randint(1, 200)]))
        if n > 128:
            out.append(Case("1 byte after a full block", [d[:128], d[128:129], d[129:], b""], [0]))
        if n % 37 == 0 or n == 4096:
            out.append(Case("1-byte chunks", [d, b"", b"", b""], [1]))
    return out


XB_SEED_LENGTHS = list(range(0, 66)) + [96, 127, 128, 129, 191, 192, 193, 200, 300]


def xb_root_cases(rng):
    out = []
    for n in XB_SEED_LENGTHS:
        seed = rbytes(rng, n)
        out.append(Case("seed", [seed, b""]))
        if n % 16 == 0 or n > 64:
            out.append(Case("seed + Write", [seed, rbytes(rng, rng.choice([1, 63, 64, 128, 200]))]))
    return out


def xb_block_cases(rng):
    out = []
    for n in XB_SEED_LENGTHS:
        root = xb_root(rbytes(rng, n))
        for i in (0, 1, 2):
            out.append(Case("block 0..2", [root], [i]))
        if n % 32 == 0:
            for i in (3, 1 << 31, (1 << 32) - 1):
                out.append(Case("block 3, 2^31, 2^32-1", [root], [i]))
    return out


@functools.lru_cache(maxsize=None)
def pick_seeds(per: int = 3):
    """seeds whose first 0..4 draws are rejected (the pick reaches XOF block 2 for 4), per of each"""
    found: dict = {}
    i = 0
    while any(len(found.get(k, [])) < per for k in range(1, 6)):
        seed = hashlib.sha256(b"pick %d" % i).digest()
        k = pc.pick_draws(seed)
        if k <= 5 and len(found.setdefault(k, [])) < per:
            found[k].append(seed)
        i += 1
    return found


def sc_pick_cases(rng):
    out = []
    for k, seeds in sorted(pick_seeds().items()):
        out += [Case(f"{k - 1} draws rejected", [s]) for s in seeds]
    for s in (b"", b"example", bytes(64), bytes(100)):
        out.append(Case("fixed seeds", [s]))
    for n in (1, 31, 33, 64, 65, 128, 129, 200):
        out.append(Case("seed lengths", [rbytes(rng, n)]))
    return out


def sc_canonical(rng):
    vals = [("l-1, l, l+1, 0, 2^256-1", v) for v in (L - 1, L, L + 1, 0, (1 << 256) - 1)]
    for j in range(8):
        vals += [("l +- 2^32j", L + (1 << 32 * j)), ("l +- 2^32j", L - (1 << 32 * j))]
    vals += [("random", rng.randrange(L)) for _ in range(20)] + [("random", rng.randrange(L, 1 << 256)) for _ in range(20)]
    return [Case(c, [le(v)]) for c, v in vals]


def reduce_inputs(rng):
    M = 1 << 512
    vals = [("edges", v) for v in (0, L - 1, L, L + 1, 2 * L - 1, 2 * L, 3 * L - 1, 1 << 252, (1 << 253) - 1, (1 << 256) - 1,
                                    M - 1, M - L, 3 * L, (1 << 256), 2 * L + 1)]
    vals += [("(mu-k) l + l-1", (MU - k) * L + L - 1) for k in range(0, 40)]
    for bits in list(range(1, 261, 7)) + [259, 260]:
        k = rng.getrandbits(bits) | (1 << (bits - 1))
        vals += [("k l +- 1", k * L + d) for d in (-1, 0, 1)]
    for _ in range(600):                                    # the low 224 bits all ones: where q3 can fall one short
        vals.append(("low 224 bits ones", (rng.getrandbits(288) << 224) | ((1 << 224) - 1)))
    vals += [("random", rng.getrandbits(512)) for _ in range(3000)]
    return [(c, v) for c, v in vals if 0 <= v < M]


def sc_reduce512(rng):
    return [Case(c, [le(v, 64)]) for c, v in reduce_inputs(rng)]


def sc_neg(rng):
    vals = [("multiples of l", k * L) for k in range(6)] + [("2^255, 2^256-1", 1 << 255), ("2^255, 2^256-1", (1 << 256) - 1)]
    vals += [("crafted", v) for v in mc.crafted_high_scalars(rng) + [1, L - 1, L + 1, (1 << 255) - 1]]
    vals += [("random", rng.getrandbits(256)) for _ in range(300)]
    return [Case(c, [le(v)]) for c, v in vals]


ALL8 = int("8" * 64, 16)
RIPPLE = int("7" * 63 + "8", 16)                          # the carry out of digit 0 ripples through all 63 digits


def sc_recode4_cases(rng):
    vals = [("all-8, all-F, ripple", v) for v in (ALL8, (1 << 256) - 1, RIPPLE, int("f" + "7" * 62 + "8", 16))]
    vals += [("crafted", v) for v in mc.crafted_high_scalars(rng) + [0, 1, L, L - 1]]
    vals += [("random", rng.getrandbits(256)) for _ in range(300)]
    return [Case(c, [le(v)]) for c, v in vals]


def sc_rule(rng):
    ks = mc.crafted_high_scalars(rng) + [rng.getrandbits(256) for _ in range(3000)] + [0, 1, L, (1 << 255) - 1, ALL8, RIPPLE,
                                                                                       (1 << 256) - 1, 0x8F << 248]
    return [Case(rule_class(k), [le(k)]) for k in ks]


def challenge_is(rng):
    out = []
    for _ in range(3):
        w = le(rng.randrange(L))
        out.append(Case("equal", [w, w]))
        for p in range(32):
            b = bytearray(w)
            b[p] ^= 1 << rng.randrange(8)
            out.append(Case("one byte differs", [bytes(b), w]))
        out.append(Case("c + l", [le(int.from_bytes(w, "little") + L), w]))
    return out


def aes_subbytes(rng):
    return [Case("all 256 inputs", [bytes(range(32 * i, 32 * i + 32))]) for i in range(8)] + \
        [Case("random", [rbytes(rng, 32)]) for _ in range(8)]


FIPS_KEY = bytes(range(32))
FIPS_PT = bytes.fromhex("00112233445566778899aabbccddeeff")
FIPS_CT = bytes.fromhex("8ea2b7ca516745bfeafc49904b496089")          # FIPS-197 C.3


def aes_expand(rng):
    return [Case("FIPS-197 key", [FIPS_KEY]), Case("zero, ones", [bytes(32)]), Case("zero, ones", [b"\xff" * 32])] + \
        [Case("random", [rbytes(rng, 32)]) for _ in range(20)]


def aes_encrypt2(rng):
    out = [Case("FIPS-197 C.3", [FIPS_KEY, FIPS_PT + bytes(16)]), Case("FIPS-197 C.3", [FIPS_KEY, rbytes(rng, 16) + FIPS_PT])]
    out += [Case("random", [rbytes(rng, 32), rbytes(rng, 32)]) for _ in range(30)]
    return out


GCM_LENGTHS = list(range(0, 81)) + [255, 256, 1000, 4096]


def ghash(rng):
    return [Case("length", [rbytes(rng, 16), rbytes(rng, n)]) for n in GCM_LENGTHS]


ZERO_KEY_TAGS = {0: bytes.fromhex("530f8afbc74536b9a963b4f1c4cb738b"),
                 16: bytes.fromhex("cea7403d4d606b6e074ec5d3baf39d18") + bytes.fromhex("d0d1c8a799996bf0265b98b5d48ab919")}


def gcm_class(n: int) -> str:
    return "length" if n % 32 == 0 else ("len % 32 in 1..16" if n % 32 <= 16 else "len % 32 in 17..31")


def gcm_seal_cases(rng):
    out = [Case(gcm_class(n), [rbytes(rng, 44), rbytes(rng, n)]) for n in GCM_LENGTHS]
    out += [Case("zero key and nonce", [bytes(44), bytes(n)]) for n in ZERO_KEY_TAGS]
    return out


def gcm_open_cases(rng):
    out = []
    for n in GCM_LENGTHS:
        k44, msg = rbytes(rng, 44), rbytes(rng, n)
        ct = ec.gcm_seal(k44[:32], k44[32:], msg)
        out.append(Case("good tag", [k44, ct], fill=0xAA))
        for pos in sorted({0, n // 2, n + 15}):
            b = bytearray(ct)
            b[pos] ^= 1
            out.append(Case("flipped byte", [k44, bytes(b)], fill=0xAA))
    for n in (0, 17, 33):
        k44, msg = rbytes(rng, 44), rbytes(rng, n)
        ct = ec.gcm_seal(k44[:32], k44[32:], msg)
        for t in range(16):                                 # a flipped bit in each tag byte
            b = bytearray(ct)
            b[n + t] ^= 1 << (t % 8)
            out.append(Case("flipped tag bit", [k44, bytes(b)], fill=0xAA))
        if n:
            b = bytearray(ct)
            b[n - 1] ^= 0x80
            out.append(Case("flipped body byte", [k44, bytes(b)], fill=0xAA))
    return out


@functools.lru_cache(maxsize=None)
def sel_points():
    rng = random.Random(77)
    return [mc.point(rng.randrange(L)), mc.point(rng.randrange(L), 3), mc.T8]


def select_cached(rng):
    pts = [ed.encode(ed.decode(p)) for p in sel_points()]
    return [Case("|d| > 8" if abs(d) > 8 else "d in [-8, 8]", [pts[(d + 8) % len(pts)]], [u32(d)]) for d in range(-8, 17)] + \
        [Case("|d| > 8" if abs(d) > 8 else "d in [-8, 8]", [pts[0]], [u32(d)]) for d in range(-8, 17)]


def select_niels(rng):
    out = []
    for d in range(-8, 17):
        for row in (0, 31, rng.randrange(1, 31)):
            out.append(Case("|d| > 8" if abs(d) > 8 else "d in [-8, 8]", [], [u32(d), row]))
    return out


def mul_scalars(rng):
    return [0, 1, L - 1, L, (1 << 256) - 1, 0x8F << 248, 0x80 << 248, ALL8, RIPPLE] + mc.crafted_high_scalars(rng)[:6] + \
        [rng.getrandbits(256) for _ in range(6)]


def mul_var(rng):
    p = ec.mul(rbytes(rng, 32))
    pts = [ed.encode(ed.IDENT), mc.T8, bytes(32), p, ed.encode(ed.add(ed.decode(p), ed.decode(mc.T8)))]
    out = []
    for i, k in enumerate(mul_scalars(rng)):
        for j in (i % len(pts), (i + 2) % len(pts)):
            out.append(Case("scalar x point", [le(k), pts[j]]))
    return out


def mul_base(rng):
    return [Case("scalar", [le(k)]) for k in mul_scalars(rng)]


GEN = {"sha256_update": sha256_update, "sha256_zero": sha256_zero, "sha256_blocks": sha256_blocks, "hmac_sha256": hmac_sha256,
       "ecies_kdf": ecies_kdf, "sha512_3": sha512_3, "sha512_challenge": sha512_challenge, "blake2b": blake2b,
       "xb_root": xb_root_cases, "xb_block": xb_block_cases, "sc_pick": sc_pick_cases, "sc_canonical": sc_canonical,
       "sc_reduce512": sc_reduce512, "sc_neg": sc_neg, "sc_recode4": sc_recode4_cases, "sc_rule": sc_rule,
       "challenge_is": challenge_is, "aes_subbytes": aes_subbytes, "aes_expand": aes_expand, "aes_encrypt2": aes_encrypt2,
       "ghash": ghash, "gcm_seal": gcm_seal_cases, "gcm_open": gcm_open_cases, "select_cached": select_cached,
       "select_niels": select_niels, "mul_var": mul_var, "mul_base": mul_base}


# one shape per operation, the bytes drawn per lane: (fragment lengths, args) -> the fragments
def uniform(op: str, rng) -> list:
    n = {"mul_var": 8, "mul_base": 8, "select_cached": 16, "select_niels": 32, "gcm_seal": 32, "gcm_open": 32}.get(op, LANES)
    out = []
    for i in range(n):
        if op in ("sha256_update", "sha256_zero"):
            d = rbytes(rng, 150)
            c = Case("uniform", [d[:40], d[40:100], d[100:]], [64])
        elif op == "sha256_blocks":
            c = Case("uniform", [rbytes(rng, 192)])
        elif op == "hmac_sha256":
            c = Case("uniform", [rbytes(rng, 32), rbytes(rng, 20), rbytes(rng, 50), b""])
        elif op in ("ecies_kdf", "sc_canonical", "sc_neg", "sc_recode4", "sc_rule", "aes_subbytes", "aes_expand"):
            c = Case("uniform", [rbytes(rng, 32)])
        elif op in ("sha512_3", "sha512_challenge"):
            c = Case("uniform", [rbytes(rng, 32), rbytes(rng, 32), rbytes(rng, 200)])
        elif op == "blake2b":
            c = Case("uniform", [rbytes(rng, 300), b"", b"", b""], [64])
        elif op == "xb_root":
            c = Case("uniform", [rbytes(rng, 32), rbytes(rng, 100)])
        elif op == "xb_block":
            c = Case("uniform", [rbytes(rng, 64)], [i % 4])
        elif op == "sc_pick":
            c = Case("uniform", [rbytes(rng, 32)])
        elif op == "sc_reduce512":
            c = Case("uniform", [rbytes(rng, 64)])
        elif op == "challenge_is":
            w = le(rng.randrange(L))
            c = Case("uniform", [w, w])
        elif op == "aes_encrypt2":
            c = Case("uniform", [rbytes(rng, 32), rbytes(rng, 32)])
        elif op == "ghash":
            c = Case("uniform", [rbytes(rng, 16), rbytes(rng, 48)])
        elif op == "gcm_seal":
            c = Case("uniform", [rbytes(rng, 44), rbytes(rng, 40)])
        elif op == "gcm_open":
            k44 = rbytes(rng, 44)
            c = Case("uniform", [k44, ec.gcm_seal(k44[:32], k44[32:], rbytes(rng, 40))], fill=0xAA)
        elif op == "select_cached":
            c = Case("uniform", [ed.encode(ed.decode(sel_points()[i % 3]))], [5])
        elif op == "select_niels":
            c = Case("uniform", [], [u32(-3), i])
        elif op == "mul_var":
            c = Case("uniform", [rbytes(rng, 32), ec.mul(rbytes(rng, 32))])
        elif op == "mul_base":
            c = Case("uniform", [rbytes(rng, 32)])
        else:
            raise KeyError(op)
        out.append(c)
    return out


@dataclass
class Batch:
    op: str
    label: str
    cases: list


@functools.lru_cache(maxsize=None)
def batches() -> tuple:
    """per operation: every class in one shuffled launch ("mixed"), then one launch of one shape ("uniform")"""
    out = []
    for k, op in enumerate(OPS):
        rng = random.Random(1000 + k)
        mixed = GEN[op](rng)
        rng.shuffle(mixed)
        uni = uniform(op, rng)
        for b in (Batch(op, "mixed", mixed), Batch(op, "uniform", uni)):
            for c in b.cases:
                c.args = (list(c.args) + [0, 0, 0, 0])[:4]
                c.frags = (list(c.frags) + [b"", b"", b"", b""])[:4]
                c.want = expect(op, c.frags, c.args)
            out.append(b)
    return tuple(out)


def run_batch(lib, b: Batch):
    """one launch of the batch; returns (status, outputs)"""
    n = len(b.cases)
    hdr = np.zeros((n, HDR), dtype=np.uint32)
    pool, outs, fill = bytearray(), 0, bytearray()
    for i, c in enumerate(b.cases):
        for k, f in enumerate(c.frags):
            hdr[i, k], hdr[i, 4 + k] = len(pool), len(f)
            pool += f
        hdr[i, 8:12] = c.args
        hdr[i, 12], hdr[i, 13] = outs, len(c.want)
        outs += len(c.want)
        fill += bytes([c.fill]) * len(c.want)
    pool_buf = (ctypes.c_uint8 * max(len(pool), 1)).from_buffer_copy(bytes(pool) or b"\x00")
    out_buf = (ctypes.c_uint8 * max(outs, 1)).from_buffer_copy(bytes(fill) or b"\x00")
    st = lib.bh_run(OPS.index(b.op), n, hdr.ctypes.data_as(ctypes.c_void_p), pool_buf, ctypes.c_uint64(len(pool)), out_buf,
                    ctypes.c_uint64(outs))
    raw = bytes(out_buf)
    return st, [raw[hdr[i, 12]:hdr[i, 12] + hdr[i, 13]] for i in range(n)]


def _short(b: bytes) -> str:
    return b.hex() if len(b) <= 48 else f"{b[:24].hex()}..{b[-8:].hex()} ({len(b)} bytes)"


def run_all(lib, where: str, ops=None) -> list:
    """every batch (of the given operations) through the library lib; one line per wrong case (at most 20 per batch)"""
    lib.bh_run.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p,
                           ctypes.c_uint64]
    failures = []
    for b in batches():
        if ops is not None and b.op not in ops:
            continue
        st, got = run_batch(lib, b)
        if st:
            failures.append(f"{where} {b.op} [{b.label}]: status {st}")
            continue
        bad = [(i, c) for i, c in enumerate(b.cases) if got[i] != c.want]
        for i, c in bad[:20]:
            frags = ", ".join(_short(f) for f in c.frags if f)
            failures.append(f"{where} {b.op} [{b.label}, class {c.cls!r}] lane {i}: args {c.args} fragment lengths "
                            f"{[len(f) for f in c.frags]} input {frags}: got {_short(got[i])}, want {_short(c.want)}")
        if len(bad) > 20:
            failures.append(f"{where} {b.op} [{b.label}]: {len(bad) - 20} more wrong cases")
    return failures


def case_counts() -> dict:
    """{(op, class): number of cases}"""
    counts: dict = {}
    for b in batches():
        for c in b.cases:
            counts[(b.op, c.cls)] = counts.get((b.op, c.cls), 0) + 1
    return counts
