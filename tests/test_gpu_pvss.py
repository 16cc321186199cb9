"""GPU: DLEQ proof verification and the PVSS share checks on edwards25519 (b2k_ed25519_dleq_verify / _dev,
b2k_ed25519_pvss_verify_enc_shares, b2k_ed25519_pvss_verify_dec_shares) against the restatement in tests/pvss_cases.py.

Bulk inputs are built with the engine's b2k_ed25519_mul_batch (tested on its own in test_gpu_ed25519.py) and
b2k_ed25519_pubpoly_eval, the challenges with hashlib and the restated Pick; a sample of every batch is re-checked with the
pure-Python oracle."""
import hashlib
import random

import pytest

import pvss_cases as pc

pytestmark = pytest.mark.gpu
L = pc.L
OK, CHALLENGE, INVALID, POINT = pc.OK, pc.CHALLENGE, pc.INVALID, pc.POINT


@pytest.fixture(scope="module")
def eng():
    from kyber_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def le(k: int) -> bytes:
    return (k % (1 << 256)).to_bytes(32, "little")


def chunks(b: bytes, w: int = 32):
    return [b[i:i + w] for i in range(0, len(b), w)]


def muls(eng, ks, pts) -> list:
    """[k_i P_i] by b2k_ed25519_mul_batch (the raw integer k_i, as Point.Mul)"""
    if isinstance(pts, bytes):
        pts = [pts] * len(ks)
    return chunks(eng.ed25519_mul_batch(b"".join(le(k) for k in ks), b"".join(pts)))


def with_r(proof: bytes, r: int) -> bytes:
    return proof[:32] + le(r) + proof[64:]


def with_c(proof: bytes, c: int) -> bytes:
    return le(c) + proof[32:]


# ---- dleq_verify ----------------------------------------------------------------------------------------------------------------
def make_dleq(eng, n: int, seed: int):
    """n honest proofs on prime-order bases (R is reduced mod l, so a torsion part in G or H would break them, in the reference
    too): (g, h, xg, xh, proofs) as lists of bytes; C is any scalar, Verify does not hash"""
    rng = random.Random(seed)
    a = [rng.randrange(1, L) for _ in range(2 * n)]
    gh = muls(eng, a, pc.G)
    g, h = gh[:n], gh[n:]
    x = [rng.randrange(L) for _ in range(n)]
    v = [rng.randrange(L) for _ in range(n)]
    c = [rng.randrange(L) for _ in range(n)]
    out = muls(eng, x + x + v + v, g + h + g + h)
    xg, xh, vg, vh = out[:n], out[n:2 * n], out[2 * n:3 * n], out[3 * n:]
    proofs = [le(ci) + le((vi - xi * ci) % L) + a_ + b_ for ci, vi, xi, a_, b_ in zip(c, v, x, vg, vh)]
    return g, h, xg, xh, proofs


def run_dleq(eng, g, h, xg, xh, proofs):
    return list(eng.ed25519_dleq_verify(*(b"".join(z) for z in (g, h, xg, xh, proofs))))


def corrupt_dleq(case, kind, rng):
    g, h, xg, xh, p = case
    c, r = int.from_bytes(p[:32], "little"), int.from_bytes(p[32:64], "little")
    other = pc.base_mul(rng.randrange(1, L))
    return {
        "c+1": (g, h, xg, xh, with_c(p, c + 1)), "c-1": (g, h, xg, xh, with_c(p, c - 1)),
        "r+1": (g, h, xg, xh, with_r(p, r + 1)), "r-1": (g, h, xg, xh, with_r(p, r - 1)),
        "vg_other": (g, h, xg, xh, p[:64] + other + p[96:]), "vh_other": (g, h, xg, xh, p[:96] + other),
        "vg_t8": (g, h, xg, xh, p[:64] + pc.add(p[64:96], pc.T8) + p[96:]), "vh_t8": (g, h, xg, xh, p[:96] + pc.add(p[96:], pc.T8)),
        "swap_gh": (h, g, xg, xh, p),
        "pt_g": (pc.undecodable(), h, xg, xh, p), "pt_h": (g, pc.undecodable(), xg, xh, p),
        "pt_xg": (g, h, pc.undecodable(), xh, p), "pt_xh": (g, h, xg, pc.undecodable(), p),
        "pt_vg": (g, h, xg, xh, p[:64] + pc.undecodable() + p[96:]), "pt_vh": (g, h, xg, xh, p[:96] + pc.undecodable()),
    }[kind]


KINDS = ["c+1", "c-1", "r+1", "r-1", "vg_other", "vh_other", "vg_t8", "vh_t8", "swap_gh",
         "pt_g", "pt_h", "pt_xg", "pt_xh", "pt_vg", "pt_vh"]


@pytest.mark.parametrize("n", [1, 2, 1000, 1 << 16])
def test_dleq_verify_honest_and_corrupted(eng, n):
    rng = random.Random(n)
    cols = list(make_dleq(eng, n, seed=n))
    assert run_dleq(eng, *cols) == [OK] * n
    where = sorted({0, n - 1} | {rng.randrange(n) for _ in range(len(KINDS))})
    want = {}
    for k, i in enumerate(where):
        kind = KINDS[k % len(KINDS)] if n > 2 else KINDS[(k + n) % len(KINDS)]
        case = corrupt_dleq(tuple(col[i] for col in cols), kind, rng)
        for col, val in zip(cols, case):
            col[i] = val
        want[i] = pc.dleq_verify(*case)
        assert want[i] == (POINT if kind.startswith("pt_") else INVALID), kind
    got = run_dleq(eng, *cols)
    assert {i: s for i, s in enumerate(got) if s != OK} == want
    for i in rng.sample(range(n), min(n, 3)):                  # a sample against the pure-Python oracle
        assert got[i] == pc.dleq_verify(*(col[i] for col in cols))


def test_dleq_every_corruption_kind(eng):
    rng = random.Random(7)
    base = make_dleq(eng, len(KINDS), seed=7)
    cases = [corrupt_dleq(tuple(col[i] for col in base), kind, rng) for i, kind in enumerate(KINDS)]
    got = run_dleq(eng, *[list(z) for z in zip(*cases)])
    assert got == [pc.dleq_verify(*cs) for cs in cases]
    assert got == [POINT if k.startswith("pt_") else INVALID for k in KINDS]


def test_dleq_raw_scalar_reading(eng):
    """R + l and R with a top digit above 8 give what ge_scalar_mult predicts, with and without torsion in G"""
    rng = random.Random(8)
    cases, want = [], []
    for torsion in (False, True):
        g, h, xg, xh, p = [c[0] for c in make_dleq(eng, 1, seed=80 + torsion)]
        if torsion:
            g = pc.add(g, pc.T8)
            p = p[:32] + p[32:64] + pc.add(pc.mul(int.from_bytes(p[32:64], "little"), g), pc.mul(int.from_bytes(p[:32], "little"), xg)) + p[96:]
        r = int.from_bytes(p[32:64], "little")
        for r2 in [r, r + L, r + 2 * L] + [k for k in pc.mc.crafted_high_scalars(rng)]:
            q = with_r(p, r2)
            cases.append((g, h, xg, xh, q))
            want.append(pc.dleq_verify(g, h, xg, xh, q))
    got = run_dleq(eng, *[list(z) for z in zip(*cases)])
    assert got == want
    assert OK in got and INVALID in got


def test_dleq_v_zero_with_noncanonical_identities(eng):
    rng = random.Random(9)
    g, h = pc.random_point(rng), pc.random_point(rng)
    proof, xg, xh = pc.new_dleq_proof(g, h, rng.randrange(L), 0)
    nc = pc.noncanonical_identity()
    assert run_dleq(eng, [g, g], [h, h], [xg, xg], [xh, xh], [proof, proof[:64] + nc + nc]) == [OK, OK]


def test_dleq_dev_matches_host(eng):
    import torch
    n = 4096
    cols = list(make_dleq(eng, n, seed=11))
    for i in range(0, n, 97):
        cols[4][i] = with_r(cols[4][i], int.from_bytes(cols[4][i][32:64], "little") + 1)
    host = bytes(run_dleq(eng, *cols))
    dev = [torch.frombuffer(bytearray(b"".join(c)), dtype=torch.uint8).cuda() for c in cols]
    d_st = torch.full((n,), 0xAA, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.ed25519_dleq_verify_dev(n, *[d.data_ptr() for d in dev], d_st.data_ptr())
    eng.synchronize()
    assert bytes(d_st.cpu().numpy()) == host
    assert host.count(bytes([INVALID])) == len(range(0, n, 97))


def test_refusals_then_a_correct_call(eng):
    from kyber_b200.capi import ERR_ARG, _buf
    g, h, xg, xh, p = [c[0] for c in make_dleq(eng, 1, seed=12)]
    lib, hd = eng.lib, eng.h
    st = bytearray(1)
    bufs = [_buf(x) for x in (g, h, xg, xh, p, st)]
    q = [b[0] for b in bufs]
    assert lib.b2k_ed25519_dleq_verify(hd, 0, *q) == ERR_ARG
    assert lib.b2k_ed25519_dleq_verify(hd, 1, q[0], None, *q[2:]) == ERR_ARG
    assert lib.b2k_ed25519_dleq_verify_dev(hd, 1, *q[:5], None) == ERR_ARG
    assert lib.b2k_ed25519_pvss_verify_enc_shares(hd, 1, 0, 1, *q[:4], q[4], q[5], q[5]) == ERR_ARG
    assert lib.b2k_ed25519_pvss_verify_enc_shares(hd, 1 << 16, 1, 1 << 15, *q[:4], q[4], q[5], q[5]) == ERR_ARG
    assert lib.b2k_ed25519_pvss_verify_enc_shares(hd, 1 << 16, 1 << 15, 1, *q[:4], q[4], q[5], q[5]) == ERR_ARG
    assert lib.b2k_ed25519_pvss_verify_dec_shares(hd, 0, *q[:5], q[5]) == ERR_ARG
    assert lib.b2k_ed25519_dleq_verify(hd, 1, *q) == 0 and bytes(st) == b"\x00"


# ---- enc shares ------------------------------------------------------------------------------------------------------------------
class Deals:
    """m honest deals of n encrypted shares, threshold t, built on the device: one polynomial for every deal (the shares are
    Python integers), a base H, keys X, commitments and proofs per deal"""

    def __init__(self, eng, m, n, t, seed):
        rng = random.Random(seed)
        self.m, self.n, self.t = m, n, t
        coeffs = [rng.randrange(L) for _ in range(t)]
        self.s = [sum(a * pow(i + 1, j, L) for j, a in enumerate(coeffs)) % L for i in range(n)]
        self.h = muls(eng, [rng.randrange(1, L) for _ in range(m)], pc.G)
        priv = [rng.randrange(1, L) for _ in range(m * n)]
        self.x = muls(eng, priv, pc.G)
        self.commits = [muls(eng, coeffs, self.h[d]) for d in range(m)]
        hs = [self.h[d] for d in range(m) for _ in range(n)]
        ss = self.s * m
        v = [rng.randrange(L) for _ in range(m * n)]
        out = muls(eng, ss + v + v, hs + hs + self.x)
        vg, vh = out[m * n:2 * m * n], out[2 * m * n:]
        self.sh = out[:m * n]                                  # s_i H = coms[i]
        self.v = muls(eng, ss, self.x)                         # s_i X_i
        self.proofs = []
        self.chal = []
        for d in range(m):
            sl = slice(d * n, (d + 1) * n)
            coms = chunks(eng.ed25519_pubpoly_eval(b"".join(self.commits[d]), list(range(n))))
            assert coms == self.sh[sl]
            c = pc.pick(pc.Xof(hashlib.sha256(b"".join(coms + self.v[sl] + vg[sl] + vh[sl])).digest()))
            self.chal.append(c)
            ci = int.from_bytes(c, "little")
            self.proofs += [c + le((vi - si * ci) % L) + a + b for vi, si, a, b in zip(v[sl], self.s, vg[sl], vh[sl])]

    def run(self, eng, h=None, commits=None, x=None, sh=None, v=None, proofs=None):
        return list(eng.ed25519_pvss_verify_enc_shares(b"".join(h or self.h), b"".join(b"".join(c) for c in (commits or self.commits)),
                                                         self.t, *(b"".join(z) for z in (x or self.x, sh or self.sh, v or self.v,
                                                                                         proofs or self.proofs))))

    def oracle(self, d, x=None, sh=None, v=None, proofs=None, commits=None, h=None):
        sl = slice(d * self.n, (d + 1) * self.n)
        return pc.verify_enc_share_batch((h or self.h)[d], (commits or self.commits)[d], (x or self.x)[sl], (sh or self.sh)[sl],
                                         (v or self.v)[sl], (proofs or self.proofs)[sl])


@pytest.mark.parametrize("m", [1, 4, 64])
@pytest.mark.parametrize("n", [1, 2, 10, 100, 1000])
@pytest.mark.parametrize("tk", ["one", "half", "all"])
def test_enc_shares_honest_deals(eng, m, n, tk):
    t = {"one": 1, "half": n // 2 + 1, "all": n}[tk]
    D = Deals(eng, m, n, t, seed=m * 100000 + n * 10 + t)
    assert D.run(eng) == [OK] * (m * n)
    if n <= 10 and m <= 4:
        assert D.oracle(m - 1) == [OK] * n


def test_enc_shares_hashed_items_flip_the_whole_deal(eng):
    m, n, t = 4, 10, 4
    D = Deals(eng, m, n, t, seed=21)
    other = pc.base_mul(12345)
    flips = {
        "v": dict(v=D.v[:n + 3] + [pc.add(D.v[n + 3], pc.G)] + D.v[n + 4:]),
        "vg": dict(proofs=D.proofs[:n + 3] + [D.proofs[n + 3][:64] + other + D.proofs[n + 3][96:]] + D.proofs[n + 4:]),
        "vh": dict(proofs=D.proofs[:n + 3] + [D.proofs[n + 3][:96] + other] + D.proofs[n + 4:]),
        "commit": dict(commits=[D.commits[0], D.commits[1][:2] + [other] + D.commits[1][3:]] + D.commits[2:]),
        "swap": dict(x=D.x[:n] + [D.x[n + 1], D.x[n]] + D.x[n + 2:], sh=D.sh[:n] + [D.sh[n + 1], D.sh[n]] + D.sh[n + 2:],
                     v=D.v[:n] + [D.v[n + 1], D.v[n]] + D.v[n + 2:],
                     proofs=D.proofs[:n] + [D.proofs[n + 1], D.proofs[n]] + D.proofs[n + 2:]),
    }
    for name, kw in flips.items():
        got = D.run(eng, **kw)
        assert got[n:2 * n] == [CHALLENGE] * n, name
        assert got[:n] + got[2 * n:] == [OK] * ((m - 1) * n), name
        assert got[n:2 * n] == D.oracle(1, **kw), name


def test_enc_shares_share_local_failures_and_points(eng):
    m, n, t = 3, 10, 3
    D = Deals(eng, m, n, t, seed=22)
    x, sh, proofs, v = D.x[:], D.sh[:], D.proofs[:], D.v[:]
    proofs[2] = with_r(proofs[2], int.from_bytes(proofs[2][32:64], "little") + 1)      # broken proof: INVALID
    sh[5] = pc.add(sh[5], pc.G)                                                       # wrong sH: INVALID
    x[n + 1] = pc.undecodable()                                                       # X: POINT for that share only
    sh[n + 4] = pc.undecodable()                                                      # sH: same
    v[2 * n + 6] = pc.undecodable()                                                   # V of deal 2: every share POINT
    got = D.run(eng, x=x, sh=sh, proofs=proofs, v=v)
    want = [OK] * (m * n)
    want[2] = want[5] = INVALID
    want[n + 1] = want[n + 4] = POINT
    want[2 * n:] = [POINT] * n
    assert got == want
    assert got[:n] == D.oracle(0, x=x, sh=sh, proofs=proofs, v=v)
    assert got[n:2 * n] == D.oracle(1, x=x, sh=sh, proofs=proofs, v=v)
    for h in ([pc.undecodable()] + D.h[1:],):
        assert D.run(eng, h=h)[:n] == [POINT] * n
    bad_commit = [D.commits[0]] + [[pc.undecodable()] + D.commits[1][1:]] + D.commits[2:]
    assert D.run(eng, commits=bad_commit)[n:2 * n] == [POINT] * n
    vg_bad = D.proofs[:n] + [D.proofs[n][:64] + pc.undecodable() + D.proofs[n][96:]] + D.proofs[n + 1:]
    got = D.run(eng, proofs=vg_bad)
    assert got[n:2 * n] == [POINT] * n and got[:n] == [OK] * n
    c_bad = D.proofs[:7] + [with_c(D.proofs[7], int.from_bytes(D.chal[0], "little") + L)] + D.proofs[8:]
    assert D.run(eng, proofs=c_bad)[:n] == [OK] * 7 + [CHALLENGE] + [OK] * (n - 8)


def test_enc_shares_zero_commitment_noncanonical_identity(eng):
    """a share whose proof commitment v is 0 (VG = VH = identity) sent with non-canonical identities keeps its deal OK: the
    challenge hashes the canonical re-encodings"""
    rng = random.Random(23)
    n, t = 4, 2
    h = pc.random_point(rng)
    priv = [rng.randrange(1, L) for _ in range(n)]
    xs = [pc.base_mul(k) for k in priv]
    coeffs = [rng.randrange(L) for _ in range(t)]
    s = [sum(a * pow(i + 1, j, L) for j, a in enumerate(coeffs)) % L for i in range(n)]
    commits = [pc.mul(a, h) for a in coeffs]
    sh = [pc.mul(si, h) for si in s]
    vs = [pc.mul(si, x) for si, x in zip(s, xs)]
    v = [rng.randrange(L) for _ in range(n)]
    v[1] = 0
    vg = [pc.mul(vi, h) for vi in v]
    vh = [pc.mul(vi, x) for vi, x in zip(v, xs)]
    c = pc.pick(pc.Xof(hashlib.sha256(b"".join(sh + vs + vg + vh)).digest()))
    ci = int.from_bytes(c, "little")
    nc = pc.noncanonical_identity()
    proofs = [c + le((vi - si * ci) % L) + (nc if i == 1 else a) + (nc if i == 1 else b) for i, (vi, si, a, b) in enumerate(zip(v, s, vg, vh))]
    got = list(eng.ed25519_pvss_verify_enc_shares(h, b"".join(commits), t, b"".join(xs), b"".join(sh), b"".join(vs), b"".join(proofs)))
    assert got == pc.verify_enc_share_batch(h, commits, xs, sh, vs, proofs) == [OK] * n


# ---- dec shares and the round trip -----------------------------------------------------------------------------------------------
def test_dec_shares_statuses_and_round_trip(eng):
    rng = random.Random(31)
    n, t = 7, 4
    h = pc.random_point(rng)
    priv = [rng.randrange(1, L) for _ in range(n)]
    xs = [pc.base_mul(k) for k in priv]
    secret = rng.randrange(L)
    commits, shares, _ = pc.enc_shares(h, xs, secret, t, pc.RandomStream("gpu round trip"))
    shs = chunks(eng.ed25519_pubpoly_eval(b"".join(commits), list(range(n))))
    vs = [v for _, v, _ in shares]
    proofs = [p for _, _, p in shares]
    st = list(eng.ed25519_pvss_verify_enc_shares(h, b"".join(commits), t, b"".join(xs), b"".join(shs), b"".join(vs), b"".join(proofs)))
    assert st == pc.verify_enc_share_batch(h, commits, xs, shs, vs, proofs) == [OK] * n
    dec = [pc.dec_share(priv[i], vs[i], rng.randrange(L)) for i in range(n)]
    dv = [d for d, _ in dec]
    dp = [p for _, p in dec]

    def run(dv_, dp_):
        return list(eng.ed25519_pvss_verify_dec_shares(pc.G, b"".join(xs), b"".join(vs), b"".join(dv_), b"".join(dp_)))

    assert run(dv, dp) == [OK] * n
    dv2, dp2 = dv[:], dp[:]
    dv2[0] = pc.add(dv2[0], pc.G)                                                      # wrong decV: INVALID
    dp2[1] = dp2[1][:64] + pc.base_mul(99) + dp2[1][96:]                               # wrong VG: CHALLENGE
    dp2[2] = with_c(dp2[2], int.from_bytes(dp2[2][:32], "little") + L)                 # C not canonical: CHALLENGE
    dp2[3] = dp2[3][:96] + pc.undecodable()                                            # POINT
    got = run(dv2, dp2)
    assert got == [INVALID, CHALLENGE, CHALLENGE, POINT, OK, OK, OK]
    assert got == [pc.verify_dec_share(pc.G, xs[i], vs[i], dv2[i], dp2[i]) for i in range(n)]
    # RecoverSecret composed as the bindings compose it: statuses, then RecoverCommit over the first t valid shares by index
    for corrupt, expect_ok in ((0, True), (n - t, True), (n - t + 1, False)):
        dvc = [pc.add(d, pc.G) if i < corrupt else d for i, d in enumerate(dv)]
        status = run(dvc, dp)
        good = [i for i in range(n) if status[i] == OK]
        assert len(good) == n - corrupt
        if not expect_ok:
            assert len(good) < t and pc.recover_secret(pc.G, xs, vs, list(zip(range(n), dvc, dp)), t) is None
            assert eng.ed25519_pvss_recover_secret(pc.G, list(range(n)), b"".join(xs), b"".join(vs), b"".join(dvc),
                                                   b"".join(dp), t) is None
            continue
        got = eng.ed25519_pvss_recover_secret(pc.G, list(range(n)), b"".join(xs), b"".join(vs), b"".join(dvc), b"".join(dp), t)
        assert got == pc.base_mul(secret) == pc.recover_secret(pc.G, xs, vs, list(zip(range(n), dvc, dp)), t)


# ---- scale -----------------------------------------------------------------------------------------------------------------------
def test_scale_enc_shares_64_deals_of_1024(eng):
    m, n, t = 64, 1024, 16
    D = Deals(eng, m, n, t, seed=41)
    proofs, v = D.proofs[:], D.v[:]
    for i in (0, 5 * n + 17, 40 * n + 1023, m * n - 1):
        proofs[i] = with_r(proofs[i], int.from_bytes(proofs[i][32:64], "little") + 1)
    v[9 * n + 100] = pc.add(v[9 * n + 100], pc.G)
    got = D.run(eng, proofs=proofs, v=v)
    want = [OK] * (m * n)
    for i in (0, 5 * n + 17, 40 * n + 1023, m * n - 1):
        want[i] = INVALID
    want[9 * n:10 * n] = [CHALLENGE] * n
    assert got == want
    rng = random.Random(42)
    for i in rng.sample([i for i in range(m * n) if i // n != 9], 4):   # the proofs themselves, by the pure-Python oracle
        d = i // n
        assert pc.dleq_holds(D.h[d], D.x[i], D.sh[i], v[i], proofs[i]) == (got[i] == OK)


def test_scale_dleq_2_20(eng):
    n = 1 << 20
    base = make_dleq(eng, 1 << 14, seed=43)
    cols = [list(c) * (n >> 14) for c in base]
    where = {3: "r+1", 77777: "vh_t8", n // 2 + 5: "pt_xg", n - 1: "swap_gh"}
    rng = random.Random(44)
    want = {}
    for i, kind in where.items():
        case = corrupt_dleq(tuple(col[i] for col in cols), kind, rng)
        for col, val in zip(cols, case):
            col[i] = val
        want[i] = pc.dleq_verify(*case)
    got = run_dleq(eng, *cols)
    assert {i: s for i, s in enumerate(got) if s != OK} == want
