"""GPU: the edwards25519 MSM (b2k_ed25519_msm / _dev) and the share/poly entry points on it (RecoverCommit, PubPoly.Eval,
PubPoly.Check) against the oracle: every input set with forced windows and slice lengths, scalars on both sides of
geScalarMult's top-digit rule, points of every order, identity inputs, error reporting and a VSS round trip."""
import random
import struct

import pytest

from kyber_b200 import B2KError
from oracle import ed25519 as ed
import ed25519_msm_cases as cases

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_POINT = -2, -5


@pytest.fixture
def eng(engine):
    yield engine
    engine.set_msm_window(0)
    engine.set_msm_slice(0)


def _run(eng, scalars, ab):
    return eng.ed25519_msm(cases.le(scalars), cases.points(ab))


@pytest.mark.parametrize("n", [1, 2, 1000, 1 << 16])
@pytest.mark.parametrize("name", cases.SETS)
def test_msm_sets_match_the_oracle(eng, name, n):
    if name == "plus_minus" and n == 1:
        n = 2
    scalars, ab = cases.build_set(name, n)
    assert _run(eng, scalars, ab) == cases.msm_expected(scalars, ab), (name, n)
    plan = eng.last_msm_plan()
    assert plan["W"] == (256 + plan["c"]) // plan["c"] and plan["buckets_per_window"] == 1 << (plan["c"] - 1)


def test_msm_2_20(eng):
    scalars, ab = cases.build_set("uniform", 1 << 20)
    assert _run(eng, scalars, ab) == cases.msm_expected(scalars, ab)
    plan = eng.last_msm_plan()
    assert plan["c"] >= 12 and plan["W"] == (256 + plan["c"]) // plan["c"]
    t = eng.last_timings()
    assert len(t) >= 10 and t[0] > 0 and t[4] > 0 and t[8] >= t[0] + t[4]


@pytest.mark.parametrize("c", [4, 5, 8, 12, 16])
@pytest.mark.parametrize("L", [0, 3, 64])
@pytest.mark.parametrize("name", ["uniform", "equal", "plus_minus", "zeros", "small"])
def test_msm_forced_windows_and_slices(eng, name, c, L):
    eng.set_msm_window(c)
    eng.set_msm_slice(L)
    scalars, ab = cases.build_set(name, 2000, seed=c)
    assert _run(eng, scalars, ab) == cases.msm_expected(scalars, ab), (name, c, L)
    plan = eng.last_msm_plan()
    assert plan["c"] == c and (L == 0 or plan["slice_len"] == L)


def test_equal_scalars_at_scale_with_short_slices(eng):
    eng.set_msm_slice(4)
    scalars, ab = [1] * (1 << 16), [(12345, 3)] * (1 << 16)         # a cosi-style sum: unit scalars, one point
    assert _run(eng, scalars, ab) == cases.msm_expected(scalars, ab)


def test_mixed_order_points_term_by_term(eng):
    rng = random.Random(2)
    n = 96
    pts = [cases.mixed_point(i) for i in range(n - 3)] + [cases.T8, cases.ZERO, cases.IDENTITY]
    ks = [rng.getrandbits(256) for _ in range(n)]
    ks[:8] = cases.crafted_high_scalars(rng)
    acc = ed.IDENT
    for k, p in zip(ks, pts):
        acc = ed.add(acc, cases.ge_scalar_mult(k.to_bytes(32, "little"), ed.decode(p)))
    assert eng.ed25519_msm(cases.le(ks), b"".join(pts)) == ed.encode(acc)


def test_high_scalars_on_both_sides_of_the_rule(eng):
    rng = random.Random(7)
    ks = cases.crafted_high_scalars(rng)
    assert {cases.top_digit(k) for k in ks} >= {8, 9, 16}
    for k in ks:
        for p in (ed.encode(ed.BASE), cases.mixed_point(11)):
            want = ed.encode(cases.ge_scalar_mult(k.to_bytes(32, "little"), ed.decode(p)))
            assert eng.ed25519_msm(k.to_bytes(32, "little"), p) == want, hex(k)


def test_identity_inputs(eng):
    n = 500
    assert eng.ed25519_msm(cases.le([random.Random(1).getrandbits(256) for _ in range(n)]), cases.IDENTITY * n) == cases.IDENTITY
    assert eng.ed25519_msm(cases.le([0] * n), cases.points([(5, 1)] * n)) == cases.IDENTITY
    assert eng.ed25519_msm((1).to_bytes(32, "little"), cases.ZERO) == cases.ZERO               # all-zero is a point, not the identity
    assert eng.ed25519_msm((4).to_bytes(32, "little"), cases.ZERO) == cases.IDENTITY           # of order 4
    assert eng.ed25519_msm(cases.le([1, 1]), cases.ZERO * 2) != cases.IDENTITY


def test_undecodable_point_and_recovery(eng):
    scalars, ab = cases.build_set("uniform", 300)
    pts = bytearray(cases.points(ab))
    pts[32 * 9:32 * 10] = (2).to_bytes(32, "little")
    with pytest.raises(B2KError) as e:
        eng.ed25519_msm(cases.le(scalars), bytes(pts))
    assert e.value.code == ERR_POINT
    assert _run(eng, scalars, ab) == cases.msm_expected(scalars, ab)


def test_dev_form_matches_host_and_reports_at_wait(eng):
    import torch
    scalars, ab = cases.build_set("mixed", 5000)
    s, p = cases.le(scalars), cases.points(ab)
    host = eng.ed25519_msm(s, p)
    dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    d_s, d_p, d_o = dev(s), dev(p), torch.zeros(32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.ed25519_msm_dev(5000, d_s.data_ptr(), d_p.data_ptr(), d_o.data_ptr())
    eng.wait()
    assert bytes(d_o.cpu().numpy().tobytes()) == host == cases.msm_expected(scalars, ab)
    d_p[32 * 3:32 * 4] = torch.tensor(list((2).to_bytes(32, "little")), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.ed25519_msm_dev(5000, d_s.data_ptr(), d_p.data_ptr(), d_o.data_ptr())
    with pytest.raises(B2KError) as e:
        eng.wait()
    assert e.value.code == ERR_POINT
    eng.ed25519_msm_dev(5000, d_s.data_ptr(), dev(p).data_ptr(), d_o.data_ptr())
    eng.wait()
    assert bytes(d_o.cpu().numpy().tobytes()) == host


def test_bad_arguments(eng):
    lib, h = eng.lib, eng.h
    assert lib.b2k_ed25519_msm(h, 4, None, None, None) == ERR_ARG
    assert lib.b2k_ed25519_msm_dev(h, 4, None, None, None) == ERR_ARG
    with pytest.raises(B2KError) as e:
        eng.ed25519_msm(b"", b"")                                                # n = 0
    assert e.value.code == ERR_ARG


# ---- VSS round trip -------------------------------------------------------------------------------------------------------
def _poly(rng, t):
    a = [rng.randrange(ed.L) for _ in range(t)]
    return a, b"".join(ed.encode(ed.scalar_mult(x)) for x in a)


def _f(a, x):
    return sum(c * pow(x, j, ed.L) for j, c in enumerate(a)) % ed.L


def test_pubpoly_check_over_dealers(eng):
    rng = random.Random(13)
    m, t, n = 4, 6, 20
    polys = [_poly(rng, t) for _ in range(m)]
    idx = [[rng.randrange(1 << 32) if k == 0 else k for k in range(n)] for _ in range(m)]
    shares = [[_f(a, i + 1) for i in row] for (a, _), row in zip(polys, idx)]
    want = [[1] * n for _ in range(m)]
    for d in range(m):                                   # corruptions: off by one, another dealer's share, a high-scalar form
        shares[d][3] = (shares[d][3] + 1) % ed.L; want[d][3] = 0
        shares[d][5] = shares[(d + 1) % m][5]; want[d][5] = 0
        shares[d][7] += ed.L                             # same point (prime order): still valid
        k = shares[d][9] | (0x9 << 252)                  # top digit >= 9: geScalarMult drops it, so this is not f(x) B
        shares[d][9] = k; want[d][9] = int(ed.encode(cases.ge_scalar_mult(k.to_bytes(32, "little"), ed.BASE)) ==
                                           ed.encode(ed.scalar_mult(_f(polys[d][0], idx[d][9] + 1))))
    ok = eng.ed25519_pubpoly_check(b"".join(c for _, c in polys), t, idx, cases.le([s for row in shares for s in row]))
    assert list(ok) == [w for row in want for w in row]


def test_pubpoly_eval_matches_the_oracle(eng):
    rng = random.Random(17)
    a, commits = _poly(rng, 9)
    idx = [0, 1, 2, 77, 65535, 0xffffffff]
    out = eng.ed25519_pubpoly_eval(commits, idx)
    for k, i in enumerate(idx):
        assert out[32 * k:32 * k + 32] == ed.encode(ed.scalar_mult(_f(a, i + 1))), i


@pytest.mark.parametrize("t", [1, 2, 1024])
def test_recover_commit_returns_the_secret_commitment(eng, t):
    rng = random.Random(t)
    a, commits = _poly(rng, t)
    idx = rng.sample(range(5000), t)
    pub = eng.ed25519_pubpoly_eval(commits, idx)
    assert eng.ed25519_recover_commit(idx, pub) == commits[:32]
    assert eng.last_msm_plan()["W"] > 0


def test_recover_commit_duplicate_indices(eng):
    rng = random.Random(3)
    a, commits = _poly(rng, 3)
    pub = eng.ed25519_pubpoly_eval(commits, [4, 9, 4])
    with pytest.raises(B2KError) as e:
        eng.ed25519_recover_commit([4, 9, 4], pub)
    assert e.value.code == ERR_ARG
    assert eng.ed25519_recover_commit([4, 9, 11], eng.ed25519_pubpoly_eval(commits, [4, 9, 11])) == commits[:32]
