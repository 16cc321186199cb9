"""GPU parity of the Pippenger MSM in every group it is instantiated for (BLS12-381 G1 and G2, bn254 G1 and G2, bn256 G1 and
G2): skewed input sets through forced windows, slice lengths, reduction chunks and levels, the grouped tail and the
one-thread-per-bucket variant, every plan checked against the oracle and against what last_msm_plan() reports.

The six instantiations are compiled separately (Fp, Fp2, 8, 10 and 12 limbs), so a bug in one of them, e.g. in the
block-parallel fix-up of a bucket cut into more than 64 slices, or in the doubling branch of xyzz_add between equal slice
partials, shows only in that group.  Input sets and expected values: tests/msm_cases.py."""
import random
import re

import pytest

import msm_cases as mc
from kyber_b200 import B2KError

pytestmark = pytest.mark.gpu

GROUP_NAMES = list(mc.GROUPS)
# group -> (host MSM, fixed-base batch that returns operand-form points, curve config of the kernels' template argument)
ENTRY = {
    "bls12381_g1": ("b2k_bls12381_g1_msm", "b2k_bls12381_g1_mul_batch_affine", "Bls381G1"),
    "bls12381_g2": ("b2k_bls12381_g2_msm", "b2k_bls12381_g2_mul_batch_affine", "Bls381G2"),
    "bn254_g1": ("b2k_bn254_g1_msm", "b2k_bn254_g1_mul_batch", "Bn254G1"),
    "bn254_g2": ("b2k_bn254_g2_msm", "b2k_bn254_g2_mul_batch", "Bn254G2"),
    "bn256_g1": ("b2k_bn256_g1_msm", "b2k_bn256_g1_mul_batch", "Bn256G1"),
    "bn256_g2": ("b2k_bn256_g2_msm", "b2k_bn256_g2_mul_batch", "Bn256G2"),
}
N_SET = 2000            # pairs of every input set: the all-equal set puts 2000 entries into one bucket per window

# c = window bits, L = slice length, m = reduction chunk (b2k_set_msm_chunk), reduce = (levels, m1, m2), groups = window groups
# of the overlapped tail, variant = one thread per bucket
PLANS = (
    {},
    {"c": 4}, {"c": 5}, {"c": 7}, {"c": 12}, {"c": 16},
    {"L": 1}, {"L": 3}, {"L": 64}, {"c": 16, "L": 1},
    {"c": 7, "m": 1}, {"c": 7, "m": 64}, {"c": 12, "m": 1}, {"c": 12, "m": 2048},
    {"c": 12, "reduce": (1, 0, 0)}, {"c": 12, "reduce": (2, 0, 0)}, {"c": 12, "reduce": (2, 1, 4)}, {"c": 16, "reduce": (2, 0, 0)},
    {"c": 5, "reduce": (2, 0, 0)},            # 16 buckets per window are not a multiple of 8 x 4: one level
    {"c": 7, "groups": 2}, {"c": 5, "groups": 8},
    {"variant": True}, {"c": 12, "variant": True},
)


@pytest.fixture(autouse=True)
def _reset_msm_knobs(engine):
    yield
    _reset(engine)


def _reset(engine):
    engine.set_msm_window(0)
    engine.set_msm_slice(0)
    engine._check(engine.lib.b2k_set_msm_chunk(engine.h, 0))
    engine.set_msm_reduce(0, 0, 0)
    engine.set_msm_groups(1)
    engine.set_msm_variant(False)
    engine._check(engine.lib.b2k_set_msm_layout(engine.h, 0))
    engine.set_msm_glv(True)
    engine.set_msm_affine(-1, 0)


def _apply(engine, plan):
    _reset(engine)
    engine.set_msm_window(plan.get("c", 0))
    engine.set_msm_slice(plan.get("L", 0))
    engine._check(engine.lib.b2k_set_msm_chunk(engine.h, plan.get("m", 0)))
    engine.set_msm_reduce(*plan.get("reduce", (0, 0, 0)))
    engine.set_msm_groups(plan.get("groups", 1))
    engine.set_msm_variant(plan.get("variant", False))


def _pipeline_bits(g):
    return 127 if g.name == "bls12381_g1" else g.scalar_bits      # BLS12-381 G1 runs over the 127-bit halves of the GLV split


def _check_plan(engine, g, plan, launches, ctx):
    """last_msm_plan() reports what the plan asked for, or the documented fallback"""
    got = engine.last_msm_plan()
    c = got["c"]
    if "c" in plan:
        assert c == plan["c"], (ctx, got)
    assert got["W"] == (_pipeline_bits(g) + c) // c and got["buckets_per_window"] == 1 << (c - 1), (ctx, got)
    if "L" in plan:
        assert got["slice_len"] == plan["L"], (ctx, got)
    if "m" in plan:
        assert got["chunk"] == plan["m"], (ctx, got)
    if "reduce" in plan:
        levels, m1, m2 = plan["reduce"]
        m1, m2 = m1 or 8, m2 or 4
        if levels == 2 and (1 << (c - 1)) % (m1 * m2) == 0:
            assert got["reduce_levels"] == 2 and got["reduce_chunks"] == [m1, m2], (ctx, got)
        else:
            assert got["reduce_levels"] == 1, (ctx, got)
    if "groups" in plan:
        # the grouped tail: point load, count, 3 scan passes, scatter, group ranges, final, and per group the accumulate,
        # fix-up, big-bucket fix-up, chunk reduction and window sum
        assert launches == 8 + 5 * plan["groups"], (ctx, launches)


def _operands(engine, g, a, spot=(0, 1, -1)):
    """P_i = a_i G by the engine's fixed-base batch (operand form), a few re-checked against the oracle"""
    n = len(a)
    pts = engine.call_host(ENTRY[g.name][1], n, mc.scalars_to_bytes(a), g.gen * n, g.in_bytes * n)
    for i in list(spot) + ([a.index(0)] if 0 in a else []):
        i %= n
        assert pts[g.in_bytes * i:g.in_bytes * (i + 1)] == g.operand(g.mul(a[i])), (g.name, i)
    return pts


def _msm(engine, g, sb, pts):
    return engine.call_host(ENTRY[g.name][0], len(sb) // 32, sb, pts, g.out_bytes)


@pytest.mark.parametrize("set_name", mc.SETS)
@pytest.mark.parametrize("group", GROUP_NAMES)
def test_msm_input_set_through_every_plan(engine, group, set_name):
    g = mc.GROUPS[group]
    a, s = mc.build_set(g, set_name, N_SET, mc.multipliers(g, N_SET))
    pts = _operands(engine, g, a)
    want = g.expected(a, s)
    sb = mc.scalars_to_bytes(s)
    for plan in PLANS:
        _apply(engine, plan)
        l0 = engine.launch_count()
        got = _msm(engine, g, sb, pts)
        launches = engine.launch_count() - l0
        ctx = (group, set_name, plan)
        assert got == want, ctx
        _check_plan(engine, g, plan, launches, ctx)


@pytest.mark.parametrize("group", GROUP_NAMES)
def test_msm_sizes(engine, group):
    """n = 1, 2, 127, 128, 129 on the automatic plan and at c = 16; n = 1 with a zero scalar and with an operand at infinity"""
    g = mc.GROUPS[group]
    rng = random.Random(f"sizes/{group}")
    for n in (1, 2, 127, 128, 129):
        a = mc.multipliers(g, n, seed=f"sizes{n}")
        s = [rng.randrange(g.r) for _ in range(n)]
        pts = _operands(engine, g, a, spot=(0, -1))
        want = g.expected(a, s)
        for plan in ({}, {"c": 16}):
            _apply(engine, plan)
            assert _msm(engine, g, mc.scalars_to_bytes(s), pts) == want, (group, n, plan)
            _check_plan(engine, g, plan, None, (group, n, plan))
    inf = g.encode(None)
    for plan in ({}, {"c": 16}):
        _apply(engine, plan)
        assert _msm(engine, g, mc.scalars_to_bytes([0]), g.gen) == inf, (group, "s = 0", plan)
        assert _msm(engine, g, mc.scalars_to_bytes([rng.randrange(1, g.r)]), bytes(g.in_bytes)) == inf, (group, "P = inf", plan)


@pytest.mark.parametrize("group", ["bls12381_g1", "bls12381_g2"])
def test_msm_affine_output(engine, group):
    """b2k_bls12381_{g1,g2}_msm_affine: the operand bytes (x || y) of the sum, all zero for infinity"""
    g = mc.GROUPS[group]
    enc = mc.AFFINE_ENCODE[group]
    name = ENTRY[group][0] + "_affine"
    for set_name in ("uniform", "equal", "plus_minus", "edges"):
        a, s = mc.build_set(g, set_name, 600, mc.multipliers(g, 600))
        pts = _operands(engine, g, a)
        acc = 0
        for x, y in zip(a, s):
            acc += x * y
        want = enc(g.mul(acc % g.r))
        sb = mc.scalars_to_bytes(s)
        for plan in ({}, {"c": 16}, {"c": 4, "L": 1}, {"variant": True}):
            _apply(engine, plan)
            assert engine.call_host(name, len(a), sb, pts, g.in_bytes) == want, (group, set_name, plan)


def _dev(data: bytes):
    import torch
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _msm_dev(engine, name, n, sb, pts, out_bytes):
    import torch
    ds, dp, do = _dev(sb), _dev(pts), torch.zeros(256, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.call_dev(name, n, ds.data_ptr(), dp.data_ptr(), do.data_ptr())
    engine.wait()
    return bytes(do[:out_bytes].cpu().numpy())


@pytest.mark.parametrize("group,dev_name", [("bls12381_g2", "b2k_bls12381_g2_msm_dev"), ("bn254_g1", "b2k_bn254_g1_msm_dev")])
def test_msm_dev_matches_host(engine, group, dev_name):
    """the device-pointer entry points give the host call's bytes"""
    g = mc.GROUPS[group]
    for set_name in ("uniform", "equal", "zeros", "small"):
        a, s = mc.build_set(g, set_name, N_SET, mc.multipliers(g, N_SET))
        pts = _operands(engine, g, a)
        sb = mc.scalars_to_bytes(s)
        want = g.expected(a, s)
        for plan in ({}, {"c": 5}, {"c": 16}, {"L": 1}, {"c": 7, "groups": 2}):
            _apply(engine, plan)
            host = _msm(engine, g, sb, pts)
            assert host == want, (group, set_name, plan)
            assert _msm_dev(engine, dev_name, len(a), sb, pts, g.out_bytes) == host, (group, set_name, plan)


def test_g1_inlined_layout_matches_default(engine):
    """b2k_set_msm_layout(1): the MSM and Point.Mul batch compiled with every field product inlined (b2k_msm_inlined.cu)
    give the bytes of the default layout on the same sets and plans"""
    import torch
    g = mc.GROUPS["bls12381_g1"]
    plans = ({}, {"c": 4}, {"c": 16}, {"L": 1}, {"c": 7, "m": 64}, {"c": 12, "reduce": (2, 1, 4)}, {"c": 5, "groups": 8},
             {"variant": True})
    for set_name in mc.SETS:
        a, s = mc.build_set(g, set_name, N_SET, mc.multipliers(g, N_SET))
        pts = _operands(engine, g, a)
        sb = mc.scalars_to_bytes(s)
        want = g.expected(a, s)
        for plan in plans:
            got = []
            for layout in (0, 1):
                _apply(engine, plan)
                engine._check(engine.lib.b2k_set_msm_layout(engine.h, layout))
                got.append(_msm_dev(engine, "b2k_bls12381_g1_msm_dev", N_SET, sb, pts, 48))
            assert got[0] == got[1] == want, (set_name, plan, got)
    # Point.Mul batch: compressed k_i P_i in both layouts
    rng = random.Random(5)
    n = 300
    ks = [0, 1, g.r - 1, g.r - 2, (g.r - 1) // 2] + [rng.randrange(g.r) for _ in range(n - 5)]
    a = mc.multipliers(g, n, seed="layout")
    pts = _operands(engine, g, a)
    pts = bytes(96) + pts[96:]                                  # one operand at infinity
    ds, dp = _dev(mc.scalars_to_bytes(ks)), _dev(pts)
    outs = []
    for layout in (0, 1):
        _reset(engine)
        engine._check(engine.lib.b2k_set_msm_layout(engine.h, layout))
        do = torch.zeros(48 * n, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        engine.call_dev("b2k_bls12381_g1_mul_batch_dev", n, ds.data_ptr(), dp.data_ptr(), do.data_ptr())
        engine.wait()
        outs.append(bytes(do.cpu().numpy()))
    assert outs[0] == outs[1]
    for i in (0, 1, 2, 3, 4, n - 1):
        assert outs[1][48 * i:48 * i + 48] == g.encode(g.mul(ks[i] * (a[i] if i else 0) % g.r)), i


@pytest.mark.parametrize("group", GROUP_NAMES)
def test_msm_refusals_and_recovery(engine, group):
    """a scalar equal to r is refused with -3; an operand off the curve with -5, and so is a coordinate >= p where the group
    refuses non-canonical encodings (bn256 reduces them, like its reference Unmarshal); the next clean call is correct"""
    g = mc.GROUPS[group]
    n = 300
    a, s = mc.build_set(g, "uniform", n, mc.multipliers(g, n, seed="refusal"))
    pts = _operands(engine, g, a)
    sb = mc.scalars_to_bytes(s)
    want = g.expected(a, s)
    assert _msm(engine, g, sb, pts) == want
    # a coordinate + p that still fits the encoding (bn256's p is 256 bits: pick an operand whose first element is small enough)
    w = g.coord_bytes
    k = next(i for i in range(n) if int.from_bytes(pts[g.in_bytes * i:g.in_bytes * i + w], "big") + g.p < 1 << (8 * w))
    noncanon = bytearray(pts)
    noncanon[g.in_bytes * k:g.in_bytes * k + w] = (int.from_bytes(pts[g.in_bytes * k:g.in_bytes * k + w], "big") + g.p).to_bytes(w, "big")
    offcurve = bytearray(pts)
    offcurve[g.in_bytes * 7 + g.in_bytes - 1] ^= 1
    bad_scalar = mc.scalars_to_bytes(s[:5] + [g.r] + s[6:])
    for plan in ({}, {"c": 16}, {"L": 1}):
        _apply(engine, plan)
        with pytest.raises(B2KError) as e:
            _msm(engine, g, bad_scalar, pts)
        assert e.value.code == -3, (group, plan)
        assert _msm(engine, g, sb, pts) == want, (group, plan, "after -3")
        with pytest.raises(B2KError) as e:
            _msm(engine, g, sb, bytes(offcurve))
        assert e.value.code == -5, (group, plan)
        assert _msm(engine, g, sb, pts) == want, (group, plan, "after -5")
        if g.canonical:
            with pytest.raises(B2KError) as e:
                _msm(engine, g, sb, bytes(noncanon))
            assert e.value.code == -5, (group, plan, "non-canonical")
        else:
            assert _msm(engine, g, sb, bytes(noncanon)) == want, (group, plan, "non-canonical reduced")
        assert _msm(engine, g, sb, pts) == want, (group, plan, "after non-canonical")


@pytest.mark.parametrize("group", GROUP_NAMES)
def test_msm_kernel_paths_run(engine, group):
    """Under torch.profiler: the all-equal set at L = 1 (a bucket cut into far more than 64 slices) runs k_msm_fixup_big,
    the grouped tail runs its range kernels, the variant runs the one-thread-per-bucket accumulate -- each with the
    oracle's bytes, in this group's instantiation of the kernels"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    g = mc.GROUPS[group]
    cv = ENTRY[group][2]
    a, s = mc.build_set(g, "equal", N_SET, mc.multipliers(g, 1))
    pts = _operands(engine, g, a)
    sb = mc.scalars_to_bytes(s)
    want = g.expected(a, s)
    plans = ({"c": 8, "L": 1}, {"c": 8, "m": 1}, {"c": 7, "groups": 2}, {"c": 8, "variant": True})
    # GLV splits every scalar in two, so each bucket of BLS12-381 G1 holds N_SET entries as well
    assert mc.largest_bucket(s, 8, g.scalar_bits) >= N_SET > 64
    names = []
    for plan in plans:
        _apply(engine, plan)
        engine.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            l0 = engine.launch_count()
            got = _msm(engine, g, sb, pts)
            launches = engine.launch_count() - l0
        assert got == want, (group, plan)
        _check_plan(engine, g, plan, launches, (group, plan))
        names.append([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])

    def ran(i, kernel):
        return any(re.search(rf"\b{kernel}<(b2k::)?{cv}[,>]", nm) for nm in names[i])
    assert ran(0, "k_msm_fixup_big") and ran(0, "k_msm_accumulate_slices"), (group, names[0])
    assert ran(1, "k_msm_reduce_chunks"), (group, names[1])
    assert ran(2, "k_msm_accumulate_slices_range") and ran(2, "k_msm_fixup_range") and ran(2, "k_msm_reduce_chunks_range"), (group, names[2])
    assert ran(3, "k_msm_accumulate") and not ran(3, "k_msm_fixup_big"), (group, names[3])
