"""The SM compute probe (cro_probe_compute) on one H100, against the C oracle's answers and oracle/compute.py's folds.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import json
import struct

import numpy as np
import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
INT_MASK = 1 << 4              # integer legs: v ^ 16 always differs from v
FLOAT_MASK = 1 << 30           # float legs: flips the exponent's top bit, so every value (0 included) changes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def co(_built):
    import compute
    return compute.CComputeOracle()


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_compute(0)


def is_float(cro, leg):
    return leg in (cro.COMPUTE_LEG_BF16, cro.COMPUTE_LEG_E4M3, cro.COMPUTE_LEG_FFMA)


def cvt_rni(bits):
    """cvt.rni.s32.f32 of a float's bit pattern: round half to even, saturate, NaN -> 0."""
    f = struct.unpack("<f", struct.pack("<I", bits & 0xFFFFFFFF))[0]
    if f != f:
        return 0
    if f >= 2.0 ** 31:
        return 2 ** 31 - 1
    if f < -2.0 ** 31:
        return -2 ** 31
    return int(round(f))


def injected(cro, leg, v, mask):
    if is_float(cro, leg):
        return cvt_rni(struct.unpack("<I", struct.pack("<f", float(v)))[0] ^ mask)
    return v ^ mask


def tiles(co, seed):
    return {0: co.answer(0, seed), 1: co.answer(1, seed)}


def check_clean(cro, ctx, co, r, sms, faults, iterations, alu_iterations):
    import compute
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.COMPUTE_NONE and not faults
    assert r.sm_count == n and r.legs == cro.COMPUTE_ALL_LEGS and r.bad_sms == 0 and r.host_ref_ns > 0
    want = tiles(co, r.seed)
    for leg in range(cro.COMPUTE_LEGS):
        L = r.leg[leg]
        it = iterations if leg < 3 else alu_iterations
        assert L.iterations == it
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered, L.unpublished)
        assert L.mismatches == 0 and L.fold_mismatches == 0 and L.recorded == 0 and L.failed_sms == 0
        assert L.fold == L.expect_fold == compute.cta_fold(want[compute.LEG_ANSWER[leg]], it), leg
        assert L.ns > 0 and L.timer_ns > 0 and L.ops == 2 * 128 * 256 * 256 * it * L.ctas
    # the three float legs computed the same answer: the same fold per iteration
    f = [r.leg[leg].fold for leg in (cro.COMPUTE_LEG_BF16, cro.COMPUTE_LEG_E4M3)]
    assert f[0] == f[1] == compute.cta_fold(want[1], iterations)
    assert r.leg[cro.COMPUTE_LEG_FFMA].fold == compute.cta_fold(want[1], alu_iterations)
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    for s in sms:
        for leg in range(cro.COMPUTE_LEGS):
            assert s.leg[leg].ctas >= 1 and s.leg[leg].ns > 0 and s.leg[leg].cycles > 0 and s.leg[leg].mark == 0


def test_clean_default_call(cro, ctx, co, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, co, r, sms, faults, r.leg[0].iterations, r.leg[cro.COMPUTE_LEG_FFMA].iterations)
    ann = json.loads(cro.emit_compute_annotations_json(r))
    n = ctx.own_devices()[0].sm_count
    assert ann["cohdi.io/probe-compute-verdict"] == "ok" and ann["cohdi.io/probe-compute-sms"] == "%d/%d" % (n, n)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 61) + r.call * STRIDE) & MASK


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, co, iterations):
    r, sms, faults = ctx.probe_compute(0, iterations=iterations, alu_iterations=2)
    check_clean(cro, ctx, co, r, sms, faults, iterations, 2)


def test_second_call_uses_a_new_seed(ctx):
    a, _, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    b, _, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + STRIDE) & MASK and a.status == b.status == 0


ROW, COL = 77, 133


@pytest.mark.parametrize("leg", range(5), ids=["s8", "bf16", "e4m3", "ffma", "imad"])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_injection_names_the_sm_and_the_leg(cro, ctx, co, clean, leg, where, when):
    import compute
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    iteration = 2 if when == "last" else 1
    mask = FLOAT_MASK if is_float(cro, leg) else INT_MASK
    r, sms, faults = ctx.probe_compute(0, iterations=3, alu_iterations=3,
                                       inject=(leg, smid, iteration, ROW, COL, mask))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_SM
    assert r.bad_sms == 1 and r.bad_sm[0] == smid
    entry = [s for s in sms if s.smid == smid]
    assert len(entry) == 1
    ctas = entry[0].leg[leg].ctas
    assert ctas >= 1
    for lg in range(cro.COMPUTE_LEGS):
        L = r.leg[lg]
        if lg != leg:
            assert L.mismatches == L.fold_mismatches == L.failed_sms == 0
            continue
        assert L.failed_sms == 1 and L.fold_mismatches == ctas
        assert entry[0].leg[leg].fold_mismatches == ctas
        for s in sms:
            if s.smid != smid:
                assert s.leg[leg].mark == 0 and s.leg[leg].mismatches == 0 and s.leg[leg].fold_mismatches == 0
        if when == "last":
            v = int(tiles(co, r.seed)[compute.LEG_ANSWER[leg]][ROW, COL])
            assert L.mismatches == ctas and L.recorded == ctas
            assert entry[0].leg[leg].mark == cro.COMPUTE_PERSISTENT
            assert [(f.leg, f.smid, f.row, f.col, f.expected, f.actual) for f in faults] == \
                [(leg, smid, ROW, COL, v, injected(cro, leg, v, mask))] * ctas
        else:
            assert L.mismatches == 0 and not faults
            assert entry[0].leg[leg].mark == cro.COMPUTE_INTERMITTENT
    ann = json.loads(cro.emit_compute_annotations_json(r))
    assert ann["cohdi.io/probe-compute-verdict"] == "sm"
    assert ann["cohdi.io/probe-compute-bad-sms"] == str(smid)
    assert ann["cohdi.io/probe-compute-failed-legs"] == compute.LEG_NAMES[leg]


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    r, sms, _ = ctx.probe_compute(0, iterations=3, alu_iterations=3,
                                  inject=(cro.COMPUTE_LEG_BF16, -1, 2, ROW, COL, FLOAT_MASK))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_ALL
    L = r.leg[cro.COMPUTE_LEG_BF16]
    assert L.failed_sms == L.sms_covered == len(sms) and L.mismatches == L.ctas
    assert json.loads(cro.emit_compute_annotations_json(r))["cohdi.io/probe-compute-verdict"] == "all"


@pytest.mark.parametrize("leg", [0, 2], ids=["s8", "e4m3"])
def test_injection_into_every_element_counts_exactly(cro, ctx, co, leg):
    import compute
    mask = FLOAT_MASK if is_float(cro, leg) else INT_MASK
    r, sms, faults = ctx.probe_compute(0, iterations=2, legs=1 << leg, inject=(leg, -1, 1, -1, -1, mask),
                                       cap=cro.COMPUTE_RECORDS + 16)
    L = r.leg[leg]
    tile = tiles(co, r.seed)[compute.LEG_ANSWER[leg]]
    bad = np.vectorize(lambda v: injected(cro, leg, int(v), mask))(tile).astype(np.int64)
    assert (bad != tile).all()
    changed = int((compute.thread_folds(bad) != compute.thread_folds(tile)).sum())
    assert r.verdict == cro.COMPUTE_ALL and L.failed_sms == L.sms_covered
    assert L.mismatches == 128 * 256 * L.ctas and L.fold_mismatches == changed * L.ctas
    assert L.recorded == cro.COMPUTE_RECORDS and len(faults) == cro.COMPUTE_RECORDS
    for f in faults[:64]:
        assert f.leg == leg and f.expected == tile[f.row, f.col] and f.actual == bad[f.row, f.col]


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(legs=0x20), dict(iterations=cro.COMPUTE_MAX_ITERATIONS + 1),
             dict(alu_iterations=cro.COMPUTE_MAX_ALU_ITERATIONS + 1), dict(max_rounds=cro.COMPUTE_MAX_ROUNDS + 1),
             dict(inject=(0, 256, 0, 0, 0, 1)), dict(inject=(5, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 3, 0, 0, 1), iterations=3),
             dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)),
             dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_compute(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
