"""The SM precision probe (cro_probe_precision and its helper form) on one H100, against oracle/precision.py's answers
and folds.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import json

import numpy as np
import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
# the top exponent bit of each leg's element: every value, 0 included, changes
EXP_MASK = [1 << 62, 1 << 62, 1 << 30, 1 << 30, 1 << 14, 1 << 30, 1 << 14]
ROW, COL = 77, 45                 # inside every leg's tile (the F64 legs have 64 columns)
LEG_IDS = ["f64", "dfma", "tf32", "f16", "f16acc", "e5m2", "hfma2"]

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_precision(0)


def answers(seed):
    import precision
    return {a: precision.answer(a, seed) for a in range(4)}


def canon(leg, bits):
    import precision
    return 0 if bits == 1 << (precision.LEG_BITS[leg] - 1) else bits


def expect_bits(leg, v):
    import precision
    return int(precision.encode(leg, np.array([v], dtype=np.int64))[0])


def check_clean(cro, ctx, r, sms, faults, iterations, alu_iterations):
    import precision
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.COMPUTE_NONE and not faults, [f.leg for f in faults[:8]]
    assert r.sm_count == n and r.legs == cro.PRECISION_ALL_LEGS and r.bad_sms == 0 and r.host_ref_ns > 0
    want = answers(r.seed)
    for leg in range(cro.PRECISION_LEGS):
        L = r.leg[leg]
        it = alu_iterations if leg in (cro.PRECISION_LEG_DFMA, cro.PRECISION_LEG_HFMA2) else iterations
        assert L.iterations == it
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered, L.unpublished)
        assert L.mismatches == 0 and L.fold_mismatches == 0 and L.recorded == 0 and L.failed_sms == 0, leg
        assert L.fold == L.expect_fold == precision.cta_fold(leg, want[precision.LEG_ANSWER[leg]], it), leg
        m, nn, k = precision.SHAPE[precision.LEG_ANSWER[leg]]
        assert L.ns > 0 and L.timer_ns > 0 and L.ops == 2 * m * nn * k * it * L.ctas
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    for s in sms:
        for leg in range(cro.PRECISION_LEGS):
            assert s.leg[leg].ctas >= 1 and s.leg[leg].ns > 0 and s.leg[leg].cycles > 0 and s.leg[leg].mark == 0


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, r.leg[0].iterations, r.leg[cro.PRECISION_LEG_DFMA].iterations)
    ann = json.loads(cro.emit_precision_annotations_json(r))
    n = ctx.own_devices()[0].sm_count
    assert ann["cohdi.io/probe-precision-verdict"] == "ok" and ann["cohdi.io/probe-precision-sms"] == "%d/%d" % (n, n)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 58) + r.call * STRIDE) & MASK


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_precision(0, iterations=iterations, alu_iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations, iterations)


def test_second_call_uses_a_new_seed(ctx):
    a, _, _ = ctx.probe_precision(0, iterations=1, alu_iterations=1)
    b, _, _ = ctx.probe_precision(0, iterations=1, alu_iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + STRIDE) & MASK and a.status == b.status == 0


def check_one_sm(cro, r, sms, faults, leg, smid, when, mask):
    import precision
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_SM
    assert r.bad_sms == 1 and r.bad_sm[0] == smid
    entry = [s for s in sms if s.smid == smid]
    assert len(entry) == 1
    ctas = entry[0].leg[leg].ctas
    assert ctas >= 1
    for lg in range(cro.PRECISION_LEGS):
        L = r.leg[lg]
        if lg != leg:
            assert L.mismatches == L.fold_mismatches == L.failed_sms == 0
            continue
        assert L.failed_sms == 1 and L.fold_mismatches == ctas and entry[0].leg[leg].fold_mismatches == ctas
        for s in sms:
            if s.smid != smid:
                assert s.leg[leg].mark == 0 and s.leg[leg].mismatches == 0 and s.leg[leg].fold_mismatches == 0
        if when == "last":
            v = int(answers(r.seed)[precision.LEG_ANSWER[leg]][ROW, COL])
            assert L.mismatches == ctas and L.recorded == ctas
            assert entry[0].leg[leg].mark == cro.COMPUTE_PERSISTENT
            assert [(f.leg, f.smid, f.row, f.col, f.expected) for f in faults] == [(leg, smid, ROW, COL, v)] * ctas
            for f in faults:
                assert canon(leg, f.actual_bits ^ mask) == expect_bits(leg, v) and f.actual_bits >> precision.LEG_BITS[leg] == 0
        else:
            assert L.mismatches == 0 and not faults
            assert entry[0].leg[leg].mark == cro.COMPUTE_INTERMITTENT
    ann = json.loads(cro.emit_precision_annotations_json(r))
    assert ann["cohdi.io/probe-precision-verdict"] == "sm"
    assert ann["cohdi.io/probe-precision-bad-sms"] == str(smid)
    assert ann["cohdi.io/probe-precision-failed-legs"] == precision.LEG_NAMES[leg]


@pytest.mark.parametrize("leg", range(7), ids=LEG_IDS)
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_injection_names_the_sm_and_the_leg(cro, ctx, clean, leg, where, when):
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    r, sms, faults = ctx.probe_precision(0, iterations=3, alu_iterations=3,
                                         inject=(leg, smid, 2 if when == "last" else 1, ROW, COL, EXP_MASK[leg]))
    check_one_sm(cro, r, sms, faults, leg, smid, when, EXP_MASK[leg])


@pytest.mark.parametrize("leg", range(7), ids=LEG_IDS)
def test_the_lowest_mantissa_bit_is_caught(cro, ctx, clean, leg):
    """A flip worth far less than 0.5: the compute probe's rounding compare would pass it."""
    smid = clean[1][0].smid
    r, sms, faults = ctx.probe_precision(0, iterations=2, alu_iterations=2, inject=(leg, smid, 1, ROW, COL, 1))
    check_one_sm(cro, r, sms, faults, leg, smid, "last", 1)


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    leg = cro.PRECISION_LEG_F16
    r, sms, _ = ctx.probe_precision(0, iterations=3, alu_iterations=3, inject=(leg, -1, 2, ROW, COL, 1))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_ALL
    L = r.leg[leg]
    assert L.failed_sms == L.sms_covered == len(sms) and L.mismatches == L.ctas
    assert json.loads(cro.emit_precision_annotations_json(r))["cohdi.io/probe-precision-verdict"] == "all"


def thread_folds(leg, tile):
    """Per thread: sum over its values of canon(bits) * (2e + 1) mod 2^64 (include/croprobe.h's fragment)."""
    import precision
    f64 = precision.LEG_BITS[leg] == 64
    t = np.arange(256)[:, None]
    j = np.arange(32 if f64 else 128)[None, :]
    r0 = 16 * (t // 32) + (t % 32) // 4 if f64 else 64 * (t // 128) + 16 * ((t // 32) % 4) + (t % 32) // 4
    rows, cols = r0 + 8 * ((j // 2) % 2), 8 * (j // 4) + 2 * (t % 4) + j % 2
    n = tile.shape[1]
    v = tile[rows, cols]
    w = (2 * (rows * n + cols) + 1).astype(np.uint64)
    with np.errstate(over="ignore"):
        return (v * w).sum(axis=1, dtype=np.uint64)


@pytest.mark.parametrize("leg", [0, 4], ids=["f64", "f16acc"])
def test_injection_into_every_element_counts_exactly(cro, ctx, leg):
    import precision
    mask = EXP_MASK[leg]
    r, sms, faults = ctx.probe_precision(0, iterations=2, alu_iterations=2, legs=1 << leg, inject=(leg, -1, 1, -1, -1, mask),
                                         cap=cro.PRECISION_RECORDS + 16)
    L = r.leg[leg]
    tile = answers(r.seed)[precision.LEG_ANSWER[leg]]
    good = precision.encode(leg, tile)
    bad = good ^ np.uint64(mask)
    changed = int((thread_folds(leg, bad) != thread_folds(leg, good)).sum())
    assert r.verdict == cro.COMPUTE_ALL and L.failed_sms == L.sms_covered
    assert L.mismatches == tile.size * L.ctas and L.fold_mismatches == changed * L.ctas
    assert L.recorded == cro.PRECISION_RECORDS and len(faults) == cro.PRECISION_RECORDS
    for f in faults[:64]:
        assert f.leg == leg and f.expected == tile[f.row, f.col] and canon(leg, f.actual_bits ^ mask) == int(good[f.row, f.col])


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_precision(0, iterations=1, alu_iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_precision(0, iterations=1, alu_iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(legs=0x80), dict(iterations=cro.PRECISION_MAX_ITERATIONS + 1),
             dict(alu_iterations=cro.PRECISION_MAX_ALU_ITERATIONS + 1), dict(max_rounds=cro.PRECISION_MAX_ROUNDS + 1),
             dict(inject=(0, 256, 0, 0, 0, 1)), dict(inject=(7, 0, 0, 0, 0, 1)), dict(inject=(2, 0, 3, 0, 0, 1), iterations=3),
             dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 64, 1)), dict(inject=(2, 0, 0, 0, 256, 1)),
             dict(inject=(2, 0, 0, 0, 0, 1 << 32)), dict(inject=(6, 0, 0, 0, 0, 1 << 16)),
             dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_precision(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw


# ---- the helper form ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def uuid(ctx):
    return ctx.own_devices()[0].gpu_uuid.decode()


def test_helper_clean_call(cro, ctx, uuid):
    r, sms, faults, ns = cro.probe_precision_uuid(ctx, uuid, iterations=2, alu_iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2, 2)
    assert ns > 0
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.call == 0 and r.seed != (dev + (1 << 58)) & MASK         # the helper's own seed base, not the context's


@pytest.mark.parametrize("leg", [0, 4, 6], ids=["f64", "f16acc", "hfma2"])
def test_helper_injection_names_what_the_in_process_form_names(cro, ctx, clean, uuid, leg):
    smid = clean[1][-1].smid
    inj = (leg, smid, 2, ROW, COL, 1)
    a = ctx.probe_precision(0, iterations=3, alu_iterations=3, inject=inj)
    b = cro.probe_precision_uuid(ctx, uuid, iterations=3, alu_iterations=3, inject=inj)[:3]
    for r, sms, faults in (a, b):
        check_one_sm(cro, r, sms, faults, leg, smid, "last", 1)
    assert [(f.leg, f.smid, f.row, f.col) for f in a[2]] == [(f.leg, f.smid, f.row, f.col) for f in b[2]]


def test_helper_refuses_bad_options_before_any_launch(cro, ctx, uuid):
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_precision_uuid(ctx, uuid, inject=(4, 0, 0, 0, 0, 1 << 16))
    assert e.value.code == cro.ERR_INVALID_ARG
