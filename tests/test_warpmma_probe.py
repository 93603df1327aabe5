"""The SM warp-MMA probe (cro_probe_warpmma and its helper form) on one H100, against oracle/warpmma.py's answers,
folds and substituted rows.

Faults come only from the probe's software injections (test_inject_*, test_addr_*); nothing here repeats a call to
catch a real one.  The fragment-address substitutions pin the fragment mapping: each must change exactly the row the
restatement predicts, on that SM and leg only, to the predicted values."""
import json

import numpy as np
import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
DEFAULT_ITERATIONS = 128
EXP_MASK = [1 << 30] * 4 + [1 << 14] * 2   # an f32 exponent bit / an int32 high bit / an f16 exponent bit / a word bit
ROW, COL = 77, 45
LEG_IDS = ["s8", "f16", "bf16", "tf32", "f16acc", "move"]
# (leg, row, k-step) of each substitution: the first three columns on the first covered SM, the rest on the last
ADDR_CASES = [(0, 93, 3), (0, 6, 15), (1, 93, 0), (1, 6, 31), (2, 93, 17), (2, 6, 30), (3, 93, 1), (3, 6, 26),
              (4, 93, 8), (4, 6, 21)]

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_warpmma(0)


def answers(seed):
    import warpmma
    return {a: warpmma.answer(a, seed) for a in range(5)}


def check_clean(cro, ctx, r, sms, faults, iterations):
    import warpmma
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.COMPUTE_NONE and not faults, [(f.leg, f.row, f.col) for f in faults[:8]]
    assert r.sm_count == n and r.legs == cro.WARPMMA_ALL_LEGS and r.bad_sms == 0 and r.host_ref_ns > 0
    want = answers(r.seed)
    for leg in range(cro.WARPMMA_LEGS):
        L = r.leg[leg]
        assert L.iterations == iterations
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered, L.unpublished)
        assert L.mismatches == 0 and L.fold_mismatches == 0 and L.recorded == 0 and L.failed_sms == 0, leg
        assert L.fold == L.expect_fold == warpmma.cta_fold(leg, want[warpmma.LEG_ANSWER[leg]], iterations), leg
        assert L.ns > 0 and L.timer_ns > 0 and L.ops == warpmma.ops(leg) * iterations * L.ctas
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    for s in sms:
        for leg in range(cro.WARPMMA_LEGS):
            assert s.leg[leg].ctas >= 1 and s.leg[leg].ns > 0 and s.leg[leg].cycles > 0 and s.leg[leg].mark == 0


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, DEFAULT_ITERATIONS)
    ann = json.loads(cro.emit_warpmma_annotations_json(r))
    n = ctx.own_devices()[0].sm_count
    assert ann["cohdi.io/probe-warpmma-verdict"] == "ok" and ann["cohdi.io/probe-warpmma-sms"] == "%d/%d" % (n, n)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 55) + r.call * STRIDE) & MASK


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_warpmma(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


def test_second_call_uses_a_new_seed(ctx):
    a, _, _ = ctx.probe_warpmma(0, iterations=1)
    b, _, _ = ctx.probe_warpmma(0, iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + STRIDE) & MASK and a.status == b.status == 0


def check_one_sm(cro, r, sms, faults, leg, smid, mark):
    import warpmma
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_SM
    assert r.bad_sms == 1 and r.bad_sm[0] == smid
    entry = [s for s in sms if s.smid == smid]
    assert len(entry) == 1 and entry[0].leg[leg].ctas >= 1
    for lg in range(cro.WARPMMA_LEGS):
        L = r.leg[lg]
        if lg != leg:
            assert L.mismatches == L.fold_mismatches == L.failed_sms == 0
            continue
        assert L.failed_sms == 1 and entry[0].leg[leg].mark == mark
        for s in sms:
            if s.smid != smid:
                assert s.leg[leg].mark == 0 and s.leg[leg].mismatches == 0 and s.leg[leg].fold_mismatches == 0
    assert all(f.leg == leg and f.smid == smid for f in faults)
    ann = json.loads(cro.emit_warpmma_annotations_json(r))
    assert ann["cohdi.io/probe-warpmma-verdict"] == "sm" and ann["cohdi.io/probe-warpmma-bad-sms"] == str(smid)
    assert ann["cohdi.io/probe-warpmma-failed-legs"] == warpmma.LEG_NAMES[leg]
    return entry[0].leg[leg].ctas


@pytest.mark.parametrize("leg", range(6), ids=LEG_IDS)
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_accumulator_injection_names_the_sm_and_the_leg(cro, ctx, clean, leg, where, when):
    import warpmma
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    mask = EXP_MASK[leg]
    r, sms, faults = ctx.probe_warpmma(0, iterations=3, inject=(leg, smid, 2 if when == "last" else 1, ROW, COL, mask))
    ctas = check_one_sm(cro, r, sms, faults, leg, smid, cro.COMPUTE_PERSISTENT if when == "last" else cro.COMPUTE_INTERMITTENT)
    L = r.leg[leg]
    assert L.fold_mismatches == ctas
    if when == "last":
        v = int(answers(r.seed)[warpmma.LEG_ANSWER[leg]][ROW, COL])
        assert L.mismatches == ctas and L.recorded == ctas
        assert [(f.row, f.col, f.expected, f.actual_bits) for f in faults] == \
            [(ROW, COL, v, warpmma.value_bits(leg, v) ^ mask)] * ctas
    else:
        assert L.mismatches == 0 and not faults


@pytest.mark.parametrize("case", range(len(ADDR_CASES)), ids=["%s-r%d-k%d" % (LEG_IDS[c[0]], c[1], c[2]) for c in ADDR_CASES])
def test_fragment_address_substitution_gives_the_predicted_row(cro, ctx, clean, case):
    """In the last iteration, the lane that supplies row R's address for one k-step's A ldmatrix passes row R ^ 1:
    only row R changes, in exactly the columns the restatement predicts, each to its predicted value.  This pins which
    lane supplies which row and K half, and shows an operand-delivery fault is caught and located."""
    import warpmma
    leg, row, kstep = ADDR_CASES[case]
    smid = clean[1][0].smid if row == 93 else clean[1][-1].smid
    r, sms, faults = ctx.probe_warpmma(0, iterations=3, addr=(leg, smid, 2, row, kstep), cap=4096)
    good = answers(r.seed)[warpmma.LEG_ANSWER[leg]]
    bad = warpmma.substituted_row(leg, r.seed, row, kstep)
    cols = [int(c) for c in np.nonzero(bad != good[row])[0]]
    assert cols, "the substitution changes the row"
    ctas = check_one_sm(cro, r, sms, faults, leg, smid, cro.COMPUTE_PERSISTENT)
    L = r.leg[leg]
    assert L.mismatches == len(cols) * ctas and L.recorded == len(cols) * ctas
    got = sorted((f.row, f.col, f.expected, f.actual_bits) for f in faults)
    want = sorted([(row, c, int(good[row, c]), warpmma.value_bits(leg, int(bad[c]))) for c in cols] * ctas)
    assert got == want


def test_a_middle_iteration_substitution_is_intermittent(cro, ctx, clean):
    smid = clean[1][0].smid
    r, sms, faults = ctx.probe_warpmma(0, iterations=3, addr=(cro.WARPMMA_LEG_F16, smid, 1, 10, 21))
    check_one_sm(cro, r, sms, faults, cro.WARPMMA_LEG_F16, smid, cro.COMPUTE_INTERMITTENT)
    assert r.leg[cro.WARPMMA_LEG_F16].mismatches == 0 and not faults


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    for kw in (dict(inject=(cro.WARPMMA_LEG_MOVE, -1, 2, ROW, COL, 1)), dict(addr=(cro.WARPMMA_LEG_S8, -1, 2, ROW, 3))):
        r, sms, _ = ctx.probe_warpmma(0, iterations=3, **kw)
        leg = (kw.get("inject") or kw.get("addr"))[0]
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_ALL
        L = r.leg[leg]
        assert L.failed_sms == L.sms_covered == len(sms)
        assert json.loads(cro.emit_warpmma_annotations_json(r))["cohdi.io/probe-warpmma-verdict"] == "all"


def test_records_stop_at_the_cap_and_counts_stay_exact(cro, ctx, clean):
    import warpmma
    leg, smid = cro.WARPMMA_LEG_TF32, clean[1][0].smid
    r, sms, faults = ctx.probe_warpmma(0, iterations=2, legs=1 << leg, inject=(leg, smid, 1, -1, -1, EXP_MASK[leg]),
                                       cap=cro.WARPMMA_RECORDS + 16)
    L = r.leg[leg]
    ctas = [s for s in sms if s.smid == smid][0].leg[leg].ctas
    assert L.mismatches == warpmma.M * warpmma.N * ctas and L.recorded == cro.WARPMMA_RECORDS
    assert len(faults) == cro.WARPMMA_RECORDS
    tile = answers(r.seed)[warpmma.LEG_ANSWER[leg]]
    for f in faults[:64]:
        assert f.smid == smid and f.expected == tile[f.row, f.col]
        assert f.actual_bits == warpmma.value_bits(leg, int(tile[f.row, f.col])) ^ EXP_MASK[leg]


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_warpmma(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_warpmma(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(legs=0x40), dict(iterations=cro.WARPMMA_MAX_ITERATIONS + 1), dict(max_rounds=cro.WARPMMA_MAX_ROUNDS + 1),
             dict(inject=(0, 256, 0, 0, 0, 1)), dict(inject=(6, 0, 0, 0, 0, 1)), dict(inject=(2, 0, 3, 0, 0, 1), iterations=3),
             dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)), dict(inject=(2, 0, 0, 0, 0, 1 << 32)),
             dict(inject=(4, 0, 0, 0, 0, 1 << 16)), dict(inject=(5, 0, 0, 0, 0, 1 << 16)),
             dict(addr=(5, 0, 0, 0, 0)), dict(addr=(0, 256, 0, 0, 0)), dict(addr=(0, 0, 3, 0, 0), iterations=3),
             dict(addr=(0, 0, 0, 128, 0)), dict(addr=(0, 0, 0, 0, 16)), dict(addr=(3, 0, 0, 0, 32)),
             dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_warpmma(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw


# ---- the helper form ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def uuid(ctx):
    return ctx.own_devices()[0].gpu_uuid.decode()


def test_helper_clean_call(cro, ctx, uuid):
    r, sms, faults, ns = cro.probe_warpmma_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert ns > 0
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.call == 0 and r.seed != (dev + (1 << 55)) & MASK         # the helper's own seed base, not the context's


@pytest.mark.parametrize("kind", ["inject", "addr"])
def test_helper_names_what_the_in_process_form_names(cro, ctx, clean, uuid, kind):
    smid = clean[1][-1].smid
    kw = dict(inject=(cro.WARPMMA_LEG_BF16, smid, 2, ROW, COL, 1)) if kind == "inject" else \
        dict(addr=(cro.WARPMMA_LEG_BF16, smid, 2, ROW, 5))
    a = ctx.probe_warpmma(0, iterations=3, **kw)
    b = cro.probe_warpmma_uuid(ctx, uuid, iterations=3, **kw)[:3]
    for r, sms, faults in (a, b):
        check_one_sm(cro, r, sms, faults, cro.WARPMMA_LEG_BF16, smid, cro.COMPUTE_PERSISTENT)
    # the two forms have their own seeds: a substitution's columns follow the seed, its row does not
    assert {f.row for f in a[2]} == {f.row for f in b[2]} == {ROW}
    if kind == "inject":
        assert [(f.row, f.col) for f in a[2]] == [(f.row, f.col) for f in b[2]]


def test_helper_refuses_bad_options_before_any_launch(cro, ctx, uuid):
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_warpmma_uuid(ctx, uuid, addr=(0, 0, 0, 0, 16))
    assert e.value.code == cro.ERR_INVALID_ARG
