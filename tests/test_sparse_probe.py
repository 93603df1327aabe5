"""The SM sparse probe (cro_probe_sparse and its helper form) on one H100, against oracle/sparse.py's answers, folds and
substituted answers.

Faults come only from the probe's software injections (test_inject_*, test_meta_*); nothing here repeats a call to
catch a real one.  The metadata substitutions pin the layout of the sparsity metadata: each must change exactly the
answer the restatement predicts for that row, on that SM and leg only."""
import json

import numpy as np
import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
EXP_MASK = 1 << 30                # an f32 exponent bit / an int32 high bit: every value, 0 included, changes
ROW, COL = 77, 45
LEG_IDS = ["s8", "e4m3", "e5m2", "bf16", "f16", "tf32"]
# groups of one row per instruction: 16 for the 8-bit forms, 8 otherwise; (leg, group) of each substitution, the
# 16- and 32-bit forms once in an even instruction (selector 0) and once in an odd one (selector 1)
META_CASES = [(0, 37), (1, 100), (2, 5), (3, 18), (3, 27), (4, 0), (4, 63), (5, 42), (5, 20)]
META_IDS = ["s8", "e4m3", "e5m2", "bf16-sel0", "bf16-sel1", "f16-sel0", "f16-sel1", "tf32-sel1", "tf32-sel0"]

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_sparse(0)


def answers(seed):
    import sparse
    return {a: sparse.answer(a, seed) for a in range(4)}


def check_clean(cro, ctx, r, sms, faults, iterations):
    import sparse
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.COMPUTE_NONE and not faults, [(f.leg, f.row, f.col) for f in faults[:8]]
    assert r.sm_count == n and r.legs == cro.SPARSE_ALL_LEGS and r.bad_sms == 0 and r.host_ref_ns > 0
    want = answers(r.seed)
    for leg in range(cro.SPARSE_LEGS):
        L = r.leg[leg]
        assert L.iterations == iterations
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered, L.unpublished)
        assert L.mismatches == 0 and L.fold_mismatches == 0 and L.recorded == 0 and L.failed_sms == 0, leg
        assert L.fold == L.expect_fold == sparse.cta_fold(leg, want[sparse.LEG_ANSWER[leg]], iterations), leg
        assert L.ns > 0 and L.timer_ns > 0 and L.ops == 2 * sparse.M * sparse.N * sparse.K[sparse.LEG_ANSWER[leg]] * iterations * L.ctas
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    for s in sms:
        for leg in range(cro.SPARSE_LEGS):
            assert s.leg[leg].ctas >= 1 and s.leg[leg].ns > 0 and s.leg[leg].cycles > 0 and s.leg[leg].mark == 0


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, 256)
    ann = json.loads(cro.emit_sparse_annotations_json(r))
    n = ctx.own_devices()[0].sm_count
    assert ann["cohdi.io/probe-sparse-verdict"] == "ok" and ann["cohdi.io/probe-sparse-sms"] == "%d/%d" % (n, n)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 57) + r.call * STRIDE) & MASK


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_sparse(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


def test_second_call_uses_a_new_seed(ctx):
    a, _, _ = ctx.probe_sparse(0, iterations=1)
    b, _, _ = ctx.probe_sparse(0, iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + STRIDE) & MASK and a.status == b.status == 0


def check_one_sm(cro, r, sms, faults, leg, smid, mark):
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_SM
    assert r.bad_sms == 1 and r.bad_sm[0] == smid
    entry = [s for s in sms if s.smid == smid]
    assert len(entry) == 1 and entry[0].leg[leg].ctas >= 1
    for lg in range(cro.SPARSE_LEGS):
        L = r.leg[lg]
        if lg != leg:
            assert L.mismatches == L.fold_mismatches == L.failed_sms == 0
            continue
        assert L.failed_sms == 1 and entry[0].leg[leg].mark == mark
        for s in sms:
            if s.smid != smid:
                assert s.leg[leg].mark == 0 and s.leg[leg].mismatches == 0 and s.leg[leg].fold_mismatches == 0
    assert all(f.leg == leg and f.smid == smid for f in faults)
    import sparse
    ann = json.loads(cro.emit_sparse_annotations_json(r))
    assert ann["cohdi.io/probe-sparse-verdict"] == "sm" and ann["cohdi.io/probe-sparse-bad-sms"] == str(smid)
    assert ann["cohdi.io/probe-sparse-failed-legs"] == sparse.LEG_NAMES[leg]
    return entry[0].leg[leg].ctas


@pytest.mark.parametrize("leg", range(6), ids=LEG_IDS)
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_accumulator_injection_names_the_sm_and_the_leg(cro, ctx, clean, leg, where, when):
    import sparse
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    r, sms, faults = ctx.probe_sparse(0, iterations=3, inject=(leg, smid, 2 if when == "last" else 1, ROW, COL, EXP_MASK))
    ctas = check_one_sm(cro, r, sms, faults, leg, smid, cro.COMPUTE_PERSISTENT if when == "last" else cro.COMPUTE_INTERMITTENT)
    L = r.leg[leg]
    assert L.fold_mismatches == ctas
    if when == "last":
        v = int(answers(r.seed)[sparse.LEG_ANSWER[leg]][ROW, COL])
        assert L.mismatches == ctas and L.recorded == ctas
        assert [(f.row, f.col, f.expected, f.actual_bits) for f in faults] == \
            [(ROW, COL, v, sparse.value_bits(leg, v) ^ EXP_MASK)] * ctas
    else:
        assert L.mismatches == 0 and not faults


@pytest.mark.parametrize("leg,group", META_CASES, ids=META_IDS)
@pytest.mark.parametrize("where", ["first", "last"])
def test_metadata_substitution_gives_the_predicted_wrong_row(cro, ctx, clean, leg, group, where):
    """The next legal pair for one group of one row, in the last iteration: only that row's elements change, each to
    the restatement's answer with that pair, so the metadata layout is what the kernels assume."""
    import sparse
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    row = 93 if where == "first" else 6
    r, sms, faults = ctx.probe_sparse(0, iterations=3, meta=(leg, smid, 2, row, group), cap=4096)
    a = sparse.LEG_ANSWER[leg]
    good, bad = answers(r.seed)[a], sparse.substituted(a, r.seed, row, group)
    cols = [int(c) for c in np.nonzero(bad[row] != good[row])[0]]
    assert cols, "the substitution changes the row"
    ctas = check_one_sm(cro, r, sms, faults, leg, smid, cro.COMPUTE_PERSISTENT)
    L = r.leg[leg]
    assert L.mismatches == len(cols) * ctas and L.recorded == len(cols) * ctas
    got = sorted((f.row, f.col, f.expected, f.actual_bits) for f in faults)
    want = sorted([(row, c, int(good[row, c]), sparse.value_bits(leg, int(bad[row, c]))) for c in cols] * ctas)
    assert got == want


def test_a_middle_iteration_substitution_is_intermittent(cro, ctx, clean):
    smid = clean[1][0].smid
    r, sms, faults = ctx.probe_sparse(0, iterations=3, meta=(cro.SPARSE_LEG_F16, smid, 1, 10, 21))
    check_one_sm(cro, r, sms, faults, cro.SPARSE_LEG_F16, smid, cro.COMPUTE_INTERMITTENT)
    assert r.leg[cro.SPARSE_LEG_F16].mismatches == 0 and not faults


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    for kw in (dict(inject=(cro.SPARSE_LEG_S8, -1, 2, ROW, COL, 1)), dict(meta=(cro.SPARSE_LEG_E5M2, -1, 2, ROW, 3))):
        r, sms, _ = ctx.probe_sparse(0, iterations=3, **kw)
        leg = (kw.get("inject") or kw.get("meta"))[0]
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_ALL
        L = r.leg[leg]
        assert L.failed_sms == L.sms_covered == len(sms)
        assert json.loads(cro.emit_sparse_annotations_json(r))["cohdi.io/probe-sparse-verdict"] == "all"


def test_records_stop_at_the_cap_and_counts_stay_exact(cro, ctx, clean):
    import sparse
    leg, smid = cro.SPARSE_LEG_TF32, clean[1][0].smid
    r, sms, faults = ctx.probe_sparse(0, iterations=2, legs=1 << leg, inject=(leg, smid, 1, -1, -1, EXP_MASK),
                                      cap=cro.SPARSE_RECORDS + 16)
    L = r.leg[leg]
    ctas = [s for s in sms if s.smid == smid][0].leg[leg].ctas
    assert L.mismatches == sparse.M * sparse.N * ctas and L.recorded == cro.SPARSE_RECORDS
    assert len(faults) == cro.SPARSE_RECORDS
    tile = answers(r.seed)[sparse.LEG_ANSWER[leg]]
    for f in faults[:64]:
        assert f.smid == smid and f.expected == tile[f.row, f.col]
        assert f.actual_bits == sparse.value_bits(leg, int(tile[f.row, f.col])) ^ EXP_MASK


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_sparse(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_sparse(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(legs=0x40), dict(iterations=cro.SPARSE_MAX_ITERATIONS + 1), dict(max_rounds=cro.SPARSE_MAX_ROUNDS + 1),
             dict(inject=(0, 256, 0, 0, 0, 1)), dict(inject=(6, 0, 0, 0, 0, 1)), dict(inject=(2, 0, 3, 0, 0, 1), iterations=3),
             dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)), dict(inject=(2, 0, 0, 0, 0, 1 << 32)),
             dict(meta=(6, 0, 0, 0, 0)), dict(meta=(0, 256, 0, 0, 0)), dict(meta=(0, 0, 3, 0, 0), iterations=3),
             dict(meta=(0, 0, 0, 128, 0)), dict(meta=(0, 0, 0, 0, 128)), dict(meta=(3, 0, 0, 0, 64)),
             dict(meta=(5, 0, 0, 0, 64)), dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_sparse(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw


# ---- the helper form ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def uuid(ctx):
    return ctx.own_devices()[0].gpu_uuid.decode()


def test_helper_clean_call(cro, ctx, uuid):
    r, sms, faults, ns = cro.probe_sparse_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert ns > 0
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.call == 0 and r.seed != (dev + (1 << 57)) & MASK         # the helper's own seed base, not the context's


@pytest.mark.parametrize("kind", ["inject", "meta"])
def test_helper_names_what_the_in_process_form_names(cro, ctx, clean, uuid, kind):
    smid = clean[1][-1].smid
    kw = dict(inject=(cro.SPARSE_LEG_BF16, smid, 2, ROW, COL, 1)) if kind == "inject" else \
        dict(meta=(cro.SPARSE_LEG_BF16, smid, 2, ROW, 45))
    a = ctx.probe_sparse(0, iterations=3, **kw)
    b = cro.probe_sparse_uuid(ctx, uuid, iterations=3, **kw)[:3]
    for r, sms, faults in (a, b):
        check_one_sm(cro, r, sms, faults, cro.SPARSE_LEG_BF16, smid, cro.COMPUTE_PERSISTENT)
    # the two forms have their own seeds: a substitution's columns follow the seed, its row does not
    assert {f.row for f in a[2]} == {f.row for f in b[2]} == {ROW}
    if kind == "inject":
        assert [(f.row, f.col) for f in a[2]] == [(f.row, f.col) for f in b[2]]


def test_helper_refuses_bad_options_before_any_launch(cro, ctx, uuid):
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sparse_uuid(ctx, uuid, meta=(0, 0, 0, 0, 128))
    assert e.value.code == cro.ERR_INVALID_ARG
