"""The cross-lane probe (cro_probe_xlane, cro_probe_xlane_uuid) on one H100, against oracle/xlane.py.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import json

import pytest

pytestmark = pytest.mark.gpu

# One injected op per leg and a mask that changes its result wherever the lane sits: an idx shuffle (source lane + 5), a
# seeded ballot, a .b64 match.any over one class, a seeded add.u32 reduction and the CTA-wide add.u32 shared atomic.
INJECT = {0: (5, 1 << 19), 1: (70 * 4, 1), 2: (2, 1 << 40), 3: (130 * 9, 1 << 7), 4: (0, 1 << 3)}


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_xlane(0)


def check_clean(cro, ctx, r, sms, faults, iterations, legs=0x1F):
    import xlane
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.XLANE_NONE and not faults, (r.status, r.verdict, faults[:4])
    assert r.sm_count == n and r.sms_covered == n and r.complete == 1 and r.unpublished == 0 and r.threads_unpublished == 0
    assert r.iterations == iterations and r.legs == legs and r.bad_sms == 0 and r.failed_legs == 0 and r.recorded == 0
    for leg in range(cro.XLANE_LEGS):
        if legs >> leg & 1:
            assert r.mismatches[leg] == 0 and r.fold_mismatches[leg] == 0 and r.leg_ns[leg] > 0
            assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == xlane.fold(leg, r.seed, iterations), leg
            assert r.ops_checked[leg] >= cro.XLANE_OPS[leg] * 256 * iterations * n
    assert r.ns > 0 and r.timer_ns > 0 and r.wall_ns > 0
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    assert all(s.ctas >= 1 and s.mark == 0 and s.cycles > 0 and s.fold_mismatches == 0 for s in sms)


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, r.iterations)
    print("xlane default: %d iterations, %d rounds, %.2f ms of launches (%s us per leg), %.2f ms the call"
          % (r.iterations, r.rounds, r.ns / 1e6, [round(x / 1e3) for x in r.leg_ns], r.wall_ns / 1e6))


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_xlane(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


def test_seeds_follow_the_formula_and_are_fresh_per_call(cro, ctx):
    import xlane
    a, _, _ = ctx.probe_xlane(0, iterations=1)
    b, _, _ = ctx.probe_xlane(0, iterations=1)
    assert b.call == a.call + 1 and a.status == b.status == 0
    s, _, _ = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=1)        # seed_dev + 2^60 + 8k strides
    seed_dev = (s.seed - (1 << 60) - 8 * s.call * xlane.STRIDE) & xlane.U64
    assert a.seed == xlane.call_seed(seed_dev, a.call) and b.seed == xlane.call_seed(seed_dev, b.call)
    assert b.seed == (a.seed + 4096 * xlane.STRIDE) & xlane.U64
    assert [tuple(f) for f in b.fold] != [tuple(f) for f in a.fold]


@pytest.mark.parametrize("leg", range(5))
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("warp", [0, 7])
@pytest.mark.parametrize("lane", [0, 31])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_one_injection_names_the_sm_leg_and_records(cro, ctx, clean, leg, where, warp, lane, when):
    import xlane
    iterations = 3
    it = iterations - 1 if when == "last" else 1
    smid = clean[1][0 if where == "first" else -1].smid
    op, mask = INJECT[leg]
    r, sms, faults = ctx.probe_xlane(0, iterations=iterations, legs=1 << leg, inject=(leg, smid, warp, lane, op, it, mask),
                                     cap=cro.XLANE_RECORDS)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.XLANE_SM, (r.status, r.verdict)
    assert r.bad_sms == 1 and list(r.bad_sm[:1]) == [smid] and r.failed_legs == 1 << leg
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid and entry.failed_legs == 1 << leg
    assert entry.mark == (cro.XLANE_PERSISTENT if when == "last" else cro.XLANE_INTERMITTENT)
    want = xlane.injected(leg, r.seed, it, op, warp, lane, mask)
    assert want
    assert r.mismatches[leg] == len(want) * entry.ctas and r.fold_mismatches[leg] == (entry.ctas if when == "last" else 0)
    got = {}
    for f in faults:
        assert (f.leg, f.op, f.iteration, f.smid) == (leg, op, it, smid)
        got.setdefault((f.warp, f.lane), []).append((f.expected, f.actual, f.peer))
    assert sorted(got) == sorted(want)
    assert all(v == [want[k]] * entry.ctas for k, v in got.items())


def test_injection_into_every_sm_is_a_common_cause_and_records_cap(cro, ctx):
    op, mask = INJECT[0]                    # every lane's shuffle source is injected: every lane fails, once
    r, sms, faults = ctx.probe_xlane(0, iterations=2, legs=1, inject=(0, -1, -1, -1, op, 0, mask), cap=cro.XLANE_RECORDS + 16)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.XLANE_ALL
    assert r.failed_sms == r.sms_covered == len(sms) and r.bad_sms == len(sms)
    assert r.mismatches[0] == 256 * r.ctas and r.recorded == cro.XLANE_RECORDS and len(faults) == cro.XLANE_RECORDS
    assert all(s.mark == cro.XLANE_INTERMITTENT for s in sms)
    assert faults == sorted(faults, key=lambda f: (f.smid, f.iteration, f.op, f.warp, f.lane))
    assert json.loads(cro.emit_xlane_annotations_json(r))["cohdi.io/probe-xlane-verdict"] == "all"
    assert json.loads(cro.emit_xlane_annotations_json(r))["cohdi.io/probe-xlane-legs"] == "shfl"


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_xlane(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_xlane(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, clean):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_xlane_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    smid = clean[1][-1].smid
    op, mask = INJECT[0]
    inj = (0, smid, 5, 9, op, 1, mask)
    a = ctx.probe_xlane(0, iterations=2, legs=1, inject=inj)
    b = cro.probe_xlane_uuid(None, uuid, iterations=2, legs=1, inject=inj)
    for r, sms, faults in (a, b):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.XLANE_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        assert {(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, f.peer, f.expected ^ f.actual) for f in faults} == \
            {(0, op, 1, smid, 5, 4, 9, mask)}


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(iterations=cro.XLANE_MAX_ITERATIONS + 1), dict(max_rounds=cro.XLANE_MAX_ROUNDS + 1), dict(legs=0x20),
             dict(inject=(5, 0, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 0, 1)),
             dict(inject=(0, -2, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 8, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 32, 0, 0, 1)),
             dict(inject=(0, 0, 0, 0, 177, 0, 1)), dict(inject=(4, 0, 0, 0, 4, 0, 1)), dict(inject=(4, 0, 0, 0, 8, 0, 1)),
             dict(inject=(0, 0, 0, 0, 0, 3, 1), iterations=3), dict(inject=(1, 0, 0, 0, 0, 0, 1), legs=1),
             dict(dev=len(ctx.own_devices()))]
    before = ctx.launch_count()
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_xlane(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert ctx.launch_count() == before
