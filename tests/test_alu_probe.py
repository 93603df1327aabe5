"""The ALU probe (cro_probe_alu, cro_probe_alu_uuid) on one H100, against oracle/alu.py.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import json

import pytest

pytestmark = pytest.mark.gpu

# One injected (op, operand word, mask) per leg whose change the form's result shows on every lane: lop3 at LUT 0x96
# (a ^ b ^ c) on c, shf.l.wrap on b's bit 0, the 64-bit add chain on a, mad.lo.u32 on c, and mul.rn.f32 on a's sign.
INJECT = {0: (0x96 * 2 + 1, 2, 1 << 7), 1: (0, 1, 1), 2: (1, 0, 1 << 40), 3: (6 * 4 + 1, 2, 1), 4: (8 * 8 + 3, 0, 1 << 31)}


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_alu(0)


def check_clean(cro, ctx, r, sms, faults, iterations, legs=0x1F):
    import alu
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.ALU_NONE and not faults, \
        (r.status, r.verdict, [(f.leg, f.op, f.warp, f.lane, [hex(x) for x in f.in_], [hex(x) for x in f.expected],
                                [hex(x) for x in f.actual]) for f in faults[:8]])
    assert r.sm_count == n and r.sms_covered == n and r.complete == 1 and r.unpublished == 0 and r.threads_unpublished == 0
    assert r.iterations == iterations and r.legs == legs and r.bad_sms == 0 and r.failed_legs == 0 and r.recorded == 0
    for leg in range(cro.ALU_LEGS):
        if legs >> leg & 1:
            assert r.mismatches[leg] == 0 and r.fold_mismatches[leg] == 0 and r.leg_ns[leg] > 0
            assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == alu.fold(leg, r.seed), leg
            assert r.ops_checked[leg] >= cro.ALU_OPS[leg] * 256 * iterations * n
    assert r.ns > 0 and r.timer_ns > 0 and r.wall_ns > r.table_ns > 0
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    assert all(s.ctas >= 1 and s.mark == 0 and s.cycles > 0 and s.fold_mismatches == 0 for s in sms)


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, r.iterations)
    print("alu default: %d iterations, %d rounds, %.2f ms of launches (%s us per leg), table %.2f ms, %.2f ms the call"
          % (r.iterations, r.rounds, r.ns / 1e6, [round(x / 1e3) for x in r.leg_ns], r.table_ns / 1e6, r.wall_ns / 1e6))


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_alu(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


def test_seeds_follow_the_formula_and_are_fresh_per_call(cro, ctx):
    import alu
    import xlane
    a, _, _ = ctx.probe_alu(0, iterations=1)
    b, _, _ = ctx.probe_alu(0, iterations=1)
    assert b.call == a.call + 1 and a.status == b.status == 0
    s, _, _ = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=1)        # seed_dev + 2^60 + 8k strides
    seed_dev = (s.seed - (1 << 60) - 8 * s.call * xlane.STRIDE) & alu.U64
    assert a.seed == alu.call_seed(seed_dev, a.call) and b.seed == alu.call_seed(seed_dev, b.call)
    assert [tuple(f) for f in b.fold] != [tuple(f) for f in a.fold]


@pytest.mark.parametrize("leg", range(5))
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("warp", [0, 7])
@pytest.mark.parametrize("lane", [0, 31])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_one_injection_names_the_sm_leg_and_record(cro, ctx, clean, leg, where, warp, lane, when):
    import alu
    iterations = 3
    it = iterations - 1 if when == "last" else 1
    smid = clean[1][0 if where == "first" else -1].smid
    op, operand, mask = INJECT[leg]
    r, sms, faults = ctx.probe_alu(0, iterations=iterations, legs=1 << leg, inject=(leg, smid, warp, lane, op, it, operand, mask),
                                   cap=cro.ALU_RECORDS)
    want = alu.injected(leg, r.seed, op, warp, lane, operand, mask)
    assert want is not None
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.ALU_SM, (r.status, r.verdict)
    assert r.bad_sms == 1 and list(r.bad_sm[:1]) == [smid] and r.failed_legs == 1 << leg
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid and entry.failed_legs == 1 << leg
    assert entry.mark == (cro.ALU_PERSISTENT if when == "last" else cro.ALU_INTERMITTENT)
    assert r.mismatches[leg] == entry.ctas and r.fold_mismatches[leg] == (entry.ctas if when == "last" else 0)
    assert len(faults) == entry.ctas
    for f in faults:
        assert (f.leg, f.op, f.iteration, f.smid, f.warp, f.lane) == (leg, op, it, smid, warp, lane)
        assert (list(f.in_), tuple(f.expected), tuple(f.actual)) == want


def test_injection_into_every_sm_is_a_common_cause_and_records_cap(cro, ctx):
    op, operand, mask = INJECT[0]             # lop3 0x96 on c: every lane fails, once
    r, sms, faults = ctx.probe_alu(0, iterations=2, legs=1, inject=(0, -1, -1, -1, op, 0, operand, mask), cap=cro.ALU_RECORDS + 16)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.ALU_ALL
    assert r.failed_sms == r.sms_covered == len(sms) and r.bad_sms == len(sms)
    assert r.mismatches[0] == 256 * r.ctas and r.recorded == cro.ALU_RECORDS and len(faults) == cro.ALU_RECORDS
    assert all(s.mark == cro.ALU_INTERMITTENT for s in sms)
    assert faults == sorted(faults, key=lambda f: (f.smid, f.iteration, f.op, f.warp, f.lane))
    ann = json.loads(cro.emit_alu_annotations_json(r))
    assert ann["cohdi.io/probe-alu-verdict"] == "all" and ann["cohdi.io/probe-alu-legs"] == "logic"


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_alu(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_alu(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, clean):
    import alu
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_alu_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    smid = clean[1][-1].smid
    op, operand, mask = INJECT[4]
    inj = (4, smid, 5, 9, op, 1, operand, mask)
    for r, sms, faults in (ctx.probe_alu(0, iterations=2, legs=1 << 4, inject=inj),
                           cro.probe_alu_uuid(None, uuid, iterations=2, legs=1 << 4, inject=inj)):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.ALU_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        want = alu.injected(4, r.seed, op, 5, 9, operand, mask)
        assert {(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, tuple(f.in_), tuple(f.expected), tuple(f.actual))
                for f in faults} == {(4, op, 1, smid, 5, 9, tuple(want[0]), want[1], want[2])}


def test_invalid_arguments_are_refused(cro, ctx):
    from test_alu_abi import BAD_OPTIONS
    before = ctx.launch_count()
    for kw in BAD_OPTIONS + [dict(dev=len(ctx.own_devices()))]:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_alu(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert ctx.launch_count() == before
