"""The register-file probe (cro_probe_regfile, cro_probe_regfile_uuid) on one H100, against oracle/regfile.py.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import json

import pytest

BIT = 1 << 19

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_regfile(0)


def check_clean(cro, ctx, r, sms, faults, iterations):
    import regfile
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.REGFILE_NONE and not faults, (r.status, r.verdict, faults[:4])
    assert r.sm_count == n and r.sms_covered == n and r.complete == 1 and r.unpublished == 0 and r.bad_sms == 0
    assert r.iterations == iterations and r.slots == cro.REGFILE_SLOTS and r.threads == cro.REGFILE_THREADS
    assert list(r.mismatches) == [0, 0] and r.fold_mismatches == 0 and r.recorded == 0 and r.failed_sms == 0
    assert r.fold == r.expect == regfile.fold(r.seed, iterations)
    assert r.num_regs >= 250 and r.regs_per_sm == 65536
    assert r.bits_checked == 32 * 224 * 256 * 2 * iterations * (r.ctas - r.unpublished)
    assert r.ns > 0 and r.timer_ns > 0 and r.wall_ns > 0
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    assert all(s.ctas >= 1 and s.mark == 0 and s.cycles > 0 and s.fold_mismatches == 0 for s in sms)


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, r.iterations)
    assert r.iterations >= 1 and r.rounds >= 1
    print("regfile default: %d iterations, %d rounds, %.2f ms of launches, %.2f ms the call, %d registers per thread"
          % (r.iterations, r.rounds, r.ns / 1e6, r.wall_ns / 1e6, r.num_regs))


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_regfile(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


def test_seeds_follow_the_formula_and_are_fresh_per_call(cro, ctx):
    import regfile
    a, _, _ = ctx.probe_regfile(0, iterations=1)
    b, _, _ = ctx.probe_regfile(0, iterations=1)
    assert b.call == a.call + 1 and a.status == b.status == 0
    s, _, _ = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=1)        # seed_dev + 2^60 + 8k strides
    seed_dev = (s.seed - (1 << 60) - 8 * s.call * regfile.STRIDE) & regfile.U64
    assert a.seed == regfile.call_seed(seed_dev, a.call) and b.seed == regfile.call_seed(seed_dev, b.call)
    assert b.seed == (a.seed + 4096 * regfile.STRIDE) & regfile.U64
    assert b.fold != a.fold


SLOT_LAST = 223


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("warp", [0, 7])
@pytest.mark.parametrize("lane", [0, 31])
@pytest.mark.parametrize("slot", [0, SLOT_LAST])
@pytest.mark.parametrize("element", [0, 1])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_one_slot_injection_names_the_sm_warp_lane_and_slot(cro, ctx, clean, where, warp, lane, slot, element, when):
    import regfile
    iterations = 4
    it = iterations - 1 if when == "last" else 1
    smid = clean[1][0 if where == "first" else -1].smid
    r, sms, faults = ctx.probe_regfile(0, iterations=iterations, inject=(smid, warp, lane, slot, element, it, BIT))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.REGFILE_SM, (r.status, r.verdict)
    assert r.bad_sms == 1 and list(r.bad_sm[:1]) == [smid] and r.failed_sms == 1
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid
    assert entry.mark == (cro.REGFILE_PERSISTENT if when == "last" else cro.REGFILE_INTERMITTENT)
    want = [0, 0]
    want[element] = entry.ctas
    assert list(entry.mismatches) == want and list(r.mismatches) == want
    folded = element == 1 and when == "last"
    assert r.fold_mismatches == (entry.ctas if folded else 0)
    assert len(faults) == entry.ctas and r.recorded == entry.ctas
    t = 32 * warp + lane
    for f in faults:
        assert (f.element, f.iteration, f.smid, f.warp, f.lane, f.slot) == (element, it, smid, warp, lane, slot)
        e = regfile.word(r.seed, it, t, slot) ^ (0xFFFFFFFF if element else 0)
        assert f.expected == e and f.actual == e ^ BIT


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    r, sms, _ = ctx.probe_regfile(0, iterations=2, inject=(-1, 3, 5, 17, 0, 0, BIT))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.REGFILE_ALL
    assert r.failed_sms == r.sms_covered == len(sms) and r.mismatches[0] == r.ctas and r.bad_sms == len(sms)
    assert all(s.mark == cro.REGFILE_INTERMITTENT for s in sms)
    assert json.loads(cro.emit_regfile_annotations_json(r))["cohdi.io/probe-regfile-verdict"] == "all"


def test_injection_into_every_slot_of_every_thread_counts_exactly(cro, ctx, clean):
    import regfile
    smid = clean[1][0].smid
    r, sms, faults = ctx.probe_regfile(0, iterations=2, inject=(smid, -1, -1, -1, 1, 1, 0x80000001),
                                       cap=cro.REGFILE_RECORDS + 16)
    (entry,) = [s for s in sms if s.smid == smid]
    assert r.verdict == cro.REGFILE_SM and entry.mark == cro.REGFILE_PERSISTENT
    assert list(r.mismatches) == [0, 224 * 256 * entry.ctas] and r.fold_mismatches == entry.ctas
    assert r.recorded == cro.REGFILE_RECORDS and len(faults) == cro.REGFILE_RECORDS
    for f in faults[:64]:
        e = regfile.word(r.seed, 1, 32 * f.warp + f.lane, f.slot) ^ 0xFFFFFFFF
        assert f.smid == smid and f.element == 1 and f.iteration == 1 and f.expected == e and f.actual == e ^ 0x80000001


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_regfile(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_regfile(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, clean):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_regfile_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    smid = clean[1][-1].smid
    inj = (smid, 5, 9, 101, 0, 1, BIT)
    a = ctx.probe_regfile(0, iterations=2, inject=inj)
    b = cro.probe_regfile_uuid(None, uuid, iterations=2, inject=inj)
    for r, sms, faults in (a, b):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.REGFILE_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        assert {(f.element, f.iteration, f.smid, f.warp, f.lane, f.slot, f.expected ^ f.actual) for f in faults} == \
            {(0, 1, smid, 5, 9, 101, BIT)}
    assert a[0].num_regs == b[0].num_regs


def test_nvml_fields_equal_a_read_right_after(cro, ctx):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, _, _ = ctx.probe_regfile(0, iterations=1)
    h = cro.read_sram_health(uuid)
    assert (r.after.nvml, r.after.threshold_exceeded, r.after.ecc_corrected, r.after.ecc_uncorrected) == \
        (h.nvml, h.threshold_exceeded, h.ecc_corrected, h.ecc_uncorrected)
    assert r.before.nvml == h.nvml & ~cro.SRAM_NVML_STATUS


def test_invalid_arguments_are_refused(cro, ctx):
    calls = [dict(iterations=cro.REGFILE_MAX_ITERATIONS + 1), dict(max_rounds=cro.REGFILE_MAX_ROUNDS + 1),
             dict(inject=(256, 0, 0, 0, 0, 0, 1)), dict(inject=(-2, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 8, 0, 0, 0, 0, 1)),
             dict(inject=(0, 0, 32, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 224, 0, 0, 1)), dict(inject=(0, 0, 0, -2, 0, 0, 1)),
             dict(inject=(0, 0, 0, 0, 2, 0, 1)), dict(inject=(0, 0, 0, 0, 0, 3, 1), iterations=3),
             dict(dev=len(ctx.own_devices()))]
    before = ctx.launch_count()
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_regfile(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert ctx.launch_count() == before
