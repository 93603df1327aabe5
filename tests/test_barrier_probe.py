"""The barrier probe (cro_probe_barrier, cro_probe_barrier_uuid) on one H100, against oracle/barrier.py.

Faults come only from the probe's software injection (test_inject_*), which never adds or skips an arrival and never
changes a count or a byte total; nothing here repeats a call to catch a real fault."""
import json

import pytest

pytestmark = pytest.mark.gpu

# One injected row per leg that every thread of warps 0 and 7 checks: bar.red.popc over all 8 warps (row 7), an
# mbarrier COUNT row (row 2: three checks per phase) and st.async.v4 (row 5: the wait and both received words).
INJECT = {0: 7, 1: 2, 2: 5}
MASK = 1 << 9


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_barrier(0)


def check_clean(cro, ctx, r, sms, faults, iterations, legs=0x7, cluster=2):
    import barrier
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.BARRIER_NONE and not faults, \
        (r.status, r.verdict, [(f.leg, f.op, f.kind, f.phase, f.slot, f.warp, f.lane, hex(f.expected), hex(f.actual)) for f in faults[:8]])
    assert r.sm_count == n and r.unpublished == 0 and r.threads_unpublished == 0 and r.timeouts == 0
    assert r.iterations == iterations and r.legs == legs and r.cluster == cluster and r.bad_sms == 0 and r.failed_legs == 0
    assert r.recorded == 0 and r.bad_pairs == 0
    for leg in range(cro.BARRIER_LEGS):
        if legs >> leg & 1:
            assert r.mismatches[leg] == 0 and r.fold_mismatches[leg] == 0 and r.leg_ns[leg] > 0
            assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == barrier.fold(leg, r.seed, cluster), leg
            assert r.ops_checked[leg] >= cro.BARRIER_OPS[leg] * 256 * iterations * (n if leg != cro.BARRIER_LEG_CLUSTER else 1)
    if legs & 3:
        assert r.sms_covered == n and r.complete == 1
    assert r.ns > 0 and r.timer_ns > 0 and r.wall_ns > r.table_ns > 0
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == (n if legs & 3 else r.sms_covered)
    assert all(s.ctas >= 1 and s.mark == 0 and s.cycles > 0 and s.fold_mismatches == 0 for s in sms)


def test_clean_default_call(cro, ctx, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, r, sms, faults, r.iterations)
    print("barrier default: %d iterations, %d rounds, %.2f ms of launches (%s us per leg), cluster leg on %d SMs, table %.2f ms, "
          "%.2f ms the call" % (r.iterations, r.rounds, r.ns / 1e6, [round(x / 1e3) for x in r.leg_ns], r.cluster_sms,
                                r.table_ns / 1e6, r.wall_ns / 1e6))


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, iterations):
    r, sms, faults = ctx.probe_barrier(0, iterations=iterations)
    check_clean(cro, ctx, r, sms, faults, iterations)


@pytest.mark.parametrize("cluster", [2, 4, 8])
def test_cluster_leg_is_clean_at_every_size_and_reports_its_coverage(cro, ctx, cluster):
    r, sms, faults = ctx.probe_barrier(0, iterations=3, legs=1 << cro.BARRIER_LEG_CLUSTER, cluster=cluster)
    check_clean(cro, ctx, r, sms, faults, 3, legs=4, cluster=cluster)
    assert r.cluster_sms == r.sms_covered == len(sms) > 0 and r.complete == int(r.sms_covered == r.sm_count)
    print("barrier cluster %d: %d of %d SMs in %d rounds" % (cluster, r.cluster_sms, r.sm_count, r.rounds))


def test_seeds_follow_the_formula_and_are_fresh_per_call(cro, ctx):
    import barrier
    import xlane
    a, _, _ = ctx.probe_barrier(0, iterations=1, legs=1)
    b, _, _ = ctx.probe_barrier(0, iterations=1, legs=1)
    assert b.call == a.call + 1 and a.status == b.status == 0
    s, _, _ = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=1)        # seed_dev + 2^60 + 8k strides
    seed_dev = (s.seed - (1 << 60) - 8 * s.call * xlane.STRIDE) & barrier.U64
    assert a.seed == barrier.call_seed(seed_dev, a.call) and b.seed == barrier.call_seed(seed_dev, b.call)
    assert [tuple(f) for f in b.fold] != [tuple(f) for f in a.fold]


@pytest.fixture(scope="module")
def cluster_sms(ctx):
    r, sms, _ = ctx.probe_barrier(0, iterations=1, legs=4)
    assert r.status == 0
    return [s.smid for s in sms]


@pytest.mark.parametrize("leg", range(3))
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("warp", [0, 7])
@pytest.mark.parametrize("lane", [0, 31])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_one_injection_names_the_sm_leg_and_record(cro, ctx, clean, cluster_sms, leg, where, warp, lane, when):
    import barrier
    iterations = 3
    it = iterations - 1 if when == "last" else 1
    smids = cluster_sms if leg == cro.BARRIER_LEG_CLUSTER else [s.smid for s in clean[1]]
    smid = smids[0 if where == "first" else -1]
    op = INJECT[leg]
    r, sms, faults = ctx.probe_barrier(0, iterations=iterations, legs=1 << leg, inject=(leg, smid, warp, lane, op, it, MASK),
                                       cap=cro.BARRIER_RECORDS)
    want = barrier.injected(leg, r.seed, op, warp, lane, MASK)
    assert r.status == cro.ERR_CHECKSUM, (r.status, r.verdict)
    assert r.verdict == (cro.BARRIER_LINK if leg == cro.BARRIER_LEG_CLUSTER else cro.BARRIER_SM)
    assert r.bad_sms == 1 and list(r.bad_sm[:1]) == [smid] and r.failed_legs == 1 << leg and r.timeouts == 0
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid and entry.failed_legs == 1 << leg
    assert entry.mark == (cro.BARRIER_PERSISTENT if when == "last" else cro.BARRIER_INTERMITTENT)
    assert r.mismatches[leg] == len(want) * entry.ctas and r.fold_mismatches[leg] == (entry.ctas if when == "last" else 0)
    assert len(faults) == min(len(want), cro.BARRIER_THREAD_RECORDS) * entry.ctas
    for i, f in enumerate(faults):
        assert (f.leg, f.op, f.iteration, f.smid, f.warp, f.lane) == (leg, op, it, smid, warp, lane)
        assert (f.kind, f.bar, f.phase, f.slot, f.expected, f.actual) == want[i % min(len(want), cro.BARRIER_THREAD_RECORDS)]
        if leg == cro.BARRIER_LEG_CLUSTER:
            assert f.peer_smid != smid
        else:
            assert f.peer_smid == smid
    if leg == cro.BARRIER_LEG_CLUSTER:
        pairs = sorted({(f.smid, f.peer_smid) for f in faults})
        assert r.bad_pairs == len(pairs) and [(p.smid, p.peer_smid) for p in r.bad_pair[:r.bad_pairs]] == pairs
        ann = json.loads(cro.emit_barrier_annotations_json(r))
        assert ann["cohdi.io/probe-barrier-verdict"] == "link"
        assert ann["cohdi.io/probe-barrier-bad-pairs"] == ",".join("%d>%d" % p for p in pairs)


def test_injection_into_every_sm_is_a_common_cause_and_records_cap(cro, ctx):
    op = INJECT[1]
    r, sms, faults = ctx.probe_barrier(0, iterations=2, legs=2, inject=(1, -1, -1, -1, op, 0, MASK), cap=cro.BARRIER_RECORDS + 16)
    import barrier
    n_checks = len(barrier.injected(1, r.seed, op, 0, 0, MASK))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.BARRIER_ALL
    assert r.failed_sms == r.sms_covered == len(sms) and r.bad_sms == len(sms)
    assert r.mismatches[1] == 256 * n_checks * r.ctas and r.recorded == cro.BARRIER_RECORDS and len(faults) == cro.BARRIER_RECORDS
    assert all(s.mark == cro.BARRIER_INTERMITTENT for s in sms)
    assert faults == sorted(faults, key=lambda f: (f.smid, f.iteration, f.op, f.warp, f.lane))
    ann = json.loads(cro.emit_barrier_annotations_json(r))
    assert ann["cohdi.io/probe-barrier-verdict"] == "all" and ann["cohdi.io/probe-barrier-legs"] == "mbar"


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_barrier(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_barrier(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, clean):
    import barrier
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_barrier_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, r, sms, faults, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    smid = clean[1][-1].smid
    op = INJECT[1]
    inj = (1, smid, 5, 9, op, 1, MASK)
    for r, sms, faults in (ctx.probe_barrier(0, iterations=2, legs=2, inject=inj),
                           cro.probe_barrier_uuid(None, uuid, iterations=2, legs=2, inject=inj)):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.BARRIER_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        want = barrier.injected(1, r.seed, op, 5, 9, MASK)[:cro.BARRIER_THREAD_RECORDS]
        assert {(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, f.kind, f.bar, f.phase, f.slot, f.expected, f.actual)
                for f in faults} == {(1, op, 1, smid, 5, 9) + w for w in want}


def test_invalid_arguments_are_refused(cro, ctx):
    from test_barrier_abi import BAD_OPTIONS
    before = ctx.launch_count()
    for kw in BAD_OPTIONS + [dict(dev=len(ctx.own_devices()))]:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_barrier(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert ctx.launch_count() == before


# ---- every row's records against the restatement -------------------------------------------------------------------
@pytest.mark.parametrize("leg", range(3))
def test_every_rows_injection_records_match_the_restatement(cro, ctx, clean, cluster_sms, leg):
    """One injection per row (thread (3, 5) of the first covered SM, the one iteration): the device's records and
    counts are the restatement's for every form, tickets, drops, transaction bytes, reductions and CBAR included.  A
    CLUSTER CTA's rank is not reported, so its records must match the prediction for one of the cluster's ranks."""
    import barrier
    smid = (cluster_sms if leg == cro.BARRIER_LEG_CLUSTER else [s.smid for s in clean[1]])[0]
    for op in range(cro.BARRIER_OPS[leg]):
        r, sms, faults = ctx.probe_barrier(0, iterations=1, legs=1 << leg, inject=(leg, smid, 3, 5, op, 0, MASK), cap=cro.BARRIER_RECORDS)
        wants = [barrier.injected(leg, r.seed, op, 3, 5, MASK, 2, rank) for rank in range(2)]
        if not wants[0]:                 # the thread checks nothing in this row
            assert r.status == cro.OK and not faults, (leg, op)
            continue
        (entry,) = [s for s in sms if s.mark]
        assert r.status == cro.ERR_CHECKSUM and entry.smid == smid and r.timeouts == 0, (leg, op)
        assert r.mismatches[leg] == len(wants[0]) * entry.ctas, (leg, op)
        got = [(f.kind, f.bar, f.phase, f.slot, f.expected, f.actual) for f in faults]
        assert all((f.leg, f.op, f.iteration, f.smid, f.warp, f.lane) == (leg, op, 0, smid, 3, 5) for f in faults)
        kept = min(len(wants[0]), cro.BARRIER_THREAD_RECORDS)
        for j in range(entry.ctas):
            assert any(got[j * kept:(j + 1) * kept] == w[:kept] for w in wants), (leg, op, got[j * kept:(j + 1) * kept], wants[0][:kept])


# ---- with part of the GPU held busy by tests/sm_holder.cu (built here, as tests/test_held_sms.py does) ---------------
K = 8


@pytest.fixture(scope="module")
def holder(tmp_path_factory, _built):
    import subprocess
    from test_held_sms import Holder, holder_cmd
    out = str(tmp_path_factory.mktemp("holder") / "sm_holder.so")
    subprocess.check_call(holder_cmd(out))
    h = Holder(out)
    try:
        yield h
    finally:
        h.lib.holder_release()


@pytest.fixture(scope="module")
def every_sm(ctx, clean):
    got = {s.smid for s in clean[1]}
    assert len(got) == ctx.own_devices()[0].sm_count
    return got


@pytest.mark.parametrize("max_rounds", [1, 0], ids=["rounds1", "rounds-default"])
@pytest.mark.parametrize("leg", [0, 1])
def test_cta_local_leg_covers_exactly_the_free_sms_under_a_hold(cro, ctx, holder, every_sm, leg, max_rounds):
    import barrier
    n = len(every_sm)
    with holder.hold(K) as H:
        r, sms, faults = ctx.probe_barrier(0, iterations=1, legs=1 << leg, max_rounds=max_rounds)
    rounds = max_rounds or 4
    per = {s.smid: s.ctas for s in sms if s.ctas}
    assert set(per) == every_sm - H and not set(per) & H, (sorted(set(per) & H), sorted(every_sm - H - set(per)))
    assert r.sms_covered == n - K and r.complete == 0 and r.rounds == rounds
    assert r.ctas == n * rounds == sum(per.values()) and max(per.values()) >= 2
    assert r.status == cro.OK and r.verdict == cro.BARRIER_NONE and not faults and r.failed_sms == 0 and r.timeouts == 0
    assert r.unpublished == 0 and r.threads_unpublished == 0
    assert r.ops_checked[leg] == cro.BARRIER_OPS[leg] * 256 * n * rounds
    assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == barrier.fold(leg, r.seed)
    assert json.loads(cro.emit_barrier_annotations_json(r))["cohdi.io/probe-barrier-sms"] == "%d/%d" % (n - K, n)
    print("barrier leg %d under a hold: H %s, rounds %d, sms_covered %d, max ctas %d"
          % (leg, sorted(H), r.rounds, r.sms_covered, max(per.values())))


@pytest.mark.parametrize("where", ["free", "held", "every"])
@pytest.mark.parametrize("leg", [0, 1])
def test_injection_under_a_hold(cro, ctx, holder, every_sm, leg, where):
    import barrier
    n, iterations, op = len(every_sm), 2, INJECT[leg]
    with holder.hold(K) as H:
        smid = {"free": max(every_sm - H), "held": max(H), "every": -1}[where]
        r, sms, faults = ctx.probe_barrier(0, iterations=iterations, legs=1 << leg,
                                           inject=(leg, smid, 3, 17, op, iterations - 1, MASK), cap=cro.BARRIER_RECORDS)
    per = {s.smid: s.ctas for s in sms if s.ctas}
    assert set(per) == every_sm - H and r.sms_covered == n - K and r.ctas == 4 * n == sum(per.values())
    want = barrier.injected(leg, r.seed, op, 3, 17, MASK)
    if where == "held":
        assert r.status == cro.OK and r.verdict == cro.BARRIER_NONE and not faults and r.failed_sms == 0
        return
    if where == "every":
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.BARRIER_ALL and r.failed_sms == r.sms_covered == n - K
        assert r.mismatches[leg] == len(want) * r.ctas
        return
    ctas = per[smid]
    assert ctas >= 1 and r.status == cro.ERR_CHECKSUM and r.verdict == cro.BARRIER_SM and r.bad_sms == 1 and r.bad_sm[0] == smid
    assert r.mismatches[leg] == len(want) * ctas and r.fold_mismatches[leg] == ctas
    kept = min(len(want), cro.BARRIER_THREAD_RECORDS)
    assert [(f.smid, f.iteration, f.warp, f.lane, f.kind, f.bar, f.phase, f.slot, f.expected, f.actual) for f in faults] == \
        [(smid, iterations - 1, 3, 17) + w for _ in range(ctas) for w in want[:kept]]


@pytest.mark.parametrize("cluster", [2, 8])
def test_cluster_leg_under_a_hold(cro, ctx, holder, every_sm, cluster):
    """Clusters cannot use a held SM, nor a free SM whose GPC has no room left for a whole cluster: the leg stays clean,
    runs only on free SMs and states its coverage."""
    import barrier
    n = len(every_sm)
    with holder.hold(K) as H:
        r, sms, faults = ctx.probe_barrier(0, iterations=1, legs=4, cluster=cluster)
    per = {s.smid: s.ctas for s in sms if s.ctas}
    assert r.status == cro.OK and r.verdict == cro.BARRIER_NONE and not faults and r.bad_pairs == 0 and r.timeouts == 0
    assert not set(per) & H and set(per) <= every_sm - H, sorted(set(per) & H)
    assert r.cluster_sms == r.sms_covered == len(per) <= n - K and r.complete == 0 and 1 <= r.rounds <= 4
    assert r.ctas % cluster == 0 and r.ctas == sum(per.values()) and r.unpublished == 0
    assert tuple(r.fold[2]) == tuple(r.expect[2]) == barrier.fold(2, r.seed, cluster)
    print("barrier cluster %d under a hold: H %s, rounds %d, %d of the %d free SMs, %d CTAs"
          % (cluster, sorted(H), r.rounds, r.cluster_sms, n - K, r.ctas))
