"""The helper forms of the host link and compute probes (cro_probe_host_link_uuid, cro_probe_compute_uuid) on one H100,
against the C oracle and against the in-process forms with the same options.

Faults come only from the probes' software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import pytest

MASK = (1 << 64) - 1
MiB = 1 << 20
S = 256 * MiB
RAGGED = 3 * MiB + 112
STRIDE = 0xD1B54A32D192ED03
CHECK_PATTERN = [0, 0, 1, 2, 0]              # P1, P1, P2, P3, P1
REACHES = {0: {0, 1}, 1: {1}, 2: {2}, 3: {3}, 4: {4}}
HOST_BUFFER_CHECKS = {0, 2, 4}
LINK_MASK = (1 << 63) | (1 << 17) | 1
INT_MASK, FLOAT_MASK = 1 << 4, 1 << 30
ROW, COL = 77, 133

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def uuid(ctx):
    return ctx.own_devices()[0].gpu_uuid.decode()


@pytest.fixture(scope="module")
def minor(ctx):
    return ctx.own_devices()[0].device_minor


@pytest.fixture(scope="module")
def co(_built):
    import compute
    return compute.CComputeOracle()


@pytest.fixture(scope="module")
def covered(ctx):
    """The SMs of one clean in-process compute call, ascending: the first and last covered SM."""
    _, sms, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    return [s.smid for s in sms]


def device_seed(seed, offset):
    """seed_base | minor of a result's seed (offset: the probe's 2^62 or 2^61)."""
    return (seed - offset) & MASK


# ---- host link --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [64 * MiB, 0, RAGGED], ids=["64MiB", "default", "3MiB+112B"])
def test_link_clean_call(cro, coracle, ctx, uuid, minor, L):
    r, faults, ns = cro.probe_host_link_uuid(ctx, uuid, bytes=L)
    L = L or 256 * MiB
    n = L // 8
    assert r.status == cro.OK and r.first_fail == cro.LINK_NO_FAIL and faults == []
    assert r.bytes == L and r.call == 0
    dev = device_seed(r.seed[0], 1 << 62)
    assert dev & 0xFF == minor and list(r.seed) == [(dev + (1 << 62) + j * STRIDE) & MASK for j in range(3)]
    want = [coracle.checksum(r.seed[j], 0, n, threads=16) for j in range(3)]
    for k in range(cro.LINK_WORD_CHECKS):
        c = r.check[k]
        assert (c.words, c.mismatches, c.recorded, c.seed) == (n, 0, 0, r.seed[CHECK_PATTERN[k]]), k
        assert c.fold == want[CHECK_PATTERN[k]] and c.expect == want[CHECK_PATTERN[k]], k
    sm_legs = {cro.LINK_LEG_SM_H2D, cro.LINK_LEG_SM_D2H, cro.LINK_LEG_SM_DUPLEX_H2D, cro.LINK_LEG_SM_DUPLEX_D2H}
    for g in range(cro.LINK_LEGS):
        assert r.leg[g].bytes == L and r.leg[g].ns > 0 and (r.leg[g].timer_ns > 0) == (g in sm_legs), g
    assert r.chase_hops == 1024 and r.chase_end == r.chase_expect == coracle.chase_end(minor, minor, 1024) and r.chase_ns > 0
    assert ns > sum(r.leg[g].ns for g in range(cro.LINK_LEGS))
    print("link helper at L = %d: %.3f s spawn to exit, legs %.3f ms" % (L, ns / 1e9, sum(g.ns for g in r.leg) / 1e6))


@pytest.mark.parametrize("check", range(5))
@pytest.mark.parametrize("where", ["first", "last"])
def test_link_injection_reaches_the_checks_it_reaches_in_process(cro, coracle, ctx, uuid, check, where):
    L = 64 * MiB
    word = 0 if where == "first" else L // 8 - 1
    r, faults, _ = cro.probe_host_link_uuid(ctx, uuid, bytes=L, inject=(check, word, LINK_MASK))
    assert r.status == cro.ERR_CHECKSUM and r.first_fail == min(REACHES[check])
    assert {f.check for f in faults} == REACHES[check], [(f.check, f.word_index) for f in faults]
    for k in range(cro.LINK_WORD_CHECKS):
        assert r.check[k].mismatches == r.check[k].recorded == (1 if k in REACHES[check] else 0), k
    for f in faults:
        e = coracle.pattern_word(r.seed[CHECK_PATTERN[f.check]], word)
        assert (f.word_index, f.expected, f.actual) == (word, e, e ^ LINK_MASK), f.check
        assert f.host_value == (f.actual if check in HOST_BUFFER_CHECKS else f.expected), f.check


def test_link_path_and_nvml_agree_with_the_in_process_call(cro, ctx, uuid):
    a, _ = ctx.probe_host_link(0, bytes=16 * MiB)
    b, _, _ = cro.probe_host_link_uuid(ctx, uuid, bytes=16 * MiB)
    assert a.status == b.status == cro.OK
    hops = lambda r: [(r.path.hop[i].bdf, r.path.hop[i].max_speed, r.path.hop[i].max_width) for i in range(r.path.n_hops)]
    assert b.path.n_hops == a.path.n_hops and hops(b) == hops(a)
    assert (b.dev_numa, b.path.numa_node) == (a.dev_numa, a.path.numa_node)
    assert b.no_nvml == a.no_nvml
    if not b.no_nvml:
        assert b.replays_after >= b.replays_before


# ---- compute ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("iterations", [0, 1], ids=["default", "1"])
def test_compute_clean_call(cro, ctx, co, uuid, minor, iterations):
    import compute
    r, sms, faults, ns = cro.probe_compute_uuid(ctx, uuid, iterations=iterations)
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.COMPUTE_NONE and not faults and r.call == 0
    assert r.sm_count == n and r.legs == cro.COMPUTE_ALL_LEGS and r.bad_sms == 0 and r.host_ref_ns > 0
    # the helper runs without NVML: its minor comes from /proc, or is its CUDA ordinal 0 where /proc does not list the GPU
    assert device_seed(r.seed, 1 << 61) & 0xFF in (minor, 0)
    want = {0: co.answer(0, r.seed), 1: co.answer(1, r.seed)}
    for leg in range(cro.COMPUTE_LEGS):
        L = r.leg[leg]
        if iterations and leg < 3:
            assert L.iterations == iterations
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered)
        assert L.mismatches == L.fold_mismatches == L.recorded == L.failed_sms == 0
        assert L.fold == L.expect_fold == compute.cta_fold(want[compute.LEG_ANSWER[leg]], L.iterations), leg
        assert L.ns > 0 and L.timer_ns > 0
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    assert ns > sum(L.ns for L in r.leg)
    print("compute helper (iterations %d): %.3f s spawn to exit" % (r.leg[0].iterations, ns / 1e9))


@pytest.mark.parametrize("leg", range(5), ids=["s8", "bf16", "e4m3", "ffma", "imad"])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_compute_injection_names_what_the_in_process_form_names(cro, ctx, co, uuid, covered, leg, where, when):
    import compute
    smid = covered[0] if where == "first" else covered[-1]
    iteration = 2 if when == "last" else 1
    mask = FLOAT_MASK if leg in (cro.COMPUTE_LEG_BF16, cro.COMPUTE_LEG_E4M3, cro.COMPUTE_LEG_FFMA) else INT_MASK
    inj = (leg, smid, iteration, ROW, COL, mask)
    a = ctx.probe_compute(0, iterations=3, alu_iterations=3, inject=inj)
    b = cro.probe_compute_uuid(ctx, uuid, iterations=3, alu_iterations=3, inject=inj)[:3]
    named = []
    for r, sms, faults in (a, b):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.COMPUTE_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        (entry,) = [s for s in sms if s.smid == smid]
        assert r.leg[leg].failed_sms == 1 and r.leg[leg].fold_mismatches == entry.leg[leg].ctas
        named.append(([(lg, entry.leg[lg].mark) for lg in range(cro.COMPUTE_LEGS)],
                      sorted({(f.leg, f.smid, f.row, f.col) for f in faults})))
    assert named[0] == named[1]
    assert named[1][0][leg][1] == (cro.COMPUTE_PERSISTENT if when == "last" else cro.COMPUTE_INTERMITTENT)
    r, _, faults = b
    if when == "last":
        v = int(co.answer(compute.LEG_ANSWER[leg], r.seed)[ROW, COL])
        assert faults and all(f.expected == v and f.actual != v for f in faults)
    else:
        assert not faults


# ---- fresh seeds, the in-process GPU, refusals ------------------------------------------------------------------------
@pytest.mark.parametrize("with_ctx", [True, False], ids=["ctx", "no-ctx"])
def test_each_helper_call_uses_fresh_seeds(cro, ctx, uuid, with_ctx):
    c = ctx if with_ctx else None
    a, _, _ = cro.probe_host_link_uuid(c, uuid, bytes=MiB)
    b, _, _ = cro.probe_host_link_uuid(c, uuid, bytes=MiB)
    assert a.status == b.status == cro.OK and not set(a.seed) & set(b.seed)
    x = cro.probe_compute_uuid(c, uuid, iterations=1, alu_iterations=1)[0]
    y = cro.probe_compute_uuid(c, uuid, iterations=1, alu_iterations=1)[0]
    assert x.status == y.status == cro.OK and x.seed != y.seed
    if with_ctx:       # nor does a helper call repeat the context's own patterns
        own, _ = ctx.probe_host_link(0, bytes=MiB)
        assert not set(own.seed) & (set(a.seed) | set(b.seed))


@pytest.mark.parametrize("which", ["link", "compute"])
def test_a_probe_in_flight_is_collected_intact_and_both_halves_stay_known(cro, coracle, ctx, uuid, which):
    ctx.probe_begin(0)
    if which == "link":
        r = cro.probe_host_link_uuid(ctx, uuid, bytes=64 * MiB)[0]
    else:
        r = cro.probe_compute_uuid(ctx, uuid, iterations=1, alu_iterations=1)[0]
    assert r.status == cro.OK
    p = ctx.probe_end(0)
    assert p.status == cro.OK and p.checksum == coracle.checksum(p.seed, 0, S // 8, threads=16)
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == cro.OK and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


@pytest.mark.parametrize("kw", [dict(bytes=24), dict(hops=(1 << 24) + 1), dict(inject=(5, 0, 1)),
                                dict(bytes=MiB, inject=(0, MiB // 8, 1))], ids=["24B", "hops", "check5", "word-past-L"])
def test_bad_link_arguments_are_refused(cro, ctx, uuid, kw):
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_host_link_uuid(ctx, uuid, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG


@pytest.mark.parametrize("kw", [dict(legs=0x20), dict(iterations=65537), dict(max_rounds=65),
                                dict(inject=(0, 0, 3, 0, 0, 1), iterations=3)], ids=["legs", "iterations", "rounds", "iteration"])
def test_bad_compute_arguments_are_refused(cro, ctx, uuid, kw):
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_compute_uuid(ctx, uuid, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG


def test_a_gpu_the_node_does_not_list_is_no_device(cro, ctx):
    for call in (cro.probe_host_link_uuid, cro.probe_compute_uuid):
        with pytest.raises(cro.ProbeError) as e:
            call(ctx, "GPU-00000000-0000-0000-0000-0000000000ff")
        assert e.value.code == cro.ERR_NO_DEVICE
