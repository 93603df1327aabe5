"""The health check (cro_check_health_uuid, cro_check_health) on one H100: every check's clean-call assertions against
the C oracle, each check's seeds on its seed-space formula, one software injection per check failing exactly that check
with the fault its own helper form names, and the in-process form agreeing with the helper.

Faults come only from the probes' software injection (test_inject_* / test_force_*); nothing here provokes a CUDA
error or repeats a call to catch a real fault."""
import pytest

from test_compute_probe import check_clean as compute_clean
from test_hbm_scan import check_clean as scan_clean
from test_l2_probe import check_clean as l2_clean
from test_precision_probe import check_clean as precision_clean
from test_sram_probe import check_clean as sram_clean

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1
MiB, GiB = 1 << 20, 1 << 30
STRIDE = 0xD1B54A32D192ED03
CLEAN_SCAN = 4 * GiB                 # the clean call's scan: two default chunks
SMALL_SCAN = 256 * MiB               # the injection calls' scan
LINK_L = 64 * MiB
CHECK_PATTERN = [0, 0, 1, 2, 0]


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=256 * MiB, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def uuid(ctx):
    return ctx.own_devices()[0].gpu_uuid.decode()


@pytest.fixture(scope="module")
def co(_built):
    import compute
    return compute.CComputeOracle()


@pytest.fixture(scope="module")
def scan_oracle(_built):
    import scan
    return scan


@pytest.fixture(scope="module")
def clean(cro, ctx, uuid):
    return cro.check_health_uuid(ctx, uuid, scan=dict(max_bytes=CLEAN_SCAN))


@pytest.fixture(scope="module")
def covered(ctx):
    _, sms, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1)
    return [s.smid for s in sms]


def check_link_clean(cro, coracle, r, faults, L):
    n = L // 8
    assert r.status == cro.OK and r.first_fail == cro.LINK_NO_FAIL and not faults and r.bytes == L and r.call == 0
    want = [coracle.checksum(r.seed[j], 0, n, threads=16) for j in range(3)]
    for k in range(cro.LINK_WORD_CHECKS):
        c = r.check[k]
        assert (c.words, c.mismatches, c.recorded, c.seed) == (n, 0, 0, r.seed[CHECK_PATTERN[k]]), k
        assert c.fold == want[CHECK_PATTERN[k]] and c.expect == want[CHECK_PATTERN[k]], k
    assert r.chase_end == r.chase_expect == coracle.chase_end(r.chase_minor, r.chase_minor, r.chase_hops)


def seeds(r):
    """Every seed a health result reports, by check (the scan's is its own option's, or the clock's)."""
    return {"compute": {r.compute.seed}, "precision": {r.precision.seed}, "sram": {r.sram.seed},
            "l2": {r.l2.seed, r.l2.seed_atomic}, "link": set(r.link.seed)}


def test_clean_default_call(cro, ctx, coracle, co, scan_oracle, clean):
    r, rec, ns = clean
    assert r.status == cro.OK and r.ran == cro.HEALTH_ALL and r.checks == cro.HEALTH_ALL
    assert r.failed == r.errored == r.not_run == r.incomplete == 0 and list(r.check_status) == [0] * 6
    assert all(r.check_ns) and ns == r.helper_ns > sum(r.check_ns)
    compute_clean(cro, ctx, co, r.compute, rec["compute_sms"], rec["compute_faults"], r.compute.leg[0].iterations,
                  r.compute.leg[cro.COMPUTE_LEG_FFMA].iterations)
    precision_clean(cro, ctx, r.precision, rec["precision_sms"], rec["precision_faults"], r.precision.leg[0].iterations,
                    r.precision.leg[cro.PRECISION_LEG_DFMA].iterations)
    sram_clean(cro, ctx, coracle, r.sram, rec["sram_sms"], rec["sram_faults"], r.sram.leg[0].iterations)
    l2_clean(cro, ctx, coracle, r.l2, rec["l2_sms"], rec["l2_faults"], r.l2.bytes, r.l2.iterations)
    check_link_clean(cro, coracle, r.link, rec["link_faults"], 256 * MiB)
    scan_clean(cro, coracle, scan_oracle, r.scan, rec["scan_words"], CLEAN_SCAN, cro.SCAN_CHUNK_BYTES)
    for name in cro.HEALTH_NAMES:
        assert getattr(r, name).status == cro.OK, name
    print("health helper: %.3f s spawn to exit, checks %s ms" % (ns / 1e9, ", ".join(
        "%s %.1f" % (n, t / 1e6) for n, t in zip(cro.HEALTH_NAMES, r.check_ns))))


def test_every_seed_is_its_seed_space_formula(cro, ctx, clean):
    r = clean[0]
    dev = r.seed_base | ctx.own_devices()[0].device_minor
    assert r.seed_base & 0xFF == 0 and r.seed_base != 0
    assert r.compute.seed == (dev + (1 << 61)) & MASK
    assert r.precision.seed == (dev + (1 << 58)) & MASK
    assert r.sram.seed == (dev + (1 << 60)) & MASK
    assert (r.l2.seed, r.l2.seed_atomic) == ((dev + (1 << 59)) & MASK, (dev + (1 << 59) + STRIDE) & MASK)
    assert list(r.link.seed) == [(dev + (1 << 62) + j * STRIDE) & MASK for j in range(3)]
    assert r.compute.call == r.precision.call == r.sram.call == r.l2.call == r.link.call == 0


@pytest.mark.parametrize("with_ctx", [True, False], ids=["ctx", "no-ctx"])
def test_two_calls_share_no_seed(cro, ctx, uuid, with_ctx):
    c = ctx if with_ctx else None
    kw = dict(checks=cro.HEALTH_ALL & ~cro.HEALTH_SCAN, link=dict(bytes=MiB))
    a, _, _ = cro.check_health_uuid(c, uuid, **kw)
    b, _, _ = cro.check_health_uuid(c, uuid, **kw)
    assert a.status == b.status == cro.OK and a.seed_base != b.seed_base
    sa, sb = set().union(*seeds(a).values()), set().union(*seeds(b).values())
    assert len(sa) == 8 and not sa & sb


def identity(name, scan_rep, rec):
    """What a failed check names: (leg, SM, row, col), (leg, element, SM, word), (element, reader CTA, word), (check,
    word), (chunk, offset).  The L2 reader's SM is left out: which SM runs a CTA differs between processes."""
    if name in ("compute", "precision"):
        return sorted({(f.leg, f.smid, f.row, f.col) for f in rec[name + "_faults"]})
    if name == "sram":
        return sorted({(f.leg, f.element, f.smid, f.word) for f in rec["sram_faults"]})
    if name == "l2":
        return sorted({(f.element, f.cta, f.word) for f in rec["l2_faults"]})
    if name == "link":
        return sorted({(f.check, f.word_index) for f in rec["link_faults"]})
    return sorted({(w.reserved, w.word_index - scan_rep.chunk[w.reserved].word0) for w in rec["scan_words"]})


def single(cro, ctx, uuid, name, opts):
    """The same check through its own helper form, as (result, records by list name)."""
    if name == "compute":
        r, sms, f, _ = cro.probe_compute_uuid(ctx, uuid, **opts)
        return r, {"compute_faults": f}
    if name == "precision":
        r, sms, f, _ = cro.probe_precision_uuid(ctx, uuid, **opts)
        return r, {"precision_faults": f}
    if name == "sram":
        r, sms, f = cro.probe_sram_uuid(ctx, uuid, **opts)
        return r, {"sram_faults": f}
    if name == "l2":
        r, sms, f = cro.probe_l2_uuid(ctx, uuid, **opts)
        return r, {"l2_faults": f}
    if name == "link":
        r, f, _ = cro.probe_host_link_uuid(ctx, uuid, **opts)
        return r, {"link_faults": f}
    r, w = cro.scan_hbm_uuid(ctx, uuid, **opts)
    return r, {"scan_words": w}


def injections(cro, covered):
    sm = covered[-1]
    return {
        "compute": dict(iterations=3, alu_iterations=3, inject=(cro.COMPUTE_LEG_S8, sm, 2, 77, 133, 1 << 4)),
        "precision": dict(iterations=3, alu_iterations=3, inject=(cro.PRECISION_LEG_F64, sm, 2, 5, 9, 1 << 40)),
        "sram": dict(iterations=2, inject=(cro.SRAM_SMEM, sm, 3, 1, 1234, 1 << 33)),
        "l2": dict(iterations=2, inject=(cro.L2_MARCH, -1, 2, 1, 4097, 1 << 21)),
        "link": dict(bytes=LINK_L, inject=(1, 4321, 1 << 45)),
        "scan": dict(max_bytes=SMALL_SCAN, chunk_bytes=96 * MiB, seed=0x5CA9, force=(12345 * 8 + 3, 1, MASK ^ (1 << 6), 0)),
    }


def bounded(name, opts):
    """The options the other checks of an injection call run with: small and quick, all clean."""
    base = {"compute": dict(iterations=3, alu_iterations=3), "precision": dict(iterations=3, alu_iterations=3),
            "sram": dict(iterations=2), "l2": dict(iterations=2), "link": dict(bytes=LINK_L),
            "scan": dict(max_bytes=SMALL_SCAN, chunk_bytes=96 * MiB)}
    base[name] = opts
    return base


@pytest.mark.parametrize("name", ["compute", "precision", "sram", "l2", "link", "scan"])
def test_one_injection_fails_exactly_that_check(cro, ctx, uuid, covered, name):
    inj = injections(cro, covered)
    r, rec, _ = cro.check_health_uuid(ctx, uuid, **bounded(name, inj[name]))
    bit = 1 << cro.HEALTH_NAMES.index(name)
    assert r.status == cro.ERR_CHECKSUM and r.failed == bit and r.errored == 0 and r.ran == cro.HEALTH_ALL, (r.failed, r.errored)
    assert [getattr(r, n).status for n in cro.HEALTH_NAMES] == [cro.ERR_CHECKSUM if n == name else cro.OK for n in cro.HEALTH_NAMES]
    alone, alone_rec = single(cro, ctx, uuid, name, inj[name])
    assert alone.status == cro.ERR_CHECKSUM
    got, want = identity(name, r.scan, rec), identity(name, alone, alone_rec)
    assert got and got == want, (got, want)
    import json
    m = json.loads(cro.emit_health_annotations_json(r))
    assert m["cohdi.io/probe-health-verdict"] == "fail" and m["cohdi.io/probe-health-failed"] == name


def test_two_injections_are_both_failed(cro, ctx, uuid, covered):
    import json
    inj = injections(cro, covered)
    opts = bounded("sram", inj["sram"])
    opts["link"] = inj["link"]
    r, _, _ = cro.check_health_uuid(ctx, uuid, **opts)
    assert r.status == cro.ERR_CHECKSUM and r.failed == cro.HEALTH_SRAM | cro.HEALTH_LINK
    assert json.loads(cro.emit_health_annotations_json(r))["cohdi.io/probe-health-failed"] == "sram,link"


def test_a_subset_runs_only_the_selected_checks(cro, ctx, uuid):
    checks = cro.HEALTH_PRECISION | cro.HEALTH_LINK
    r, rec, _ = cro.check_health_uuid(ctx, uuid, checks=checks, precision=dict(iterations=1, alu_iterations=1),
                                      link=dict(bytes=MiB))
    assert r.status == cro.OK and r.ran == checks and r.not_run == 0
    assert r.compute.sm_count == 0 and r.scan.covered_bytes == 0 and r.check_ns[0] == 0 and r.check_ns[5] == 0
    assert r.precision.sm_count > 0 and r.link.bytes == MiB


def test_in_process_agrees_with_the_helper(cro, ctx, uuid, covered):
    inj = injections(cro, covered)
    a, arec = ctx.check_health(0, **bounded("compute", dict(iterations=3, alu_iterations=3)))
    assert a.status == cro.OK and a.ran == cro.HEALTH_ALL and a.helper_ns == 0 and a.failed == a.errored == 0
    for name in ("compute", "l2", "link"):
        x, xrec = ctx.check_health(0, **bounded(name, inj[name]))
        y, yrec, _ = cro.check_health_uuid(ctx, uuid, **bounded(name, inj[name]))
        assert x.failed == y.failed == 1 << cro.HEALTH_NAMES.index(name) and x.status == y.status == cro.ERR_CHECKSUM
        assert identity(name, x.scan, xrec) == identity(name, y.scan, yrec), name


def test_a_probe_in_flight_stays_collectable_and_both_halves_stay_known(cro, coracle, ctx, uuid):
    ctx.probe_begin(0)
    r, _, _ = cro.check_health_uuid(ctx, uuid, **bounded("link", dict(bytes=LINK_L)))
    assert r.status == cro.OK
    p = ctx.probe_end(0)
    assert p.status == cro.OK and p.checksum == coracle.checksum(p.seed, 0, (256 * MiB) // 8, threads=16)
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == cro.OK and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_a_gpu_the_node_does_not_list_is_no_device(cro, ctx):
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(ctx, "GPU-00000000-0000-0000-0000-0000000000ff")
    assert e.value.code == cro.ERR_NO_DEVICE
