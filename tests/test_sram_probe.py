"""The SRAM probe (cro_probe_sram, cro_probe_sram_uuid) on one H100, against the C oracle's checksums.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import collections
import json

import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
BIT = 1 << 37

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_sram(0)


def pattern(seed, w):
    z = (seed + w + 0x9E3779B97F4A7C15) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def check_clean(cro, ctx, coracle, r, sms, faults, iterations, legs=3):
    import sram
    n = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.SRAM_NONE and not faults, (r.status, r.verdict, faults[:4])
    assert r.sm_count == n and r.legs == legs and r.bad_sms == 0 and r.bad_pairs == 0
    n_words = r.bytes_per_sm // 8
    assert 200 << 10 <= r.bytes_per_sm <= 227 << 10 and n_words % 32 == 0
    if legs & 1:
        L = r.leg[cro.SRAM_SMEM]
        assert L.iterations == iterations and L.sms_covered == n and L.complete == 1 and L.unpublished == 0
        assert list(L.mismatches) == [0] * 6 and L.fold_mismatches == 0 and L.recorded == 0 and L.failed_sms == 0
        assert L.fold == L.expect == sram.m5_fold(coracle.checksum, r.seed, n_words, iterations)
        assert L.ns > 0 and L.timer_ns > 0 and L.bytes == 80 * n_words * iterations * L.ctas
        assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
        assert all(s.leg[0].ctas >= 1 and s.leg[0].mark == 0 and s.leg[0].cycles > 0 for s in sms)
    if legs & 2:
        L = r.leg[cro.SRAM_DSMEM]
        assert L.cluster in (2, 4, 8) and L.iterations == iterations and L.unpublished == 0 and L.rounds >= 1
        assert 0 < L.sms_covered <= n and L.complete == (L.sms_covered == n)
        assert list(L.mismatches) == [0] * 6 and L.recorded == 0 and L.failed_sms == 0
        assert L.bytes == 8 * n_words * iterations * (L.cluster + 2) * L.ctas and L.ctas % L.cluster == 0


def test_clean_default_call(cro, ctx, coracle, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, coracle, r, sms, faults, r.leg[0].iterations)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 60) + 8 * r.call * STRIDE) & MASK
    ann = json.loads(cro.emit_sram_annotations_json(r))
    assert ann["cohdi.io/probe-sram-verdict"] == "ok" and ann["cohdi.io/probe-sram-bytes-per-sm"] == str(r.bytes_per_sm)
    print("SRAM clean default: %d B/SM, local %d SMs in %d rounds, network %d/%d SMs in %d rounds" % (
        r.bytes_per_sm, r.leg[0].sms_covered, r.leg[0].rounds, r.leg[1].sms_covered, r.sm_count, r.leg[1].rounds))


@pytest.mark.parametrize("iterations", [1, 4096])
def test_clean_call_at_other_iteration_counts(cro, ctx, coracle, iterations):
    r, sms, faults = ctx.probe_sram(0, iterations=iterations)
    check_clean(cro, ctx, coracle, r, sms, faults, iterations)


@pytest.mark.parametrize("cluster", [2, 4, 8])
def test_network_leg_runs_clean_at_each_cluster_size(cro, ctx, coracle, cluster):
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_DSMEM, iterations=2, cluster=cluster)
    check_clean(cro, ctx, coracle, r, sms, faults, 2, legs=2)
    assert r.leg[1].cluster == cluster
    print("cluster %d: %d/%d SMs covered in %d rounds" % (cluster, r.leg[1].sms_covered, r.sm_count, r.leg[1].rounds))


def test_second_call_uses_a_new_seed(ctx):
    a, _, _ = ctx.probe_sram(0, iterations=1)
    b, _, _ = ctx.probe_sram(0, iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + 8 * STRIDE) & MASK and a.status == b.status == 0


def expected_word(seed, element, w):
    p = pattern(seed, w)
    return p if element in (1, 3, 5) else p ^ MASK


@pytest.mark.parametrize("element", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("word", ["first", "middle", "last"])
@pytest.mark.parametrize("when", ["last", "middle"])
def test_local_injection_names_the_sm_the_element_and_the_word(cro, ctx, clean, element, where, word, when):
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    n_words = clean[0].bytes_per_sm // 8
    w = {"first": 0, "middle": n_words // 2 + 3, "last": n_words - 1}[word]
    iteration = 2 if when == "last" else 1
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=3,
                                    inject=(cro.SRAM_SMEM, smid, element, iteration, w, BIT))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_SM
    assert r.bad_sms == 1 and r.bad_sm[0] == smid and r.bad_pairs == 0
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[0].ctas
    assert ctas >= 1
    L = r.leg[0]
    assert L.failed_sms == 1 and L.recorded == ctas
    assert list(L.mismatches) == [ctas if e == element else 0 for e in range(6)]
    assert list(entry.leg[0].mismatches) == list(L.mismatches)
    assert L.fold_mismatches == entry.leg[0].fold_mismatches == (ctas if element == 5 else 0)
    assert entry.leg[0].mark == (cro.SRAM_PERSISTENT if when == "last" else cro.SRAM_INTERMITTENT)
    for s in sms:
        if s.smid != smid:
            assert s.leg[0].mark == 0 and sum(s.leg[0].mismatches) == 0 and s.leg[0].fold_mismatches == 0
    e = expected_word(r.seed, element, w)
    assert [(f.leg, f.element, f.iteration, f.smid, f.peer_smid, f.direction, f.word, f.expected, f.actual) for f in faults] == \
        [(cro.SRAM_SMEM, element, iteration, smid, smid, cro.SRAM_DIR_LOCAL, w, e, e ^ BIT)] * ctas
    ann = json.loads(cro.emit_sram_annotations_json(r))
    assert ann["cohdi.io/probe-sram-verdict"] == "sm" and ann["cohdi.io/probe-sram-bad-sms"] == str(smid)


def network_target(clean):
    """The lowest SM that took part in a cluster of the clean call."""
    return min(s.smid for s in clean[1] if s.leg[1].ctas)


def test_network_read_injection_names_the_reader_and_owner(cro, ctx, clean):
    smid, w = network_target(clean), 1000
    r, sms, faults = ctx.probe_sram(0, iterations=2, cluster=2, inject=(cro.SRAM_DSMEM, smid, 1, 1, w, BIT))
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[1].ctas
    assert ctas >= 1, "the target SM took part in no cluster of this call"
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_LINK and r.bad_sms == 0
    L = r.leg[1]
    assert list(L.mismatches) == [0, ctas, 0, 0, 0, 0] and L.recorded == ctas and r.leg[0].failed_sms == 0
    assert all(f.leg == 1 and f.element == 1 and f.smid == smid and f.direction == cro.SRAM_DIR_READ and f.word == w and
               f.iteration == 1 and f.peer_smid != smid and f.actual == f.expected ^ BIT for f in faults) and len(faults) == ctas
    owners = sorted({f.peer_smid for f in faults})
    assert all(any(s.smid == o and s.leg[1].ctas for s in sms) for o in owners)
    for f in faults:                                                   # the owner's pattern: its rank's seed
        assert f.expected in [pattern((r.seed + rank * STRIDE) & MASK, w) for rank in (0, 1)]
    assert [(p.from_, p.owner, p.direction) for p in r.bad_pair[:r.bad_pairs]] == [(smid, o, cro.SRAM_DIR_READ) for o in owners]
    ann = json.loads(cro.emit_sram_annotations_json(r))
    assert ann["cohdi.io/probe-sram-verdict"] == "link"
    assert ann["cohdi.io/probe-sram-bad-pairs"] == ",".join("%d-%d:r" % (smid, o) for o in owners)


def test_network_write_injection_names_the_writer_and_owner(cro, ctx, clean):
    smid, w = network_target(clean), 77
    r, sms, faults = ctx.probe_sram(0, iterations=2, cluster=2, inject=(cro.SRAM_DSMEM, smid, 2, 0, w, BIT))
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[1].ctas
    assert ctas >= 1, "the target SM took part in no cluster of this call"
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_LINK and r.bad_sms == 0
    assert list(r.leg[1].mismatches) == [0, 0, 0, ctas, 0, 0] and len(faults) == ctas
    assert all(f.element == 3 and f.peer_smid == smid and f.smid != smid and f.direction == cro.SRAM_DIR_WRITE and
               f.word == w and f.iteration == 0 and f.actual == f.expected ^ BIT for f in faults)
    owners = sorted({f.smid for f in faults})
    assert [(p.from_, p.owner, p.direction) for p in r.bad_pair[:r.bad_pairs]] == [(smid, o, cro.SRAM_DIR_WRITE) for o in owners]
    assert json.loads(cro.emit_sram_annotations_json(r))["cohdi.io/probe-sram-bad-pairs"] == \
        ",".join("%d-%d:w" % (smid, o) for o in owners)


def multi_round_target(cro, ctx, cluster):
    """A clean network call at this cluster size, and the SM that ran the most of its CTAs (at least two, so some of
    its records come from rounds after the first)."""
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_DSMEM, iterations=2, cluster=cluster)
    assert r.status == cro.OK and not faults
    target = max(sms, key=lambda s: (s.leg[1].ctas, -s.smid))
    print("cluster %d: %d/%d SMs covered in %d rounds; SM %d ran %d network CTAs" % (
        cluster, r.leg[1].sms_covered, r.sm_count, r.leg[1].rounds, target.smid, target.leg[1].ctas))
    assert r.leg[1].rounds >= 2 and target.leg[1].ctas >= 2, "every SM ran one network CTA at this cluster size"
    return target.smid


def network_sms(sms):
    return {s.smid for s in sms if s.leg[1].ctas}


@pytest.mark.parametrize("cluster", [4, 8])
def test_network_read_injection_over_several_rounds(cro, ctx, cluster):
    """D1 of every network CTA on the target reads word w of each of its C - 1 peers wrong: each record names the
    owner that the record's own round placed at peer_block."""
    smid, w = multi_round_target(cro, ctx, cluster), 513
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_DSMEM, iterations=2, cluster=cluster,
                                    inject=(cro.SRAM_DSMEM, smid, 1, 1, w, BIT))
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[1].ctas
    print("cluster %d read injection: SM %d ran %d network CTAs in %d rounds" % (cluster, smid, ctas, r.leg[1].rounds))
    assert ctas >= 1 and r.leg[1].unpublished == 0
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_LINK and r.bad_sms == 0
    L = r.leg[1]
    assert list(L.mismatches) == [0, (cluster - 1) * ctas, 0, 0, 0, 0] and L.recorded == len(faults) == (cluster - 1) * ctas
    ranks = collections.Counter()
    for f in faults:
        assert (f.leg, f.element, f.direction, f.smid, f.word, f.iteration) == (1, 1, cro.SRAM_DIR_READ, smid, w, 1)
        assert f.peer_smid != smid and f.peer_smid in network_sms(sms) and f.actual == f.expected ^ BIT
        (rank,) = [q for q in range(cluster) if pattern((r.seed + q * STRIDE) & MASK, w) == f.expected]
        ranks[rank] += 1
    assert max(ranks.values()) <= ctas and len(ranks) >= cluster - 1
    owners = sorted({f.peer_smid for f in faults})
    assert r.bad_pairs == len(owners)
    assert [(p.from_, p.owner, p.direction) for p in r.bad_pair[:min(r.bad_pairs, cro.SRAM_MAX_PAIRS)]] == \
        [(smid, o, cro.SRAM_DIR_READ) for o in owners][:cro.SRAM_MAX_PAIRS]
    assert json.loads(cro.emit_sram_annotations_json(r))["cohdi.io/probe-sram-verdict"] == "link"


@pytest.mark.parametrize("cluster", [4, 8])
def test_network_write_injection_over_several_rounds(cro, ctx, cluster):
    """D2 of every network CTA on the target writes word w of its next peer wrong; that peer's D3 finds it and names
    its previous rank's SM, resolved through the record's own round, as the writer."""
    smid, w = multi_round_target(cro, ctx, cluster), 2047
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_DSMEM, iterations=2, cluster=cluster,
                                    inject=(cro.SRAM_DSMEM, smid, 2, 0, w, BIT))
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[1].ctas
    print("cluster %d write injection: SM %d ran %d network CTAs in %d rounds" % (cluster, smid, ctas, r.leg[1].rounds))
    assert ctas >= 1 and r.leg[1].unpublished == 0
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_LINK and r.bad_sms == 0
    assert list(r.leg[1].mismatches) == [0, 0, 0, ctas, 0, 0] and len(faults) == ctas
    for f in faults:
        assert (f.leg, f.element, f.direction, f.peer_smid, f.word, f.iteration) == (1, 3, cro.SRAM_DIR_WRITE, smid, w, 0)
        assert f.smid != smid and f.smid in network_sms(sms) and f.actual == f.expected ^ BIT
        assert any(f.expected == pattern((r.seed + q * STRIDE) & MASK, w) ^ MASK for q in range(cluster))
    owners = sorted({f.smid for f in faults})
    assert r.bad_pairs == len(owners)
    assert [(p.from_, p.owner, p.direction) for p in r.bad_pair[:min(r.bad_pairs, cro.SRAM_MAX_PAIRS)]] == \
        [(smid, o, cro.SRAM_DIR_WRITE) for o in owners][:cro.SRAM_MAX_PAIRS]


def test_injection_into_every_sm_is_a_common_cause(cro, ctx):
    r, sms, _ = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=2, inject=(cro.SRAM_SMEM, -1, 3, 0, 7, BIT))
    L = r.leg[0]
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_ALL
    assert L.failed_sms == L.sms_covered == len(sms) and L.mismatches[3] == L.ctas and r.bad_sms == len(sms)
    assert json.loads(cro.emit_sram_annotations_json(r))["cohdi.io/probe-sram-verdict"] == "all"


def test_injection_into_every_word_counts_exactly(cro, ctx, clean):
    smid = clean[1][0].smid
    r, sms, faults = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=2, inject=(cro.SRAM_SMEM, smid, 2, 1, -1, BIT),
                                    cap=cro.SRAM_RECORDS + 16)
    (entry,) = [s for s in sms if s.smid == smid]
    n_words = r.bytes_per_sm // 8
    L = r.leg[0]
    assert r.verdict == cro.SRAM_SM and L.mismatches[2] == n_words * entry.leg[0].ctas and sum(L.mismatches) == L.mismatches[2]
    assert L.recorded == cro.SRAM_RECORDS and len(faults) == cro.SRAM_RECORDS and r.recorded == cro.SRAM_RECORDS
    for f in faults[:64]:
        assert f.smid == smid and f.element == 2 and f.expected == expected_word(r.seed, 2, f.word) and f.actual == f.expected ^ BIT


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_sram(0, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_sram(0, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, coracle, clean):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_sram_uuid(ctx, uuid, iterations=2)
    check_clean(cro, ctx, coracle, r, sms, faults, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    smid = clean[1][-1].smid
    inj = (cro.SRAM_SMEM, smid, 4, 1, 123, BIT)
    a = ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=2, inject=inj)
    b = cro.probe_sram_uuid(None, uuid, legs=cro.SRAM_LEG_SMEM, iterations=2, inject=inj)
    for r, sms, faults in (a, b):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
        assert {(f.element, f.iteration, f.smid, f.word, f.expected ^ f.actual) for f in faults} == {(4, 1, smid, 123, BIT)}
    assert a[0].bytes_per_sm == b[0].bytes_per_sm


def test_nvml_fields_equal_a_read_right_after(cro, ctx):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, _, _ = ctx.probe_sram(0, iterations=1)
    h = cro.read_sram_health(uuid)
    assert (r.after.nvml, r.after.threshold_exceeded, r.after.ecc_corrected, r.after.ecc_uncorrected) == \
        (h.nvml, h.threshold_exceeded, h.ecc_corrected, h.ecc_uncorrected)
    assert r.before.nvml == h.nvml & ~cro.SRAM_NVML_STATUS
    ann = json.loads(cro.emit_sram_annotations_json(r))
    if h.nvml & cro.SRAM_NVML_ECC_CORRECTED:
        assert ann["cohdi.io/probe-sram-ecc-corrected"] == str(r.after.ecc_corrected - r.before.ecc_corrected)
    print("SRAM health: nvml %d, threshold %d, corrected %d, uncorrected %d" % (h.nvml, h.threshold_exceeded, h.ecc_corrected,
                                                                                h.ecc_uncorrected))


def test_invalid_arguments_are_refused(cro, ctx, clean):
    n_words = clean[0].bytes_per_sm // 8
    calls = [dict(legs=4), dict(iterations=cro.SRAM_MAX_ITERATIONS + 1), dict(cluster=3), dict(cluster=16),
             dict(max_rounds=cro.SRAM_MAX_ROUNDS + 1), dict(inject=(2, 0, 1, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 0, 1)),
             dict(inject=(0, 0, 6, 0, 0, 1)), dict(inject=(1, 0, 3, 0, 0, 1)), dict(inject=(0, 256, 1, 0, 0, 1)),
             dict(inject=(0, 0, 1, 3, 0, 1), iterations=3), dict(inject=(0, 0, 1, 0, n_words, 1)),
             dict(inject=(0, 0, 1, 0, -2, 1)), dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_sram(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
