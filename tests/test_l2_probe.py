"""The L2 probe (cro_probe_l2) on one H100, against oracle/l2.py and the C oracle's checksums.

Faults come only from the probe's software injection (test_inject_*); nothing here repeats a call to catch a real one."""
import ctypes
import json

import pytest

MASK = (1 << 64) - 1
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
BIT = 1 << 41
MIB = 1 << 20

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def clean(ctx):
    """One clean default call: the SMs it saw give the first and last covered SM."""
    return ctx.probe_l2(0)


def check_clean(cro, ctx, coracle, r, sms, faults, nbytes, iterations):
    import l2
    G = ctx.own_devices()[0].sm_count
    assert r.status == cro.OK and r.verdict == cro.L2_NONE and not faults, (r.status, r.verdict, faults[:4])
    assert r.bytes == nbytes and r.iterations == iterations and r.ctas == r.sm_count == G and r.delta == l2.delta(G)
    assert r.blocks == nbytes // cro.L2_BLOCK_BYTES and r.unpublished == 0 and r.overflow == 0
    assert list(r.mismatches) == [0] * 6 and r.bad_sms == r.bad_lines == 0
    assert r.sms_covered == sum(1 for s in sms if any(s.words_read)) and 0 < r.sms_covered <= len(sms) <= G <= r.nsmid
    assert sum(s.launches for s in sms) == 6 * iterations * G                          # every CTA of every launch published
    assert r.fold_ok == 1 and r.fold == r.expect == l2.m5_fold(coracle.checksum, r.seed, nbytes // 8, iterations)
    assert r.a1_bad == 0 and r.a2_bad == 0 and r.a2_holes == 0 and r.a2_tickets == 32 * G
    for e in range(1, 6):                                   # the rotation hands every word to exactly one reader per element
        assert sum(s.words_read[e] for s in sms) == iterations * nbytes // 8
    assert r.march_bytes == 10 * nbytes * iterations and r.march_ns > 0 and all(r.element_ns)
    assert r.a1_ns > 0 and r.a1_check_ns > 0 and r.a2_ns > 0 and r.a2_check_ns > 0 and r.wall_ns > r.march_ns


def test_clean_default_call(cro, ctx, coracle, clean):
    r, sms, faults = clean
    check_clean(cro, ctx, coracle, r, sms, faults, r.bytes, r.iterations)
    dev = SEED_BASE | ctx.own_devices()[0].device_minor
    assert r.seed == (dev + (1 << 59) + 2 * r.call * STRIDE) & MASK and r.seed_atomic == (r.seed + STRIDE) & MASK
    assert r.bytes % cro.L2_BLOCK_BYTES == 0 and r.bytes <= 8 * r.l2_bytes
    ann = json.loads(cro.emit_l2_annotations_json(r))
    assert ann["cohdi.io/probe-l2-verdict"] == "ok" and ann["cohdi.io/probe-l2-bytes"] == str(r.bytes)
    print("L2 clean default: W %d B, %d iterations, L2 %d B, %d SMs, march %.1f GB/s, wall %.2f ms" % (
        r.bytes, r.iterations, r.l2_bytes, r.sms_covered, r.march_bytes / r.march_ns, r.wall_ns / 1e6))


def l2_size_bytes(clean):
    return clean[0].l2_bytes // 16384 * 16384


@pytest.mark.parametrize("size", ["min", "l2", "ragged"])
@pytest.mark.parametrize("iterations", [1, 64])
def test_clean_call_at_other_sizes(cro, ctx, coracle, clean, size, iterations):
    G = clean[0].ctas
    nbytes = {"min": cro.L2_MIN_BYTES, "l2": l2_size_bytes(clean), "ragged": (7 * G + 3) * cro.L2_BLOCK_BYTES}[size]
    r, sms, faults = ctx.probe_l2(0, bytes=nbytes, iterations=iterations)
    check_clean(cro, ctx, coracle, r, sms, faults, nbytes, iterations)


def test_second_call_uses_new_seeds(ctx):
    a, _, _ = ctx.probe_l2(0, bytes=4 * MIB, iterations=1)
    b, _, _ = ctx.probe_l2(0, bytes=4 * MIB, iterations=1)
    assert b.call == a.call + 1 and b.seed == (a.seed + 2 * STRIDE) & MASK and a.status == b.status == 0


W4 = 4 * MIB


@pytest.mark.parametrize("element", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("word", ["first", "middle", "last"])
def test_one_word_injection_names_its_reader(cro, ctx, element, word):
    import l2
    n = W4 // 8
    w = {"first": 0, "middle": n // 2 + 5, "last": n - 1}[word]
    r, sms, faults = ctx.probe_l2(0, bytes=W4, iterations=2, inject=(cro.L2_MARCH, -1, element, 1, w, BIT))
    G = r.ctas
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and r.bad_lines == 0
    assert list(r.mismatches) == [1 if e == element else 0 for e in range(6)]
    (f,) = faults
    b = w // l2.BLOCK_WORDS
    assert (f.element, f.iteration, f.word, f.cta, f.writer_cta) == (element, 1, w, l2.owner(b, element, G), l2.owner(b, element - 1, G))
    assert f.expected == l2.expected_read(r.seed, element, w) and f.actual == f.expected ^ BIT and f.line == 0
    assert r.bad_sms == 1 and r.bad_sm[0] == f.smid and f.writer_smid != 0xFFFFFFFF
    (entry,) = [s for s in sms if s.smid == f.smid]
    assert entry.mark == cro.L2_PERSISTENT and entry.mismatches[element] == 1
    assert json.loads(cro.emit_l2_annotations_json(r))["cohdi.io/probe-l2-bad-sms"] == str(f.smid)


@pytest.mark.parametrize("element", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("where", ["first", "last"])
def test_every_word_injection_counts_what_the_sm_read(cro, ctx, clean, element, where):
    import l2
    smid = clean[1][0].smid if where == "first" else clean[1][-1].smid
    r, sms, faults = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(cro.L2_MARCH, smid, element, 0, -1, BIT),
                                  cap=cro.L2_RECORDS)
    (entry,) = [s for s in sms if s.smid == smid]
    assert entry.words_read[element] > 0, "the SM read nothing in this element"
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and list(r.bad_sm[:r.bad_sms]) == [smid]
    assert r.mismatches[element] == sum(r.mismatches) == entry.mismatches[element] == entry.words_read[element]
    ctas = {f.cta for f in faults}
    assert sum(l2.words_read(c, element, r.blocks, r.ctas) for c in ctas) == r.mismatches[element]
    assert all(f.smid == smid and f.element == element and f.actual == f.expected ^ BIT and
               f.expected == l2.expected_read(r.seed, element, f.word) and f.cta == l2.owner(f.word // l2.BLOCK_WORDS, element, r.ctas)
               for f in faults)
    assert entry.mark == cro.L2_PERSISTENT


def test_a_word_every_reader_saw_wrong_is_a_line(cro, ctx):
    w = 12345
    r, sms, faults = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(cro.L2_MARCH, -1, -1, 0, w, BIT))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_LINE
    assert r.bad_lines == 1 and r.bad_line[0] == 8 * w and r.bad_sms == 0
    assert list(r.mismatches) == [0, 1, 1, 1, 1, 1] and len(faults) == 5 and all(f.line == 1 and f.word == w for f in faults)
    assert len({f.cta for f in faults}) == 5
    assert json.loads(cro.emit_l2_annotations_json(r))["cohdi.io/probe-l2-bad-lines"] == str(8 * w)


@pytest.mark.parametrize("counter", [0, 777, 65535])
def test_a1_injection_names_the_counter(cro, ctx, counter):
    r, _, faults = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(cro.L2_A1, -1, 0, 0, counter, BIT))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ATOMIC and not faults
    assert r.a1_bad == 1 and r.a1_bad_counter[0] == counter and r.a2_bad == 0
    assert json.loads(cro.emit_l2_annotations_json(r))["cohdi.io/probe-l2-a1-bad-counters"] == str(counter)


@pytest.mark.parametrize("counter,mask", [(0, 1), (511, 1 << 20), (1023, 3)])
def test_a2_injection_leaves_exactly_one_hole(cro, ctx, counter, mask):
    r, _, _ = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(cro.L2_A2, -1, 0, 0, counter, mask))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ATOMIC
    assert r.a2_holes == 1 and r.a2_bad == 1 and r.a2_bad_counter[0] == counter and r.a1_bad == 0
    assert json.loads(cro.emit_l2_annotations_json(r))["cohdi.io/probe-l2-a2-holes"] == "1"


def test_every_sm_every_word_is_all_with_exact_counts(cro, ctx):
    r, sms, faults = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(cro.L2_MARCH, -1, 2, 0, -1, BIT), cap=cro.L2_RECORDS + 16)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ALL
    assert r.mismatches[2] == W4 // 8 and sum(r.mismatches) == W4 // 8
    assert r.recorded == cro.L2_RECORDS == len(faults) and r.overflow == 1
    assert json.loads(cro.emit_l2_annotations_json(r))["cohdi.io/probe-l2-verdict"] == "all"


def test_a_probe_in_flight_is_collected_intact(cro, ctx, coracle):
    ctx.probe_begin(0)
    r, _, _ = ctx.probe_l2(0, bytes=W4, iterations=1)
    assert r.status == 0
    p = ctx.probe_end(0)
    assert p.status == 0 and p.checksum == coracle.checksum(p.seed, 0, (64 << 20) // 8)


def test_the_sweep_region_is_untouched(cro, ctx):
    p = ctx.probe_device(0)
    assert p.status == 0
    r, _, _ = ctx.probe_l2(0, bytes=W4, iterations=1)
    assert r.status == 0
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == 0 and rep.pass_[0].halves == 3 and rep.pass_[0].mismatches == 0 and not words


def test_nvml_fields_equal_a_read_right_after(cro, ctx):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, _, _ = ctx.probe_l2(0, bytes=W4, iterations=1)
    h = cro.read_l2_health(uuid)
    assert {f: getattr(r.after, f) for f, _ in cro.L2Health._fields_} == {f: getattr(h, f) for f, _ in cro.L2Health._fields_}
    assert r.before.nvml == h.nvml & ~cro.L2_NVML_STATUS
    print("L2 health: nvml %d, threshold %d, sram %d/%d, l2 %d/%d, bucket %d" % (
        h.nvml, h.threshold_exceeded, h.sram_corrected, h.sram_uncorrected, h.l2_corrected, h.l2_uncorrected, h.unc_bucket_l2))


def test_invalid_arguments_are_refused(cro, ctx, clean):
    launches = ctx.launch_count()
    top = 8 * clean[0].l2_bytes // 16384 * 16384
    calls = [dict(bytes=cro.L2_MIN_BYTES - cro.L2_BLOCK_BYTES), dict(bytes=cro.L2_MIN_BYTES + 8), dict(bytes=top + cro.L2_BLOCK_BYTES),
             dict(iterations=cro.L2_MAX_ITERATIONS + 1), dict(a1_counters=cro.L2_MAX_A1_COUNTERS + 1),
             dict(a2_counters=cro.L2_MAX_A2_COUNTERS + 1), dict(inject=(3, 0, 1, 0, 0, 1)),
             dict(inject=(0, 256, 1, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 6, 0, 0, 1)),
             dict(inject=(0, 0, 1, 2, 0, 1), iterations=2), dict(inject=(0, 0, 1, 0, W4 // 8, 1), bytes=W4),
             dict(inject=(0, 0, 1, 0, -2, 1)), dict(inject=(1, 0, 0, 0, 65536, 1)), dict(inject=(2, 0, 0, 0, 1024, 1)),
             dict(inject=(1, 0, 0, 0, -1, 1)), dict(inject=(2, 0, 0, 0, 3, 1 << 40)), dict(dev=len(ctx.own_devices()))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            ctx.probe_l2(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    o = cro.L2Opts()
    o.deadline_ms = 1000                                   # only the helper form has a deadline of its own
    r, k, ks = cro.L2Result(), ctypes.c_int(), ctypes.c_int()
    sms, faults = (cro.L2Sm * 4)(), (cro.L2Fault * 4)()
    assert cro.lib.cro_probe_l2(ctx.handle, 0, ctypes.byref(o), ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert ctx.launch_count() == launches


def test_a_common_cause_below_one_block_per_cta_is_all(cro, ctx):
    """At 1 MiB (64 blocks, fewer than the SMs) only some SMs read in an element; every one of them failing is `all`."""
    r, sms, _ = ctx.probe_l2(0, bytes=cro.L2_MIN_BYTES, iterations=1, inject=(cro.L2_MARCH, -1, 2, 0, -1, BIT))
    readers = [s for s in sms if s.words_read[2]]
    assert 0 < len(readers) < r.ctas and all(s.mismatches[2] == s.words_read[2] for s in readers)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ALL and r.mismatches[2] == cro.L2_MIN_BYTES // 8


def test_helper_form_agrees_with_the_in_process_form(cro, ctx, coracle):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    r, sms, faults = cro.probe_l2_uuid(ctx, uuid, bytes=W4, iterations=2)
    check_clean(cro, ctx, coracle, r, sms, faults, W4, 2)
    assert r.helper_ns > r.wall_ns > 0 and r.call == 0
    w = 777
    inj = (cro.L2_MARCH, -1, 3, 1, w, BIT)
    a = ctx.probe_l2(0, bytes=W4, iterations=2, inject=inj)
    b = cro.probe_l2_uuid(None, uuid, bytes=W4, iterations=2, inject=inj)
    for r, sms, faults in (a, b):
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and r.bad_sms == 1
        (f,) = faults
        assert (f.element, f.iteration, f.word, f.cta, f.expected ^ f.actual) == (3, 1, w, a[2][0].cta, BIT)
    for leg, counter, mask in ((cro.L2_A1, 5, BIT), (cro.L2_A2, 6, 1)):
        x = ctx.probe_l2(0, bytes=W4, iterations=1, inject=(leg, -1, 0, 0, counter, mask))[0]
        y = cro.probe_l2_uuid(ctx, uuid, bytes=W4, iterations=1, inject=(leg, -1, 0, 0, counter, mask))[0]
        for q in (x, y):
            assert q.verdict == cro.L2_ATOMIC and (q.a1_bad, q.a2_bad, q.a2_holes) == ((1, 0, 0) if leg == cro.L2_A1 else (0, 1, 1))
            assert (q.a1_bad_counter[0] if leg == cro.L2_A1 else q.a2_bad_counter[0]) == counter


def test_helper_calls_use_fresh_seeds(cro, ctx):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    seeds = set()
    for c in (ctx, ctx, None, None):
        r, _, _ = cro.probe_l2_uuid(c, uuid, bytes=W4, iterations=1)
        assert r.status == cro.OK and r.call == 0
        seeds.add(r.seed)
    inproc, _, _ = ctx.probe_l2(0, bytes=W4, iterations=1)
    assert len(seeds) == 4 and inproc.seed not in seeds
