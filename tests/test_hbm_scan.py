"""The whole-HBM scan (cro_scan_hbm, cro_scan_hbm_uuid) on one H100, against the C oracle's checksums and oracle/scan.py.

Every scan here is bounded by max_bytes, so a shared card keeps its memory.  Mismatches come only from the scan's
test force (stuck bits written after each fill); nothing here repeats a call to catch a real fault."""
import os

import pytest

MASK = (1 << 64) - 1
CHUNK = 64 << 20                       # test chunks: several of them in a small scan
SMALL = (256 << 20) + (3 << 20) + 112  # ragged: the last chunk is 3 MiB + 112 B
THREADS = max(1, min(16, os.cpu_count() or 1))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def scan_oracle(_built):
    import scan
    return scan


def complement(cf, n):
    x, s, w = cf
    return (x ^ (MASK if n & 1 else 0), (-n - s) & MASK, (-n * n - w) & MASK)


def health(h):
    return {"nvml": h.nvml, "ecc_corrected": h.ecc_corrected, "ecc_uncorrected": h.ecc_uncorrected,
            "remap_corrected": h.remap_corrected, "remap_uncorrected": h.remap_uncorrected,
            "remap_pending": h.remap_pending, "remap_failure": h.remap_failure, "histogram": list(h.histogram)}


def check_clean(cro, coracle, scan_oracle, rep, words, max_bytes, chunk_bytes):
    assert rep.status == 0 and rep.cuda_error == 0 and rep.complete == 1 and not words, rep.status
    assert rep.elements_done == 4 and all(rep.element_ns)
    assert rep.covered_bytes == max_bytes and rep.free_bytes > rep.covered_bytes and rep.total_bytes >= rep.free_bytes
    n = (max_bytes + chunk_bytes - 1) // chunk_bytes
    assert rep.n_chunks == n
    word0 = 0
    for k in range(n):
        K = rep.chunk[k]
        assert K.word0 == word0 and K.bytes == min(chunk_bytes, max_bytes - 8 * word0)
        want = coracle.checksum((rep.seed + K.word0) & MASK, 0, K.bytes // 8, threads=THREADS)
        assert K.expect == want and K.fold(0) == want, k
        assert K.fold(1) == complement(want, K.bytes // 8), k
        word0 += K.bytes // 8
    assert sum(rep.chunk[k].bytes for k in range(n)) == rep.covered_bytes
    for p in range(2):
        P = rep.pass_[p]
        assert P.mismatches == P.recorded == P.granules == 0 and P.words_scanned == rep.covered_bytes // 8
        assert P.invert == (MASK if p else 0)
    assert rep.health == scan_oracle.health_bits(health(rep.before), health(rep.after))


def test_clean_scan_in_ragged_test_chunks(cro, ctx, coracle, scan_oracle):
    rep, words = ctx.scan_hbm(0, max_bytes=SMALL, chunk_bytes=CHUNK)
    check_clean(cro, coracle, scan_oracle, rep, words, SMALL, CHUNK)
    assert rep.held_bytes == 2 * (64 << 20) or rep.held_bytes == 0


def test_clean_16_gib_scan_in_default_chunks(cro, ctx, coracle, scan_oracle):
    rep, words = ctx.scan_hbm(0, max_bytes=16 << 30)
    check_clean(cro, coracle, scan_oracle, rep, words, 16 << 30, cro.SCAN_CHUNK_BYTES)
    assert rep.n_chunks == 8


def forced(cro, ctx, scan_oracle, first, count, and_mask, or_mask, seed=0x5CA9):
    rep, words = ctx.scan_hbm(0, max_bytes=SMALL, chunk_bytes=CHUNK, seed=seed, cap=8192,
                              force=(first, count, and_mask, or_mask))
    return rep, words, scan_oracle.forced_mismatches(seed, first, count, and_mask, or_mask)


def test_stuck_bit_across_a_chunk_boundary(cro, ctx, scan_oracle):
    first, count = CHUNK // 8 - 300, 600                      # 300 words either side of chunk 0's end
    rep, words, want = forced(cro, ctx, scan_oracle, first, count, ~(1 << 5) & MASK, 0)
    assert rep.status == cro.ERR_CHECKSUM and rep.complete == 1 and rep.seed == 0x5CA9
    for p in range(2):
        P = rep.pass_[p]
        assert P.mismatches == P.recorded == want[p]["mismatches"] > 0
        assert list(P.bit_flips) == want[p]["bit_flips"] and P.granules == want[p]["granules"] == 2
    assert rep.pass_[0].mismatches + rep.pass_[1].mismatches == count     # each word fails in exactly one pass
    expect = sorted([(w["word"], w["expected"], w["actual"], 1 << p) for p in range(2) for w in want[p]["words"]])
    assert [(w.word_index, w.expected, w.actual, w.passes) for w in words] == expect
    assert rep.located == len(words) == count and rep.flip_or == 1 << 5
    for w in words:
        k, off = rep.place(w)
        assert (k, off) == ((0, w.word_index) if w.word_index < CHUNK // 8 else (1, w.word_index - CHUNK // 8))


def test_a_storm_keeps_exact_counts(cro, ctx, scan_oracle):
    first, count = CHUNK // 8 - 10000, 30000
    rep, words, want = forced(cro, ctx, scan_oracle, first, count, MASK, 1 << 63)
    assert rep.status == cro.ERR_CHECKSUM and rep.complete == 0
    for p in range(2):
        P = rep.pass_[p]
        assert P.mismatches == want[p]["mismatches"] > cro.LOCATE_RECORDS and P.recorded == cro.LOCATE_RECORDS
        assert list(P.bit_flips) == want[p]["bit_flips"] and P.granules == want[p]["granules"]


def test_the_helper_finds_what_the_process_finds(cro, ctx, scan_oracle):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    first, count = CHUNK // 8 - 300, 600
    mine, my_words, _ = forced(cro, ctx, scan_oracle, first, count, ~(1 << 5) & MASK, 0)
    rep, words = cro.scan_hbm_uuid(ctx, uuid, max_bytes=SMALL, chunk_bytes=CHUNK, seed=0x5CA9, cap=8192,
                                   force=(first, count, ~(1 << 5) & MASK, 0))
    assert rep.status == cro.ERR_CHECKSUM and rep.complete == 1 and rep.helper_ns > 0 and rep.held_bytes == 0
    assert rep.covered_bytes == mine.covered_bytes and rep.n_chunks == mine.n_chunks
    for p in range(2):
        assert rep.pass_[p].mismatches == mine.pass_[p].mismatches and list(rep.pass_[p].bit_flips) == list(mine.pass_[p].bit_flips)
        assert rep.pass_[p].granules == mine.pass_[p].granules
    for k in range(rep.n_chunks):
        assert rep.chunk[k].fold(0) == mine.chunk[k].fold(0) and rep.chunk[k].fold(1) == mine.chunk[k].fold(1)
    assert [(w.word_index, w.expected, w.actual, w.passes, w.reserved) for w in words] == \
        [(w.word_index, w.expected, w.actual, w.passes, w.reserved) for w in my_words]
    ann = cro.emit_scan_annotations_json(rep)
    assert '"cohdi.io/hbm-scan-verdict":"corrupt"' in ann and '"cohdi.io/hbm-scan-mismatches":"%d,%d"' % (
        rep.pass_[0].mismatches, rep.pass_[1].mismatches) in ann


def test_a_zero_seed_is_fresh_and_reported(cro, ctx):
    a, _ = ctx.scan_hbm(0, max_bytes=CHUNK)
    b, _ = ctx.scan_hbm(0, max_bytes=CHUNK)
    assert a.status == b.status == 0 and a.seed and b.seed and a.seed != b.seed


def test_a_probe_in_flight_is_collected_and_the_region_is_untouched(cro, ctx, coracle):
    p = ctx.probe_device(0)
    assert p.status == 0
    ctx.probe_begin(0)
    rep, _ = ctx.scan_hbm(0, max_bytes=SMALL, chunk_bytes=CHUNK)
    assert rep.status == 0 and rep.held_bytes == 2 * (64 << 20)
    q = ctx.probe_end(0)
    assert q.status == 0 and q.checksum == coracle.checksum(q.seed, 0, (64 << 20) // 8)
    loc, words = ctx.locate_faults(0, retest=False)
    assert loc.status == 0 and loc.pass_[0].halves == 3 and loc.pass_[0].mismatches == 0 and not words


def test_nvml_fields_match_a_read_right_after(cro, ctx):
    uuid = ctx.own_devices()[0].gpu_uuid.decode()
    rep, _ = ctx.scan_hbm(0, max_bytes=CHUNK)
    now = cro.read_hbm_health(uuid)
    assert rep.status == 0
    assert health(rep.after) == health(now)
    assert rep.before.nvml == rep.after.nvml & ~cro.HBM_NVML_HISTOGRAM       # no histogram before E0


def test_invalid_arguments_are_refused(cro, ctx):
    n_words = SMALL // 8
    for kw in [dict(dev=len(ctx.own_devices())), dict(chunk_bytes=CHUNK + 8),
               dict(force=(n_words, 1, 0, 0)), dict(force=(n_words - 10, 11, 0, 0))]:
        kw.setdefault("max_bytes", SMALL)
        with pytest.raises(cro.ProbeError) as e:
            ctx.scan_hbm(**kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    with pytest.raises(cro.ProbeError) as e:
        ctx.scan_hbm(0, reserve_bytes=1 << 50)
    assert e.value.code == cro.ERR_OOM and "no room for one scan chunk" in str(e.value)
