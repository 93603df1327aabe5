"""The fault locator (cro_locate_faults) on one H100, against the C oracle's pattern_word and checksums.

Word indices are the region's: [0, n) is half A and [n, 2n) half B, n = S / 8; word i of either half is expected to
hold pattern_word(seed, i mod n)."""
import functools
import operator

import numpy as np
import pytest

MASK = (1 << 64) - 1
MiB = 1 << 20
RAGGED = 3 * MiB + 112
SEED_BASE = 0x00C0FFEE00000000

pytestmark = pytest.mark.gpu


def n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


def closed_form_complement(cf, n):
    x, s, w = cf
    return (x ^ (MASK if n & 1 else 0), (-n - s) & MASK, (-n * n - w) & MASK)


def retest_seed(ctx):
    minor = ctx.own_devices()[0].device_minor
    return ((SEED_BASE | minor) + (1 << 63)) & MASK


def flips(words):
    """Per-bit counts of the flip masks of (word, expected, actual) triples."""
    c = [0] * 64
    for _w, e, a in words:
        for b in range(64):
            c[b] += ((e ^ a) >> b) & 1
    return c


def granules(indices):
    return len({(w * 8) // (2 * MiB) for w in indices})


def as_tuples(words):
    return [(w.word_index, w.expected, w.actual) for w in words]


@pytest.mark.parametrize("S", [64 * MiB, RAGGED, 4 << 30], ids=["64MiB", "3MiB+112B", "4GiB"])
def test_clean_runs_after_a_passing_probe(cro, coracle, S):
    n = S // 8
    threads = 16
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=1) as ctx:
        r = ctx.probe_device(0)
        assert r.status == cro.OK
        want = coracle.checksum(r.seed, 0, n, threads=threads)
        rep, words = ctx.locate_faults(0, retest=False)
        assert (rep.status, rep.verdict, rep.complete, rep.n_passes, words) == (cro.OK, cro.FAULTS_NONE, 1, 1, [])
        p0 = rep.pass_[0]
        assert (p0.halves, p0.skipped, p0.mismatches, p0.recorded, p0.granules) == (3, 0, 0, 0, 0)
        assert p0.words_scanned == 2 * n and list(p0.seed) == [r.seed, r.seed]
        assert p0.fold(0) == want and p0.fold(1) == want
        assert p0.scan_ns > 0

        rep, words = ctx.locate_faults(0, retest=True)
        rs = retest_seed(ctx)
        assert (rep.status, rep.verdict, rep.complete, rep.n_passes, rep.retest_seed, words) == \
            (cro.OK, cro.FAULTS_NONE, 1, 3, rs, [])
        cf = coracle.checksum(rs, 0, n, threads=threads)
        for p, fold in ((1, cf), (2, closed_form_complement(cf, n))):
            P = rep.pass_[p]
            assert (P.halves, P.mismatches, P.words_scanned, list(P.seed)) == (3, 0, 2 * n, [rs, rs])
            assert P.invert == (MASK if p == 2 else 0)
            assert P.fold(0) == fold and P.fold(1) == fold, p
        assert sum(rep.bit_flips) == 0 and rep.flip_or == 0

        # the retest consumed no nonce, and the single sweeps refill before they read
        r2 = ctx.probe_device(0)
        assert r2.status == cro.OK and r2.nonce == r.nonce + 1
        rep, _ = ctx.locate_faults(0, retest=True)
        assert rep.verdict == cro.FAULTS_NONE
        want2 = coracle.checksum(ctx.seed(0), 0, n, threads=threads)
        assert ctx.hbm_read_checksum(0, cro.READ_LDG).checksum == want2
        assert ctx.hbm_copy(0, cro.COPY_TMA_FUSED).checksum == want2
        assert ctx.hbm_read_checksum(0, cro.READ_LDG, dst=True).checksum == want2


def _inject_cases():
    n = (64 * MiB) // 8
    g1 = (2 * MiB) // 8
    return {
        "first_and_last_of_A_and_B": (64 * MiB, [(0, 1), (n - 1, 1 << 40), (n, 1 << 7), (2 * n - 1, 1 << 63)]),
        "ragged_tail_words": (RAGGED, [(RAGGED // 8 - 1, 3), (2 * (RAGGED // 8) - 1, 1 << 33), (RAGGED // 8 - 14, 1)]),
        "one_bit": (64 * MiB, [(12345, 1 << 17)]),
        "all_64_bits": (64 * MiB, [(777, MASK)]),
        "two_words_one_vector": (64 * MiB, [(100, 1 << 3), (101, 1 << 60)]),
        "two_in_one_warp_tile": (64 * MiB, [(128, 1 << 1), (139, 1 << 2), (n + 128, 1 << 9)]),
        "two_granules": (64 * MiB, [(10, 1 << 5), (g1 + 7, 1 << 5), (n + 3 * g1 + 1, 1 << 6)]),
    }


@pytest.mark.parametrize("case", sorted(_inject_cases()))
def test_injected_faults_are_located_exactly(cro, coracle, case):
    S, inj = _inject_cases()[case]
    n = S // 8
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        r = ctx.probe_device(0)
        assert r.status == cro.OK
        for w, m in inj:
            ctx.inject_fault(0, w, m)
        got_now = {w: ctx.read_words(0, w, 1)[0] for w, _ in inj}
        rep, words = ctx.locate_faults(0, retest=False)
        want = sorted((w, coracle.pattern_word(r.seed, w % n), got_now[w]) for w, _ in inj)
        assert as_tuples(words) == want
        assert all(e ^ a == dict(inj)[w] for w, e, a in want)
        assert all(x.passes == 1 for x in words)
        assert (rep.status, rep.verdict, rep.complete) == (cro.ERR_CHECKSUM, cro.FAULTS_UNCLASSIFIED, 1)
        P = rep.pass_[0]
        assert (P.mismatches, P.recorded, P.granules) == (len(inj), len(inj), granules([w for w, _ in inj]))
        assert list(rep.bit_flips) == flips(want)
        assert rep.flip_or == functools.reduce(operator.or_, [m for _, m in inj])
        assert rep.recorded == rep.located == len(inj)

        rep, words = ctx.locate_faults(0, retest=True)
        assert as_tuples(words) == want and all(x.passes == 1 for x in words)
        assert (rep.verdict, rep.complete, rep.pass_[1].mismatches, rep.pass_[2].mismatches) == \
            (cro.FAULTS_NOT_REPRODUCED, 1, 0, 0)


def test_more_faults_than_the_lists_hold(cro, coracle):
    S = 64 * MiB
    n = S // 8
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        idx = [3 + 977 * k for k in range(10)]
        for w in idx:
            ctx.inject_fault(0, w, 1 << (w % 64))
        rep, words = ctx.locate_faults(0, retest=False, cap=4)
        assert (rep.pass_[0].mismatches, rep.located, rep.recorded, len(words), rep.complete) == (10, 10, 4, 4, 0)
        assert [w.word_index for w in words] == idx[:4]

        # past the device's record buffer: counts stay exact
        first, count = 1000, 3 * cro.LOCATE_RECORDS
        rs = retest_seed(ctx)
        p = [coracle.pattern_word(rs, (first + i) % n) for i in range(count)]
        rep, words = ctx.locate_faults(0, retest=True, cap=256, force=(first, count, MASK, 1 << 62))
        want1 = sum(1 for v in p if not (v >> 62) & 1)
        want2 = count - want1
        assert (rep.pass_[0].mismatches, rep.pass_[1].mismatches, rep.pass_[2].mismatches) == (10, want1, want2)
        assert [rep.pass_[k].recorded for k in range(3)] == [10, min(want1, cro.LOCATE_RECORDS), min(want2, cro.LOCATE_RECORDS)]
        assert rep.bit_flips[62] == want1 + want2 and rep.complete == 0 and rep.recorded == 256
        assert rep.verdict == cro.FAULTS_PERSISTENT


def _ping_pong_prediction(after, word, n, C=3, R=2):
    """Which halves hold the injected word at the end of a (C, R) probe, walking its launch order on the host."""
    h, i = divmod(word, n)
    bad = [False, False]         # does half A / B hold the flipped word
    sweeps = ["fill"] + ["copy"] * C + ["read"] * R
    for k, kind in enumerate(sweeps):
        if kind == "copy":
            src = (k - 1) & 1    # copy j reads half j & 1 and writes the other
            bad[1 - src] = bad[src]
        if k == after:
            bad[h] = not bad[h]
    return [hh for hh in (0, 1) if bad[hh]], i


@pytest.mark.parametrize("after", range(6))
@pytest.mark.parametrize("half", [0, 1])
def test_in_probe_injection_is_found_where_the_schedule_left_it(cro, coracle, after, half):
    S = 64 * MiB
    n = S // 8
    word, mask = half * n + 4242, 1 << 21
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=3, inject=(after, word, mask)) as ctx:
        r = ctx.probe_device(0, allow_checksum_error=True)
        rep, words = ctx.locate_faults(0, retest=False)
        halves, i = _ping_pong_prediction(after, word, n)
        e = coracle.pattern_word(r.seed, i)
        assert as_tuples(words) == [(hh * n + i, e, e ^ mask) for hh in halves]
        assert rep.complete == 1 and rep.pass_[0].halves == 3
        if r.fail_code == cro.FAIL_READ:
            read_half = [1, 0][r.fail_index]          # C = 3: read 0 reads B (the last copy's destination), read 1 A
            assert read_half in halves
            d = (e ^ mask) - e
            got = (e ^ (e ^ mask), d & MASK, (d * (2 * i + 1)) & MASK)
            want = (r.checksum_xor ^ r.expect_xor, (r.checksum_sum - r.expect_sum) & MASK,
                    (r.checksum_wsum - r.expect_wsum) & MASK)
            assert got == want


@pytest.mark.parametrize("stuck", [0, 1])
@pytest.mark.parametrize("pattern_bit", [0, 1])
def test_stuck_cell_is_flagged_in_exactly_one_retest_pass(cro, coracle, stuck, pattern_bit):
    S = 64 * MiB
    n = S // 8
    bit = 11
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        rs = retest_seed(ctx)
        i = next(k for k in range(5000, 6000) if (coracle.pattern_word(rs, k) >> bit) & 1 == pattern_bit)
        for word in (i, n + i):
            force = (word, 1, MASK, 1 << bit) if stuck else (word, 1, MASK ^ (1 << bit), 0)
            rep, words = ctx.locate_faults(0, retest=True, force=force)
            # pass 1 writes p, pass 2 writes ~p: the cell disagrees when what is written differs from the stuck value
            p_want = 1 if pattern_bit != stuck else 2
            e = coracle.pattern_word(rs, i) ^ (MASK if p_want == 2 else 0)
            assert as_tuples(words) == [(word, e, e ^ (1 << bit))], (stuck, pattern_bit)
            assert words[0].passes == 1 << p_want
            assert (rep.verdict, rep.complete, rep.pass_[0].mismatches) == (cro.FAULTS_PERSISTENT, 1, 0)
            assert rep.bit_flips[bit] == 1 and rep.flip_or == 1 << bit


def test_storm_counts_are_exact(cro, coracle, oracle):
    S = 512 * MiB
    n = S // 8
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        clean, _ = ctx.locate_faults(0, retest=False)
        rs = retest_seed(ctx)
        bit = 5
        chunk = 1 << 23
        ones = sum(int(((oracle.pattern_words_np(rs, k, min(chunk, n - k)) >> np.uint64(bit)) & np.uint64(1)).sum())
                   for k in range(0, n, chunk))
        rep, words = ctx.locate_faults(0, retest=True, force=(0, n, MASK, 1 << bit))   # all of half A, bit 5 stuck at 1
        assert (rep.pass_[1].mismatches, rep.pass_[2].mismatches) == (n - ones, ones)
        assert rep.bit_flips[bit] == n and rep.flip_or == 1 << bit
        assert rep.pass_[1].granules == rep.pass_[2].granules == S // (2 * MiB)
        assert rep.pass_[1].recorded == rep.pass_[2].recorded == cro.LOCATE_RECORDS and rep.complete == 0
        assert rep.verdict == cro.FAULTS_PERSISTENT and all(w.word_index < n for w in words)
        print("storm scan (512 MiB half A, every word bit %d forced): pass 1 %.3f ms, clean pass 0 over both halves %.3f ms"
              % (bit, rep.pass_[1].scan_ns / 1e6, clean.pass_[0].scan_ns / 1e6))


def test_pending_probes_stay_collectable(cro, coracle):
    S = 64 * MiB
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        ctx.probe_begin(0)
        ctx.probe_begin(0)
        rep, words = ctx.locate_faults(0, retest=False)
        r1, r2 = ctx.probe_end(0), ctx.probe_end(0)
        assert r1.status == r2.status == cro.OK and r2.nonce == r1.nonce + 1
        for r in (r1, r2):
            assert r.checksum == coracle.checksum(r.seed, 0, S // 8)
        assert list(rep.pass_[0].seed) == [r2.seed, r2.seed] and rep.verdict == cro.FAULTS_NONE and words == []


def test_half_bookkeeping_on_one_gpu(cro):
    S = 64 * MiB
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=1, flags=cro.F_SKIP_COPY) as ctx:
        assert ctx.probe_device(0).status == cro.OK
        rep, _ = ctx.locate_faults(0, retest=False)
        assert (rep.pass_[0].halves, rep.pass_[0].skipped, rep.pass_[0].words_scanned) == (1, 2, S // 8)
        ctx.locate_faults(0, retest=True)
        rep, _ = ctx.locate_faults(0, retest=False)
        assert (rep.pass_[0].halves, rep.pass_[0].skipped, rep.verdict) == (0, 3, cro.FAULTS_NONE)
        ctx.hbm_read_checksum(0, cro.READ_LDG)          # refills half A
        assert ctx.locate_faults(0, retest=False)[0].pass_[0].halves == 1
        ctx.hbm_copy(0, cro.COPY_LDG)                   # B takes A's pattern
        rep, _ = ctx.locate_faults(0, retest=False)
        assert rep.pass_[0].halves == 3 and rep.verdict == cro.FAULTS_NONE


def test_unknown_device_is_refused(cro):
    with cro.ProbeContext(sweep_bytes=64 * MiB, devices=[0]) as ctx:
        with pytest.raises(cro.ProbeError) as e:
            ctx.locate_faults(5)
        assert e.value.code == cro.ERR_INVALID_ARG and "helper process" in str(e.value)


@pytest.mark.skipif(n_gpus() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("push", [True, False])
def test_half_b_after_probe_all(cro, push):
    S = 64 * MiB
    flags = 0 if push else cro.F_SKIP_P2P_WRITE
    with cro.ProbeContext(sweep_bytes=S, devices=[0, 1], read_sweeps=1, copy_sweeps=1, flags=flags) as ctx:
        rs = ctx.probe_all()
        assert all(r.status == cro.OK for r in rs)
        rep, _ = ctx.locate_faults(0, retest=False)
        assert rep.pass_[0].halves == (1 if push else 3) and rep.verdict == cro.FAULTS_NONE
