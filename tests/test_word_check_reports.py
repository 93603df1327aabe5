"""The fault locator's, the whole-HBM scan's and the host link probe's reports without a GPU: the library's host code
run on caller-given device output (cro_selftest_locate_collect, cro_selftest_scan_collect, cro_selftest_link_classify,
the same functions a probe call runs once its kernels are done) against the restatements written from
include/croprobe.h (oracle/faults.py, oracle/scan.py, oracle/link.py), field for field.

A GPU reaches only the states the software force or injection can make: one force range, one injected word, records
that always explain the fold.  Each other rule has a hand-built case here that also pins the expected value; a seeded
sweep of synthetic calls covers the rest."""
import ctypes
import os
import random
import subprocess

import pytest

import faults
import link
import scan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = (1 << 64) - 1
RECORDS = 4096
MINOR = 3


# ---- plumbing ---------------------------------------------------------------------------------------------------------
def plain(x):
    """A ctypes value as plain Python: structures as dicts, arrays as lists."""
    if isinstance(x, ctypes.Structure):
        return {f: plain(getattr(x, f)) for f, _ in x._fields_}
    if isinstance(x, ctypes.Array):
        return [plain(v) for v in x]
    return x


def mk(cls, d):
    x = cls()
    for f, v in d.items():
        if isinstance(v, list):
            getattr(x, f)[:] = v
        else:
            setattr(x, f, v)
    return x


def slot(fold=(0, 0, 0), n_words=0, t0=100, t1=300):
    return dict(x=fold[0], s=fold[1], w=fold[2], t0=t0, t1=t1, stamp=0, n_words=n_words, pad=0)


def record(word, expected, actual):
    return dict(word=word, expected=expected, actual=actual)


def counters(recs, mismatches=None, claims=None, bits=None):
    """The counters a kernel keeps for these records: one claim and one mismatch per record, and their bit flips,
    unless given."""
    if bits is None:
        bits = [sum((r["expected"] ^ r["actual"]) >> b & 1 for r in recs) for b in range(64)]
    n = len(recs)
    return dict(mismatches=n if mismatches is None else mismatches, claims=n if claims is None else claims, bits=bits)


def changed(cf, recs, index):
    """The fold of a sweep whose closed form is cf after the records' words changed, word w at position index(w)."""
    d = faults.deltas(recs, index)
    return cf[0] ^ d[0], (cf[1] + d[1]) & U64, (cf[2] + d[2]) & U64


def hook_lists(cro, call):
    """A call's counters and per-pass (or per-check) records as the binding's structs."""
    return ([mk(cro.LocateCounters, c) for c in call["counters"]],
            [[mk(cro.LocateRecord, r) for r in recs] for recs in call["records"]])


# ---- the locator ------------------------------------------------------------------------------------------------------
def lpass(halves, seeds, invert=0, skipped=None):
    return dict(halves=halves, skipped=(3 & ~halves) if skipped is None else skipped, seed=list(seeds), invert=invert)


def locate_call(S, passes, recs, cf, folds=None, ctrs=None, granules=None, cap=None, gw=2):
    """A locator call over a region of S bytes.  cf: the closed-form triples, in slot order; each compared half's fold
    is its closed form (complemented for an inverted pass) changed by that half's records, unless folds[(p, h)] says
    otherwise."""
    n = S // 8
    seeds = []
    for P in passes:
        for h in range(2):
            if P["halves"] >> h & 1 and P["seed"][h] not in seeds:
                seeds.append(P["seed"][h])
    slots = [slot() for _ in range(9)]
    for k, c in enumerate(cf):
        slots[6 + k] = slot(c, n)
    for p, P in enumerate(passes):
        for h in range(2):
            if P["halves"] >> h & 1:
                c = cf[seeds.index(P["seed"][h])]
                c = faults.complement_fold(c, n) if P["invert"] else c
                mine = [r for r in recs[p] if (r["word"] >= n) == (h == 1)]
                f = (folds or {}).get((p, h)) or changed(c, mine, lambda w: w - h * n)
                slots[2 * p + h] = slot(f, n, t0=1000 * p, t1=1000 * p + 250 + h)
    return dict(sweep_bytes=S, passes=passes, counters=ctrs or [counters(r) for r in recs], records=recs,
                granules=granules or [[0] * gw for _ in passes], slots=slots,
                cap=sum(len(r) for r in recs) if cap is None else cap)


def check_locate(cro, call):
    c, r = hook_lists(cro, call)
    got_r, got_w = cro.selftest_locate_collect(call["sweep_bytes"], [mk(cro.LocatePass, dict(P)) for P in call["passes"]], c,
                                               r, call["granules"], [mk(cro.SweepSlot, s) for s in call["slots"]],
                                               cap=call["cap"])
    want_r, want_w = faults.collect(call)
    got_r, got_w = plain(got_r), [plain(w) for w in got_w]
    assert got_r == want_r
    assert got_w == want_w
    return got_r, got_w


CF = [(0x1111, 0x2222, 0x3333), (0xAAAA, 0xBBBB, 0xCCCC), (0x5555_0000_0000_0001, 7, 9)]
S0 = 1 << 12                                       # 512 words per half


def test_claims_past_the_record_cap_leave_the_report_incomplete(cro):
    recs = [record(i, i, i ^ 1) for i in range(RECORDS)]
    call = locate_call(S0 * 16, [lpass(1, (5, 0))], [recs], CF[:1],
                       ctrs=[counters(recs, mismatches=5000, claims=5000)])
    r, words = check_locate(cro, call)
    assert (r["pass_"][0]["mismatches"], r["pass_"][0]["recorded"], r["complete"]) == (5000, RECORDS, 0)
    assert r["located"] == len(words) == RECORDS and r["status"] == cro.ERR_CHECKSUM
    assert r["verdict"] == cro.FAULTS_UNCLASSIFIED
    # the same records under their own count are complete, and a cap on the caller's list takes that back
    call = locate_call(S0 * 16, [lpass(1, (5, 0))], [recs[:40]], CF[:1])
    assert check_locate(cro, call)[0]["complete"] == 1
    call["cap"] = 39
    r, words = check_locate(cro, call)
    assert (r["complete"], r["recorded"], r["located"], len(words)) == (0, 39, 40, 39)


def test_located_counts_distinct_words_over_the_passes(cro):
    n = S0 // 8
    p0 = [record(3, 10, 11), record(n + 7, 20, 22)]
    p1 = [record(3, 30, 31), record(9, 40, 44)]
    p2 = [record(n + 7, ~20 & U64, 0), record(3, 50, 51)]
    call = locate_call(S0, [lpass(3, (5, 6)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)], [p0, p1, p2], CF)
    r, words = check_locate(cro, call)
    assert r["located"] == 3 and r["complete"] == 1
    assert [(w["word_index"], w["passes"]) for w in words] == [(3, 0b111), (9, 0b010), (n + 7, 0b101)]
    assert r["verdict"] == cro.FAULTS_PERSISTENT


def test_a_word_seen_in_passes_0_and_2_keeps_pass_0s_expected(cro):
    """Passes 0b101: a cell that holds a 1 whatever is written fails against the pattern and its complement only."""
    e = 0x0123_4567_89AB_CDEF
    p0, p2 = [record(17, e, e | 1 << 40)], [record(17, ~e & U64, (~e | 1 << 4) & U64)]
    call = locate_call(S0, [lpass(1, (5, 0)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)], [p0, [], p2], CF[:2])
    r, words = check_locate(cro, call)
    assert [(w["word_index"], w["expected"], w["actual"], w["passes"]) for w in words] == [(17, e, e | 1 << 40, 0b101)]
    assert r["complete"] == 1 and r["pass_"][1]["mismatches"] == 0


def test_half_b_records_are_weighted_from_the_halfs_start(cro):
    """Half B's word n is its word 0: weighted 1, not 2n + 1.  Words n - 1, n and 2n - 1 each change the fold."""
    n = S0 // 8
    recs = [record(n - 1, 5, 9), record(n, 100, 7), record(2 * n - 1, 1 << 63, 3)]
    call = locate_call(S0, [lpass(3, (5, 6))], [recs], CF[:2])
    r, _ = check_locate(cro, call)
    assert r["complete"] == 1
    # weighted by the region index, the same records explain nothing: the fold says so
    wrong = changed(CF[1], recs[1:], lambda w: w)
    call = locate_call(S0, [lpass(3, (5, 6))], [recs], CF[:2], folds={(0, 1): wrong})
    assert check_locate(cro, call)[0]["complete"] == 0


@pytest.mark.parametrize("n", [511, 512], ids=["odd-n", "even-n"])
def test_the_complement_pass_at_odd_and_even_n(cro, n):
    """Pass 2 compares with ~pattern: its closed form is the pattern's complemented over the half's n words (the xor
    flips only for odd n)."""
    S = 8 * n
    recs = [record(4, 1, 2), record(n + 1, 8, 0)]
    passes = [lpass(3, (5, 6)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)]
    call = locate_call(S, passes, [[], [], recs], CF)
    r, _ = check_locate(cro, call)
    assert r["complete"] == 1
    assert r["pass_"][2]["fold_xor"][0] == changed(faults.complement_fold(CF[2], n), recs[:1], lambda w: w)[0]
    # a fold complemented the other way is not explained
    other = faults.complement_fold(CF[2], n + 1)
    call = locate_call(S, passes, [[], [], recs], CF, folds={(2, 0): changed(other, recs[:1], lambda w: w)})
    assert check_locate(cro, call)[0]["complete"] == 0


def test_a_fold_difference_no_record_explains_leaves_it_incomplete(cro):
    recs = [record(10, 1, 3)]
    f = changed(CF[0], recs + [record(11, 0, 1 << 20)], lambda w: w)     # a word the compare did not record
    call = locate_call(S0, [lpass(1, (5, 0))], [recs], CF[:1], folds={(0, 0): f})
    r, _ = check_locate(cro, call)
    assert (r["complete"], r["pass_"][0]["recorded"], r["pass_"][0]["mismatches"]) == (0, 1, 1)
    # no mismatch at all, and a fold off its closed form: incomplete, and still status OK
    call = locate_call(S0, [lpass(1, (5, 0))], [[]], CF[:1], folds={(0, 0): (1, 2, 3)})
    r, _ = check_locate(cro, call)
    assert (r["complete"], r["status"], r["verdict"]) == (0, cro.OK, cro.FAULTS_NONE)


def test_a_skipped_halfs_slots_are_ignored(cro):
    call = locate_call(S0, [lpass(1, (5, 0))], [[record(2, 1, 0)]], CF[:1])
    call["slots"][1] = slot((7, 7, 7), 999, t0=0, t1=1 << 40)            # half B's slot holds whatever was there
    call["slots"][7] = slot((9, 9, 9), 3)
    r, _ = check_locate(cro, call)
    P = r["pass_"][0]
    assert (P["halves"], P["skipped"], P["words_scanned"], P["scan_ns"]) == (1, 2, S0 // 8, 250)
    assert (P["fold_xor"][1], P["fold_sum"][1], P["fold_wsum"][1], r["complete"]) == (0, 0, 0, 1)


def test_the_closed_form_is_shared_only_between_equal_seeds(cro):
    """Both halves of pass 0 under one seed use one closed form (slot 6); the retest seed's is then slot 7."""
    recs = [record(1, 1, 0), record(S0 // 8 + 1, 4, 0)]
    call = locate_call(S0, [lpass(3, (5, 5)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)], [recs, [], []], CF[:2])
    call["slots"][8] = slot((1, 2, 3), 77)                                 # no third seed: never read
    assert check_locate(cro, call)[0]["complete"] == 1
    # with two seeds in pass 0 the retest's closed form moves to slot 8
    call = locate_call(S0, [lpass(3, (5, 6)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)], [recs, [], []], CF)
    assert check_locate(cro, call)[0]["complete"] == 1
    call["slots"][8], call["slots"][7] = call["slots"][7], call["slots"][8]
    assert check_locate(cro, call)[0]["complete"] == 0


def test_bit_flips_and_granules_sum_and_count_per_pass(cro):
    ctrs = [counters([], mismatches=3, claims=0, bits=[1 if b == 5 else 0 for b in range(64)]),
            counters([], mismatches=0, claims=0, bits=[2 if b in (5, 63) else 0 for b in range(64)]),
            counters([], mismatches=0, claims=0, bits=[U64 if b == 0 else 0 for b in range(64)])]
    gran = [[0b1011, 1 << 63], [0, 0], [U64, U64]]
    call = locate_call(S0, [lpass(3, (5, 6)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)], [[], [], []], CF,
                       ctrs=ctrs, granules=gran)
    r, _ = check_locate(cro, call)
    assert r["bit_flips"][5] == 3 and r["bit_flips"][63] == 2 and r["bit_flips"][0] == U64
    assert r["flip_or"] == 1 | 1 << 5 | 1 << 63
    assert [P["granules"] for P in r["pass_"]] == [4, 0, 128]


@pytest.mark.parametrize("mism,verdict,status", [
    ((0,), "NONE", "OK"), ((2,), "UNCLASSIFIED", "ERR_CHECKSUM"), ((0, 0, 0), "NONE", "OK"),
    ((2, 0, 0), "NOT_REPRODUCED", "ERR_CHECKSUM"), ((0, 0, 1), "PERSISTENT", "ERR_CHECKSUM"),
    ((0, 1, 0), "PERSISTENT", "ERR_CHECKSUM")])
def test_the_verdict_and_the_status(cro, mism, verdict, status):
    passes = [lpass(1, (5, 0)), lpass(3, (8, 8)), lpass(3, (8, 8), invert=U64)][:len(mism)]
    ctrs = [counters([], mismatches=m, claims=0) for m in mism]
    call = locate_call(S0, passes, [[] for _ in mism], CF[:2], ctrs=ctrs)
    r, _ = check_locate(cro, call)
    assert (r["verdict"], r["status"]) == (getattr(cro, "FAULTS_" + verdict), getattr(cro, status))


def random_locate_call(rng):
    n = rng.choice([1, 2, 3, 511, 512, 1 << 20, (1 << 36) - 1])
    np_ = rng.choice([1, 1, 3])
    passes = [lpass(rng.choice([0, 1, 2, 3]), (rng.choice([5, 6]), rng.choice([5, 6])))]
    r = rng.choice([8, 5])
    passes += [lpass(3, (r, r), invert=U64 * (p == 2)) for p in range(1, np_)]
    if rng.random() < 0.05:
        passes[0]["skipped"] = rng.randrange(4)
    recs, ctrs = [], []
    for p in range(np_):
        k = rng.choice([0, 0, 1, 2, 7]) if rng.random() < 0.97 else RECORDS
        words = rng.sample(range(2 * n), min(k, 2 * n)) if rng.random() < 0.5 else [rng.randrange(2 * n) for _ in range(k)]
        rr = [record(w, rng.randrange(1 << 64), rng.randrange(1 << 64)) for w in words]
        if p and recs[0] and len(rr) < RECORDS and rng.random() < 0.3:
            rr.append(dict(recs[0][0]))                                   # a word two passes saw
        recs.append(rr)
        c = counters(rr)
        if rng.random() < 0.15:
            c["claims"] = c["mismatches"] = len(rr) + rng.choice([1, 5000])
            if len(rr) < RECORDS:
                c["claims"] = len(rr)
        if rng.random() < 0.1:
            c["bits"] = [rng.randrange(3) for _ in range(64)]
        ctrs.append(c)
    cf = [(rng.randrange(1 << 64), rng.randrange(1 << 64), rng.randrange(1 << 64)) for _ in range(3)]
    folds = {}
    for p in range(np_):
        for h in range(2):
            if rng.random() < 0.1:
                folds[(p, h)] = (rng.randrange(1 << 64), rng.randrange(1 << 64), rng.randrange(1 << 64))
    gw = rng.choice([0, 1, 3])
    gran = [[rng.randrange(1 << 64) if rng.random() < 0.3 else 0 for _ in range(gw)] for _ in range(np_)]
    call = locate_call(8 * n, passes, recs, cf, folds=folds, ctrs=ctrs, granules=gran,
                       cap=rng.choice([None, None, 0, 1, 3]))
    for i in range(9):
        if rng.random() < 0.05:
            call["slots"][i]["n_words"] = rng.randrange(1 << 64)
    return call


def test_random_locate_calls_equal_the_restatement(cro):
    rng = random.Random(20261016)
    seen = set()
    for _ in range(500):
        r, _ = check_locate(cro, random_locate_call(rng))
        seen.add((r["verdict"], r["complete"]))
    assert {v for v, _ in seen} == {cro.FAULTS_NONE, cro.FAULTS_UNCLASSIFIED, cro.FAULTS_NOT_REPRODUCED,
                                    cro.FAULTS_PERSISTENT} and {c for _, c in seen} == {0, 1}, seen


# ---- the scan ---------------------------------------------------------------------------------------------------------
def scan_call(chunk_bytes, recs, cf=None, elements_done=4, cuda_error=0, ctrs=None, folds=None, granules=None, cap=None):
    """A scan over chunks of the given sizes, back to back from word 0; each chunk's fold in pass p is its closed form
    (complemented over its own words in pass 1) changed by its records, unless folds[(p, k)] says otherwise."""
    chunks, at = [], 0
    for b in chunk_bytes:
        chunks.append((at, b))
        at += b // 8
    cf = cf or [(0x1000 + k, 0x2000 + k, 0x3000 + k) for k in range(len(chunks))]
    slots = [slot() for _ in range(3 * 128)]
    for k, (w0, b) in enumerate(chunks):
        slots[256 + k] = slot(cf[k], b // 8)
        for p in range(2):
            c = faults.complement_fold(cf[k], b // 8) if p else cf[k]
            mine = [r for r in recs[p] if w0 <= r["word"] < w0 + b // 8]
            f = (folds or {}).get((p, k)) or changed(c, mine, lambda w: w - w0)
            slots[p * 128 + k] = slot(f, b // 8)
    return dict(chunks=chunks, elements_done=elements_done, cuda_error=cuda_error,
                counters=ctrs or [counters(r) for r in recs], records=recs, granules=granules or [[0, 0], [0, 0]],
                slots=slots, cap=sum(len(r) for r in recs) if cap is None else cap)


def check_scan(cro, call):
    c, r = hook_lists(cro, call)
    got_r, got_w = cro.selftest_scan_collect(call["chunks"], call["elements_done"], call["cuda_error"], c, r, call["granules"],
                                             [mk(cro.SweepSlot, s) for s in call["slots"]], cap=call["cap"])
    want_r, want_w = scan.collect(call)
    d = plain(got_r)
    blank_chunk = dict(word0=0, bytes=0, fold_xor=[0, 0], fold_sum=[0, 0], fold_wsum=[0, 0], expect_xor=0, expect_sum=0,
                       expect_wsum=0)
    assert d.pop("chunk") == want_r.pop("chunk") + [blank_chunk] * (128 - len(call["chunks"]))
    health = dict(nvml=0, remap_corrected=0, remap_uncorrected=0, remap_pending=0, remap_failure=0, histogram=[0] * 5,
                  ecc_corrected=0, ecc_uncorrected=0)
    device_only = dict(health=0, seed=0, total_bytes=0, free_bytes=0, held_bytes=0, element_ns=[0] * 4, alloc_ns=0,
                       nvml_ns=0, wall_ns=0, helper_ns=0, before=health, after=health)
    for f, v in device_only.items():
        assert d.pop(f) == v, f
    assert d == want_r
    got_w = [plain(w) for w in got_w]
    assert got_w == want_w
    return plain(got_r), got_w


CHUNK = 1 << 12                                    # 512 words


def test_a_record_at_a_chunks_first_word_belongs_to_that_chunk(cro):
    """Chunk k starts at word0_k: that word is chunk k's (its offset 0), the word before it chunk k - 1's last."""
    w1 = CHUNK // 8
    recs = [record(w1 - 1, 1, 2), record(w1, 3, 5), record(2 * w1, 0, 9), record(3 * w1 - 1, 7, 0)]
    call = scan_call([CHUNK, CHUNK, CHUNK], [recs, []])
    r, words = check_scan(cro, call)
    assert [(w["word_index"], w["reserved"]) for w in words] == [(w1 - 1, 0), (w1, 1), (2 * w1, 2), (3 * w1 - 1, 2)]
    assert r["complete"] == 1 and r["status"] == cro.ERR_CHECKSUM


def test_the_ragged_last_chunk_complements_over_its_own_words(cro):
    """Pass 1 (E3) compares with ~P: the ragged chunk's closed form is complemented over its own n, odd here."""
    recs = [record(2 * (CHUNK // 8) + 2, 0, 1)]
    call = scan_call([CHUNK, CHUNK, 24], [[], recs])
    r, _ = check_scan(cro, call)
    assert r["complete"] == 1 and r["covered_bytes"] == 2 * CHUNK + 24
    w0, cf = 2 * CHUNK // 8, (0x1002, 0x2002, 0x3002)
    assert r["chunk"][2]["fold_sum"][1] == changed(faults.complement_fold(cf, 3), recs, lambda w: w - w0)[1]
    # the same chunk complemented over the whole scan's words is not explained
    call = scan_call([CHUNK, CHUNK, 24], [[], recs],
                     folds={(1, 2): changed(faults.complement_fold(cf, w0 + 3), recs, lambda w: w - w0)})
    assert check_scan(cro, call)[0]["complete"] == 0


@pytest.mark.parametrize("done", range(5))
def test_a_cuda_error_keeps_what_the_scan_got_to(cro, done):
    """An error that stopped the scan after `done` elements: below E2 nothing is collected; at 2 or 3 only pass 0 (E1);
    at 4 both passes, without closed forms.  The status is CRO_ERR_CUDA and the report never complete."""
    recs = [[record(5, 1, 0)], [record(9, 0, 1 << 9)]]
    call = scan_call([CHUNK, CHUNK], recs, elements_done=done, cuda_error=719)
    r, words = check_scan(cro, call)
    assert (r["status"], r["cuda_error"], r["complete"]) == (cro.ERR_CUDA, 719, 0)
    ran = [] if done < 2 else [0] if done < 4 else [0, 1]
    assert [P["mismatches"] for P in r["pass_"]] == [1 if p in ran else 0 for p in range(2)]
    assert [w["word_index"] for w in words] == [[5, 9][p] for p in ran]
    assert [P["invert"] for P in r["pass_"]] == [0, U64 if 1 in ran else 0]
    assert r["flip_or"] == sum([1, 1 << 9][p] for p in ran)
    # without closed forms, expect_* stays 0 even where a pass was collected
    assert all(K["expect_xor"] == K["expect_sum"] == K["expect_wsum"] == 0 for K in r["chunk"])


def test_a_whole_scan_without_an_error(cro):
    recs = [[record(5, 1, 0)], [record(9, 0, 1 << 9)]]
    r, _ = check_scan(cro, scan_call([CHUNK, CHUNK], recs))
    assert (r["status"], r["cuda_error"], r["complete"]) == (cro.ERR_CHECKSUM, 0, 1)
    assert r["chunk"][1]["expect_xor"] == 0x1001
    r, _ = check_scan(cro, scan_call([CHUNK], [[], []]))
    assert (r["status"], r["complete"], r["located"]) == (cro.OK, 1, 0)


def test_flip_or_comes_from_the_counters(cro):
    """A storm past the record cap: the records show bit 0 flipped, and the exact counters also bit 40, which only
    unrecorded words flipped."""
    recs = [record(i, 0, 1) for i in range(RECORDS)]
    bits = [0] * 64
    bits[0], bits[40] = RECORDS, 900
    ctrs = [counters(recs, mismatches=RECORDS + 900, claims=RECORDS + 900, bits=bits), counters([])]
    r, _ = check_scan(cro, scan_call([1 << 16], [recs, []], ctrs=ctrs))
    assert r["flip_or"] == 1 | 1 << 40
    assert (r["pass_"][0]["recorded"], r["complete"]) == (RECORDS, 0)


def random_scan_call(rng):
    nc = rng.choice([1, 2, 3, 128])
    sizes = [rng.choice([8, 16, 24, CHUNK, 1 << 20, (1 << 31)]) for _ in range(nc)]
    total = sum(sizes) // 8
    starts = [0]
    for b in sizes[:-1]:
        starts.append(starts[-1] + b // 8)
    recs, ctrs = [], []
    for p in range(2):
        k = rng.choice([0, 0, 1, 2, 9]) if rng.random() < 0.97 else RECORDS
        pool = starts + [s - 1 for s in starts[1:]] + [total - 1]
        words = [rng.choice(pool) if rng.random() < 0.5 else rng.randrange(total) for _ in range(k)]
        rr = [record(w, rng.randrange(1 << 64), rng.randrange(1 << 64)) for w in words]
        recs.append(rr)
        c = counters(rr)
        if rng.random() < 0.15 and len(rr) == RECORDS:
            c["claims"] = c["mismatches"] = RECORDS + rng.randrange(1, 10000)
            c["bits"] = [b + rng.choice([0, 0, 5]) for b in c["bits"]]
        ctrs.append(c)
    folds = {(p, k): (rng.randrange(1 << 64), 1, 2) for p in range(2) for k in range(nc) if rng.random() < 0.03}
    done, err = (4, 0) if rng.random() < 0.6 else (rng.randrange(5), rng.choice([0, 2, 214, 719]))
    gran = [[rng.randrange(1 << 64) if rng.random() < 0.2 else 0 for _ in range(2)] for _ in range(2)]
    call = scan_call(sizes, recs, elements_done=done, cuda_error=err, ctrs=ctrs, folds=folds, granules=gran,
                     cap=rng.choice([None, None, 0, 2]))
    return call


def test_random_scan_calls_equal_the_restatement(cro):
    rng = random.Random(20261018)
    seen = set()
    for _ in range(500):
        r, _ = check_scan(cro, random_scan_call(rng))
        seen.add((r["status"], r["complete"]))
    assert seen >= {(cro.OK, 1), (cro.ERR_CHECKSUM, 1), (cro.ERR_CHECKSUM, 0), (cro.ERR_CUDA, 0)}, seen


# ---- the host link ----------------------------------------------------------------------------------------------------
SEEDS = [0x51, 0x52, 0x53]
PAT_CF = [(0xA1, 0xB1, 0xC1), (0xA2, 0xB2, 0xC2), (0xA3, 0xB3, 0xC3)]


def link_call(L, recs, ctrs=None, folds=None, chase=None, hops=16, host=None, cap=None, coracle=None):
    """A link call of L bytes: each check's fold is its pattern's closed form changed by its records (unless folds[k]
    says otherwise), the chase ended where the host walk does, and each host buffer holds the records' actual
    values."""
    n = L // 8
    slots = [slot() for _ in range(10)]
    for j in range(3):
        slots[7 + j] = slot(PAT_CF[j], n)
    for k in range(5):
        f = (folds or {}).get(k) or changed(PAT_CF[link.CHECK_PATTERN[k]], recs[k], lambda w: w)
        slots[k] = slot(f, n)
    if host is None:
        host = [[0x77] * n for _ in range(5)]
        for k in range(5):
            for r in recs[k]:
                if r["word"] < n:
                    host[k][r["word"]] = r["actual"]
    if chase is None:
        chase = [coracle.chase_end(MINOR, MINOR, hops), 12345]
    return dict(bytes=L, seeds=SEEDS, minor=MINOR, hops=hops, counters=ctrs or [counters(r) for r in recs], records=recs,
                host=host, slots=slots, chase_out=chase, cap=sum(len(r) for r in recs) if cap is None else cap)


def check_link(cro, coracle, call):
    c, r = hook_lists(cro, call)
    got_r, got_f = cro.selftest_link_classify(call["bytes"], call["seeds"], call["minor"], call["hops"], c, r, call["host"],
                                              [mk(cro.SweepSlot, s) for s in call["slots"]], call["chase_out"],
                                              cap=call["cap"])
    want_r, want_f = link.classify(call, coracle.chase_end)
    d = plain(got_r)
    hop = dict(bdf=b"", cur_speed=0, cur_width=0, max_speed=0, max_width=0)
    device_only = dict(call=0, leg=[dict(bytes=0, ns=0, timer_ns=0)] * 8, ce_duplex_span_ns=0, dev_numa=-1,
                       host_numa=[-1, -1, -1], no_nvml=0, degraded=0, replays_before=0, replays_after=0,
                       path=dict(numa_node=-1, n_hops=0, bottleneck=0, truncated=0, hop=[hop] * 8))
    for f, v in device_only.items():
        assert d.pop(f) == v, f
    assert d == want_r
    got_f = [plain(f) for f in got_f]
    assert got_f == want_f
    return plain(got_r), got_f


def test_several_failing_checks_name_the_lowest(cro, coracle):
    recs = [[], [], [record(4, 1, 0)], [], [record(0, 2, 3)]]
    r, faults_ = check_link(cro, coracle, link_call(64, recs, coracle=coracle))
    assert r["first_fail"] == 2 and r["status"] == cro.ERR_CHECKSUM
    assert [(f["check"], f["word_index"]) for f in faults_] == [(2, 4), (4, 0)]
    r, _ = check_link(cro, coracle, link_call(64, recs, folds={3: (1, 2, 3)}, coracle=coracle))
    assert r["first_fail"] == 2


def test_a_stale_slot_fails_with_no_mismatch(cro, coracle):
    """A read slot whose n_words is another call's (its kernel did not run) fails the check although the fold matches
    and nothing mismatched; so does a stale closed form (P3's reaches only check 3)."""
    call = link_call(64, [[]] * 5, coracle=coracle)
    call["slots"][1]["n_words"] = 7
    r, _ = check_link(cro, coracle, call)
    assert (r["first_fail"], r["check"][1]["mismatches"]) == (1, 0)
    call = link_call(64, [[]] * 5, coracle=coracle)
    call["slots"][9]["n_words"] = 0
    assert check_link(cro, coracle, call)[0]["first_fail"] == 3
    r, _ = check_link(cro, coracle, link_call(64, [[]] * 5, coracle=coracle))
    assert (r["first_fail"], r["status"], r["chase_ns"]) == (cro.LINK_NO_FAIL, cro.OK, 12345)


def test_a_fold_only_failure(cro, coracle):
    call = link_call(4096 + 16, [[]] * 5, folds={4: (PAT_CF[0][0], PAT_CF[0][1], PAT_CF[0][2] + 1)}, coracle=coracle)
    r, faults_ = check_link(cro, coracle, call)
    assert (r["first_fail"], r["check"][4]["mismatches"], faults_) == (4, 0, [])


def test_an_armed_chase_output(cro, coracle):
    """The chase did not publish: no time, and a failure only when no word check failed first."""
    r, _ = check_link(cro, coracle, link_call(64, [[]] * 5, chase=[U64, U64], coracle=coracle))
    assert (r["first_fail"], r["chase_ns"], r["chase_end"]) == (cro.LINK_CHECK_CHASE, 0, 0xFFFFFFFF)
    r, _ = check_link(cro, coracle, link_call(64, [[], [], [], [record(1, 0, 1)], []], chase=[U64, U64], coracle=coracle))
    assert (r["first_fail"], r["chase_ns"]) == (3, 0)
    r, _ = check_link(cro, coracle, link_call(64, [[]] * 5, chase=[5, 99], hops=1 << 24, coracle=coracle))
    assert r["first_fail"] == cro.LINK_CHECK_CHASE and r["chase_ns"] == 99


def test_faults_are_sorted_per_check_capped_and_read_the_host_buffer(cro, coracle):
    L = 1 << 15
    n = L // 8
    rng = random.Random(7)
    words = rng.sample(range(2 * n), RECORDS)                  # some past L / 8: no host word there
    recs = [[], [], [record(w, w, w ^ 1) for w in words], [], []]
    ctrs = [counters(r) for r in recs]
    ctrs[2]["claims"] = ctrs[2]["mismatches"] = 5000
    r, faults_ = check_link(cro, coracle, link_call(L, recs, ctrs=ctrs, coracle=coracle))
    assert [f["word_index"] for f in faults_] == sorted(words)
    assert all(f["host_value"] == (f["actual"] if f["word_index"] < n else 0) for f in faults_)
    assert (r["check"][2]["recorded"], r["check"][2]["mismatches"]) == (RECORDS, 5000)
    r, faults_ = check_link(cro, coracle, link_call(L, recs, ctrs=ctrs, cap=10, coracle=coracle))
    assert [f["word_index"] for f in faults_] == sorted(words)[:10]


def random_link_call(rng, coracle):
    L = rng.choice([16, 64, 4096 + 16])
    n = L // 8
    recs, ctrs = [], []
    for k in range(5):
        m = rng.choice([0, 0, 0, 1, 3]) if rng.random() < 0.98 else RECORDS
        rr = [record(w, rng.randrange(1 << 64), rng.randrange(1 << 64)) for w in rng.sample(range(RECORDS + n + 8), m)]
        recs.append(rr)
        c = counters(rr)
        if rng.random() < 0.05:
            c["mismatches"] = rng.randrange(1 << 64)
            if len(rr) == RECORDS:
                c["claims"] = RECORDS + rng.randrange(1, 100)
        ctrs.append(c)
    folds = {k: (rng.randrange(1 << 64), 0, 0) for k in range(5) if rng.random() < 0.05}
    hops = rng.choice([1, 2, 1024, 65536])
    chase = rng.choice([None, None, None, [U64, U64], [rng.randrange(1 << 17), rng.randrange(1 << 64)]])
    host = [[rng.randrange(1 << 64) for _ in range(n)] for _ in range(5)] if rng.random() < 0.5 else None
    call = link_call(L, recs, ctrs=ctrs, folds=folds, chase=chase, hops=hops, host=host, cap=rng.choice([None, 0, 2]),
                     coracle=coracle)
    for i in list(range(5)) + [7, 8, 9]:
        if rng.random() < 0.03:
            call["slots"][i]["n_words"] = rng.randrange(n + 2)
    return call


def test_random_link_calls_equal_the_restatement(cro, coracle):
    rng = random.Random(20261019)
    seen = set()
    for _ in range(500):
        r, _ = check_link(cro, coracle, random_link_call(rng, coracle))
        seen.add(r["first_fail"])
    assert seen == {0, 1, 2, 3, 4, 5, cro.LINK_NO_FAIL}, seen


# ---- the C ABI --------------------------------------------------------------------------------------------------------
FIELDS = {
    "cro_locate_counters": ("LocateCounters", ["mismatches", "claims", "bits"]),
    "cro_locate_record": ("LocateRecord", ["word", "expected", "actual"]),
    "cro_sweep_slot": ("SweepSlot", ["x", "s", "w", "t0", "t1", "stamp", "n_words", "pad"]),
    "cro_opts": ("Opts", ["abi_version", "flags", "sweep_bytes", "p2p_bytes", "seed_base", "read_sweeps", "copy_sweeps",
                          "latency_hops", "read_variant", "copy_variant", "deadline_ms", "n_devices", "devices", "rank_base",
                          "world_override", "test_inject_after", "test_inject_count", "test_inject_word", "test_inject_mask"]),
}


def test_ctypes_layout_of_the_mirrors_matches_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = {}
    for ln in subprocess.check_output([str(exe)], text=True).splitlines():
        name, field, v = ln.split()
        got[(name, field)] = int(v)
    for cname, (py, fields) in FIELDS.items():
        cls = getattr(cro, py)
        assert ctypes.sizeof(cls) == got[(cname, "sizeof")], cname
        assert [f for f, _ in cls._fields_] == fields, cname
        for f in fields:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)


def test_a_slots_mismatch_count_is_the_word_its_pad_was(cro, tmp_path):
    """cro_sweep_slot.mismatches and .pad name one word, the slot's last; the ctypes mirror reads it as mismatches."""
    c = tmp_path / "slot.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "croprobe.h"\nint main(void) {\n'
                 'cro_sweep_slot s = {0};\ns.pad = 7;\nprintf("%zu %zu %zu %llu\\n", offsetof(cro_sweep_slot, mismatches), '
                 'offsetof(cro_sweep_slot, pad), sizeof s, (unsigned long long)s.mismatches);\nreturn 0; }\n')
    exe = tmp_path / "slot"
    subprocess.check_call(["gcc", "-std=c11", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).split() == ["56", "56", "64", "7"]
    assert cro.SweepSlot(pad=1 << 40).mismatches == 1 << 40 and cro.SweepSlot.pad.offset == 56


def test_locate_hook_refuses_bad_arguments(cro):
    lib = cro.lib
    passes = (cro.LocatePass * 3)(*[mk(cro.LocatePass, lpass(3, (5, 5))) for _ in range(3)])
    ctr, recs, gran = (cro.LocateCounters * 3)(), (cro.LocateRecord * 4)(), (ctypes.c_uint64 * 8)()
    slots, out, words, n = (cro.SweepSlot * 9)(), cro.FaultReport(), (cro.FaultWord * 4)(), ctypes.c_int(-1)

    def call(**kw):
        a = dict(S=4096, passes=passes, np=3, ctr=ctr, recs=recs, gran=gran, gw=2, slots=slots, out=ctypes.byref(out),
                 words=words, cap=4, n=ctypes.byref(n))
        a.update(kw)
        return lib.cro_selftest_locate_collect(*a.values())
    assert call() == cro.OK and n.value == 0
    for kw in (dict(S=0), dict(S=12), dict(np=0), dict(np=4), dict(passes=None), dict(ctr=None), dict(slots=None),
               dict(out=None), dict(n=None), dict(cap=-1), dict(words=None), dict(gw=8193), dict(gran=None)):
        assert call(**kw) == cro.ERR_INVALID_ARG, kw
    assert call(gran=None, gw=0) == cro.OK and call(words=None, cap=0) == cro.OK and call(S=8) == cro.OK
    passes[2].halves = 4
    assert call() == cro.ERR_INVALID_ARG and call(np=2) == cro.OK               # pass 2 not run: not read
    passes[2].halves = 3
    passes[0].seed[1], passes[1].seed[1], passes[2].seed[1] = 6, 7, 8
    assert call() == cro.ERR_INVALID_ARG                                        # four closed forms for three slots
    assert out.status == cro.ERR_INVALID_ARG
    assert call(np=2) == cro.OK
    ctr[1].claims = 1
    assert call(recs=None) == cro.ERR_INVALID_ARG and call(recs=None, np=1) == cro.OK


def test_scan_hook_refuses_bad_arguments(cro):
    lib = cro.lib
    ctr, recs, gran = (cro.LocateCounters * 2)(), (cro.LocateRecord * 4)(), (ctypes.c_uint64 * 4)()
    slots, out, words, n = (cro.SweepSlot * cro.SCAN_SLOTS)(), cro.ScanReport(), (cro.FaultWord * 4)(), ctypes.c_int(-1)

    def call(chunks=((0, 64), (8, 32)), done=4, **kw):
        out.n_chunks, out.elements_done = len(chunks), done
        for k, (w0, b) in enumerate(chunks[:cro.SCAN_MAX_CHUNKS]):
            out.chunk[k].word0, out.chunk[k].bytes = w0, b
        a = dict(err=0, ctr=ctr, recs=recs, gran=gran, gw=2, slots=slots, out=ctypes.byref(out), words=words, cap=4,
                 n=ctypes.byref(n))
        a.update(kw)
        return lib.cro_selftest_scan_collect(*a.values())
    assert call() == cro.OK
    for chunks, done in ((((0, 64), (8, 32)), 5), ((), 4), (((1, 64),), 4), (((0, 64), (7, 32)), 4), (((0, 64), (9, 32)), 4),
                         (((0, 0),), 4), (((0, 12),), 4), (((0, (8 << 37) + 8),), 4), (tuple((k, 8) for k in range(129)), 4)):
        assert call(chunks, done) == cro.ERR_INVALID_ARG, (chunks, done)
    for kw in (dict(ctr=None), dict(slots=None), dict(out=None), dict(n=None), dict(cap=-1), dict(words=None),
               dict(gw=8193), dict(gran=None)):
        assert call(**kw) == cro.ERR_INVALID_ARG, kw
    assert call(((0, 8 << 37),)) == cro.OK and call(((0, 8),), 0) == cro.OK and call(words=None, cap=0) == cro.OK
    ctr[1].claims = 2
    assert call(recs=None) == cro.ERR_INVALID_ARG


def test_link_hook_refuses_bad_arguments(cro):
    lib, u64 = cro.lib, ctypes.c_uint64
    seeds, ctr, recs = (u64 * 3)(1, 2, 3), (cro.LocateCounters * 5)(), (cro.LocateRecord * 4)()
    host, slots, chase = (u64 * 40)(), (cro.SweepSlot * cro.LINK_SLOTS)(), (u64 * 2)()
    out, faults_, n = cro.LinkResult(), (cro.LinkFault * 4)(), ctypes.c_int(-1)

    def call(**kw):
        a = dict(L=64, seeds=seeds, minor=0, hops=4, ctr=ctr, recs=recs, host=host, slots=slots, chase=chase,
                 out=ctypes.byref(out), faults=faults_, cap=4, n=ctypes.byref(n))
        a.update(kw)
        return lib.cro_selftest_link_classify(*a.values())
    assert call() == cro.ERR_CHECKSUM                   # zero slots cover no words: every check fails
    for kw in (dict(L=0), dict(L=8), dict(L=24), dict(hops=0), dict(hops=(1 << 24) + 1), dict(seeds=None), dict(ctr=None),
               dict(host=None), dict(slots=None), dict(chase=None), dict(out=None), dict(n=None), dict(cap=-1),
               dict(faults=None)):
        assert call(**kw) == cro.ERR_INVALID_ARG, kw
    assert call(hops=1 << 24) == cro.ERR_CHECKSUM and call(faults=None, cap=0) == cro.ERR_CHECKSUM
    ctr[4].claims = 1
    assert call(recs=None) == cro.ERR_INVALID_ARG
