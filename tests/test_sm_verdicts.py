"""The compute, precision and SRAM probes' verdicts without a GPU: the library's classification of caller-given rounds
and records (cro_selftest_sm_legs_classify, cro_selftest_sram_classify, which run the same host code as a probe call)
against the restatements written from include/croprobe.h (oracle/sm_legs.py, oracle/sram.py), field for field.

Each rule a healthy H100 cannot reach by software injection has a hand-built case that also pins the expected value;
a seeded sweep of synthetic calls covers the rest."""
import ctypes
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = (1 << 64) - 1
ARMED = U64                                # a CTA that did not publish leaves its record armed
SILENT = 0xFFFFFFFF
COMPUTE_OPS = 2 * 128 * 256 * 256


# ---- plumbing ---------------------------------------------------------------------------------------------------------
def plain(x):
    """A ctypes value as plain Python: structures as dicts, arrays as lists."""
    if isinstance(x, ctypes.Structure):
        return {f: plain(getattr(x, f)) for f, _ in x._fields_}
    if isinstance(x, ctypes.Array):
        return [plain(v) for v in x]
    return x


def cta(k, smid, **kw):
    d = dict(stamp=k, t0=1000, t1=2000, cycles=5000, mismatches=0, fold_mismatches=0, fold=0, smid=smid, nsmid=132)
    d.update(kw)
    return d


def bitmap(smids):
    w = [0, 0, 0, 0]
    for s in smids:
        w[s // 64] |= 1 << (s % 64)
    return w


def covered_rounds(per_round):
    """(ctas, bits) per round, with bits the cumulative coverage of the CTAs that published so far."""
    seen, out = set(), []
    for ctas in per_round:
        seen |= {c["smid"] for c in ctas if c["stamp"] != ARMED}
        out.append((ctas, bitmap(seen)))
    return out


def sm_call(n_legs, grid, k, rounds, legs=0, iterations=None, claims=None, records=None):
    return {"legs": legs, "iterations": iterations or [4] * n_legs, "grid": grid, "call": k,
            "rounds": rounds, "claims": claims or [0] * n_legs, "records": records or [[] for _ in range(n_legs)]}


def run_sm(cro, probe, call):
    """The library's (result, sms, faults) for a call, as plain dicts."""
    n_legs = cro.COMPUTE_LEGS if probe == cro.SM_LEGS_COMPUTE else cro.PRECISION_LEGS
    fault = cro.ComputeFault if probe == cro.SM_LEGS_COMPUTE else cro.PrecisionFault
    rounds = [[([cro.SmCta(**c) for c in ctas], bits) for ctas, bits in call["rounds"][l]] for l in range(n_legs)]
    records = [[fault(**f) for f in call["records"][l]] for l in range(n_legs)]
    r, sms, faults = cro.selftest_sm_legs_classify(probe, call["iterations"], call["grid"], call["call"], rounds,
                                                   call["claims"], records, legs=call["legs"])
    return plain(r), [plain(s) for s in sms], [plain(f) for f in faults]


def check_sm(cro, probe, call):
    """The library and the restatement agree on every field; returns the library's answer."""
    import compute
    import precision
    got = run_sm(cro, probe, call)
    want = (compute if probe == cro.SM_LEGS_COMPUTE else precision).classify(call)
    assert got[0] == want[0]
    assert got[1] == want[1]
    key = lambda f: (f["leg"], f["smid"], f["row"], f["col"])
    assert [key(f) for f in got[2]] == sorted(key(f) for f in got[2])
    full = lambda f: sorted(f.items())
    assert sorted(got[2], key=full) == sorted(want[2], key=full)
    return got


def sram_cta(k, smid, block=0, rank=0, fold=(0, 0, 0), **kw):
    d = dict(stamp=k, t0=1000, t1=2000, cycles=7000, count=[0] * 6, last=0, fold_x=fold[0], fold_s=fold[1], fold_w=fold[2],
             smid=smid, nsmid=132, rank=rank, block=block)
    d.update(kw)
    return d


def sram_record(element, smid, peer_block=0, round=0, word=5, iteration=0, expected=1, actual=3):
    return dict(element=element, iteration=iteration, smid=smid, peer_block=peer_block, round=round, word=word,
                expected=expected, actual=actual)


def run_sram(cro, call):
    def mk(cls, d):
        x = cls()
        for f, v in d.items():
            if isinstance(v, list):
                getattr(x, f)[:] = v
            else:
                setattr(x, f, v)
        return x
    rounds = [[[mk(cro.SramCta, c) for c in ctas] for ctas in call["rounds"][l]] for l in range(2)]
    records = [[mk(cro.SramRecord, q) for q in call["records"][l]] for l in range(2)]
    r, sms, faults = cro.selftest_sram_classify(call["iterations"], call["n_words"], call["seed"], call["cluster"],
                                                call["sm_count"], call["net_grid"], call["call"], rounds, call["claims"],
                                                records, legs=call["legs"])
    d = plain(r)
    d["bad_pair"] = [(p["from_"], p["owner"], p["direction"]) for p in d["bad_pair"]]
    return d, [plain(s) for s in sms], [plain(f) for f in faults]


def check_sram(cro, coracle, call):
    import sram
    got = run_sram(cro, call)
    want = sram.classify(call, coracle.checksum)
    r = dict(got[0])
    device_only = {"cuda_error": 0, "health": 0, "wall_ns": 0, "helper_ns": 0,
                   "before": dict(nvml=0, threshold_exceeded=0, ecc_corrected=0, ecc_uncorrected=0)}
    device_only["after"] = device_only["before"]
    for f, v in device_only.items():
        assert r.pop(f) == v, f
    assert r.pop("sms_listed") == len(got[1]) and r.pop("recorded") == len(got[2])
    assert r == want[0]
    assert got[1] == want[1]
    key = lambda f: (f["leg"], f["element"], f["smid"], f["iteration"], f["word"])
    assert [key(f) for f in got[2]] == sorted(key(f) for f in got[2])
    full = lambda f: sorted(f.items())
    assert sorted(got[2], key=full) == sorted(want[2], key=full)
    return got


def sram_call(k, sm_count, net_grid, cluster, rounds, legs=0, claims=(0, 0), records=([], []), n_words=64, iterations=2,
              seed=0x1234):
    return {"legs": legs, "iterations": iterations, "n_words": n_words, "seed": seed, "cluster": cluster,
            "sm_count": sm_count, "net_grid": net_grid, "call": k, "rounds": rounds, "claims": list(claims),
            "records": [list(records[0]), list(records[1])]}


def local_fold(coracle, call):
    import sram
    return sram.m5_fold(coracle.checksum, call["seed"], call["n_words"], call["iterations"])


# ---- compute and precision: hand-built cases -------------------------------------------------------------------------
def one_leg(cro, per_round, k=7, grid=4, leg=0, iterations=4, **kw):
    rounds = [[] for _ in range(cro.COMPUTE_LEGS)]
    rounds[leg] = covered_rounds(per_round)
    its = [4] * cro.COMPUTE_LEGS
    its[leg] = iterations
    return sm_call(cro.COMPUTE_LEGS, grid, k, rounds, legs=1 << leg, iterations=its, **kw)


def test_an_unpublished_cta_is_a_common_cause(cro):
    k = 7
    call = one_leg(cro, [[cta(k, 0), cta(k, 1), cta(ARMED, 2), cta(k, 3)]])
    r, sms, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    assert r["leg"][0]["unpublished"] == 1 and r["leg"][0]["failed_sms"] == 0 and r["leg"][0]["sms_covered"] == 3
    assert (r["status"], r["verdict"], r["bad_sms"]) == (cro.ERR_CHECKSUM, cro.COMPUTE_ALL, 0)
    assert [s["smid"] for s in sms] == [0, 1, 3]
    # a record stamped for another call did not publish either
    call = one_leg(cro, [[cta(k, 0), cta(k + 1, 1), cta(k, 2), cta(k, 3)]])
    assert check_sm(cro, cro.SM_LEGS_COMPUTE, call)[0]["verdict"] == cro.COMPUTE_ALL


def test_an_sm_bad_in_one_round_and_clean_in_another_keeps_its_mark(cro):
    k = 9
    for bad, mark in ((dict(mismatches=3, fold_mismatches=1), cro.COMPUTE_PERSISTENT),
                      (dict(fold_mismatches=2), cro.COMPUTE_INTERMITTENT)):
        # round 0: SM 5 bad, SM 6 silent; round 1: SM 5 again, clean, and SM 6
        call = one_leg(cro, [[cta(k, 4), cta(k, 5, **bad), cta(ARMED, 6)],
                             [cta(k, 4), cta(k, 5), cta(k, 6)]], k=k, grid=3)
        r, sms, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
        (s5,) = [s for s in sms if s["smid"] == 5]
        assert s5["leg"][0]["ctas"] == 2 and s5["leg"][0]["mark"] == mark
        assert r["leg"][0]["rounds"] == 2 and r["leg"][0]["ctas"] == 6 and r["leg"][0]["failed_sms"] == 1
        assert r["bad_sms"] == 1 and r["bad_sm"][0] == 5 and r["verdict"] == cro.COMPUTE_ALL   # round 0's silent CTA


def test_short_coverage_with_a_failure_is_an_sm_verdict(cro):
    k = 3
    # max_rounds reached with 3 of 5 SMs seen: complete = 0, still an SM verdict
    call = one_leg(cro, [[cta(k, 0), cta(k, 1), cta(k, 0), cta(k, 1), cta(k, 2, mismatches=1)]] * 2, k=k, grid=5)
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    L = r["leg"][0]
    assert (L["sms_covered"], L["complete"], L["rounds"], L["failed_sms"]) == (3, 0, 2, 1)
    assert (r["status"], r["verdict"]) == (cro.ERR_CHECKSUM, cro.COMPUTE_SM)


def test_every_covered_sm_failing_is_all_and_one_fewer_is_sm(cro):
    k = 11
    every = [cta(k, s, mismatches=1) for s in range(4)]
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, one_leg(cro, [every], k=k))
    assert r["leg"][0]["failed_sms"] == r["leg"][0]["sms_covered"] == 4 and r["verdict"] == cro.COMPUTE_ALL
    but_one = every[:3] + [cta(k, 3)]
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, one_leg(cro, [but_one], k=k))
    assert r["leg"][0]["failed_sms"] == 3 and r["verdict"] == cro.COMPUTE_SM and r["bad_sm"][:3] == [0, 1, 2]
    # each leg on its own: SMs 0 .. 2 fail leg 0, SM 3 fails leg 1; no leg failed on every SM it covered
    rounds = [[] for _ in range(5)]
    rounds[0] = covered_rounds([but_one])
    rounds[1] = covered_rounds([[cta(k, s) for s in range(3)] + [cta(k, 3, fold_mismatches=1)]])
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, sm_call(5, 4, k, rounds, legs=3))
    assert r["verdict"] == cro.COMPUTE_SM and r["bad_sms"] == 4


def test_more_than_sixteen_bad_sms_are_counted_and_the_first_sixteen_listed(cro):
    k = 2
    smids = random.Random(5).sample(range(256), 20)
    call = one_leg(cro, [[cta(k, s, mismatches=1) for s in smids] + [cta(k, 300 - 256)]], k=k, grid=21)
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    assert r["bad_sms"] == 20 and r["bad_sm"] == sorted(smids)[:16] and r["verdict"] == cro.COMPUTE_SM


@pytest.mark.parametrize("cycles,slowest,permille", [
    ({1: 400, 2: 800, 3: 1200}, 3, 1500),                 # odd count: the middle one
    ({1: 400, 2: 800, 3: 1200, 4: 1600}, 4, 1333),        # even count: the upper of the two middle ones
    ({1: 400, 2: 1600, 3: 1600, 4: 100}, 2, 1000),        # a tie: the lowest SM id; median 1600
    ({5: 0, 6: 0, 7: 4}, 7, 0),                           # median 0: no ratio
    ({9: 0}, 9, 0),
])
def test_slowest_sm_and_its_ratio_to_the_median(cro, cycles, slowest, permille):
    k = 4
    call = one_leg(cro, [[cta(k, s, cycles=4 * c) for s, c in cycles.items()]], k=k, grid=len(cycles), iterations=4)
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    assert (r["leg"][0]["slowest_sm"], r["leg"][0]["slow_permille"]) == (slowest, permille)


def test_slowest_sm_divides_by_ctas_and_iterations(cro):
    k = 4
    # SM 1 ran two CTAs of 300 cycles: 150 a CTA; SM 2 one CTA of 200; 2 iterations each
    call = one_leg(cro, [[cta(k, 1, cycles=300), cta(k, 2, cycles=200)], [cta(k, 1, cycles=300), cta(k, 2, cycles=200)]],
                   k=k, grid=2, iterations=2)
    call["rounds"][0][1] = ([cta(k, 1, cycles=300), cta(k, 3, cycles=100)], bitmap([1, 2, 3]))
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    # per iteration: SM 1 600 / 4 = 150, SM 2 200 / 2 = 100, SM 3 100 / 2 = 50; median 100
    assert (r["leg"][0]["slowest_sm"], r["leg"][0]["slow_permille"]) == (1, 1500)


def test_the_fold_is_the_lowest_sm_ids_first_cta(cro):
    k = 6
    call = one_leg(cro, [[cta(k, 9, fold=90), cta(k, 4, fold=40), cta(k, 7, fold=70)],
                         [cta(k, 4, fold=41), cta(k, 2, fold=20), cta(k, 2, fold=21)]], k=k, grid=3)
    r, _, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    assert r["leg"][0]["fold"] == 20


def test_timer_and_ops_sum_over_rounds(cro):
    k = 1
    call = one_leg(cro, [[cta(k, 0, t0=100, t1=300), cta(k, 1, t0=150, t1=400), cta(ARMED, 2, t0=0, t1=10 ** 9)],
                         [cta(k, 2, t0=900, t1=800), cta(k, 0, t0=1000, t1=1100), cta(k, 1, t0=1000, t1=1000)]],
                   k=k, grid=3, iterations=3)
    r, sms, _ = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    L = r["leg"][0]
    assert L["timer_ns"] == 300 + 200 and L["ops"] == 2 * COMPUTE_OPS * 3 * 3 and L["ctas"] == 6
    assert [s["leg"][0]["ns"] for s in sms] == [300, 250, 0]


def test_nsmid_beyond_the_bitmaps_fails_with_a_blank_result(cro):
    for probe, n_legs in ((cro.SM_LEGS_COMPUTE, 5), (cro.SM_LEGS_PRECISION, 7)):
        k = 12
        rounds = [covered_rounds([[cta(k, 0, mismatches=2), cta(k, 1)]]) for _ in range(n_legs)]
        rounds[1] = covered_rounds([[cta(k, 0), cta(k, 1, nsmid=257)]])
        recs = [[dict(leg=0, smid=0, row=1, col=2, **({"expected": 1, "actual": 2} if probe == cro.SM_LEGS_COMPUTE else
                                                       {"expected": 1, "actual_bits": 2}))]] + [[] for _ in range(n_legs - 1)]
        call = sm_call(n_legs, 2, k, rounds, claims=[1] + [0] * (n_legs - 1), records=recs)
        r, sms, faults = check_sm(cro, probe, call)
        assert r["status"] == cro.ERR_UNSUPPORTED and r["verdict"] == 0 and not sms and not faults
        assert (r["call"], r["sm_count"], r["legs"], r["nsmid"]) == (k, 2, (1 << n_legs) - 1, 0)
        assert all(v == 0 for L in r["leg"] for v in L.values())
        # %nsmid = 256 still fits
        rounds[1] = covered_rounds([[cta(k, 0), cta(k, 255, nsmid=256)]])
        r, _, _ = check_sm(cro, probe, sm_call(n_legs, 2, k, rounds, legs=2))
        assert r["status"] == cro.OK and r["nsmid"] == 256 and r["leg"][1]["sms_covered"] == 2


def test_records_are_capped_and_sorted(cro):
    k = 5
    rng = random.Random(3)
    recs = [dict(leg=0, smid=rng.randrange(4), row=rng.randrange(128), col=rng.randrange(256), expected=1, actual=2)
            for _ in range(cro.COMPUTE_RECORDS)]
    call = one_leg(cro, [[cta(k, s, mismatches=10 ** 6) for s in range(4)]], k=k, claims=[10 ** 6, 0, 0, 0, 0],
                   records=[recs, [], [], [], []])
    r, _, faults = check_sm(cro, cro.SM_LEGS_COMPUTE, call)
    assert r["leg"][0]["recorded"] == cro.COMPUTE_RECORDS and len(faults) == cro.COMPUTE_RECORDS


# ---- compute and precision: seeded sweep -----------------------------------------------------------------------------
def random_sm_call(rng, n_legs, records_cap, precision):
    grid = rng.choice([1, 2, 3, 5, 8, 16, 33])
    k = rng.randrange(1 << 40)
    legs = rng.choice([0, 0, rng.randrange(1, 1 << n_legs)])
    pool = rng.sample(range(256), rng.choice([1, max(1, grid // 2), grid, grid + 3]))
    unsupported = rng.random() < 0.03
    rounds, claims, records, its = [], [], [], []
    for leg in range(n_legs):
        per_round = []
        for _ in range(rng.choice([0, 1, 1, 1, 2, 3, 4]) if rng.random() < 0.1 else rng.choice([1, 1, 2, 4])):
            ctas = []
            for _ in range(grid):
                smid = rng.choice(pool)
                bad = rng.random() < 0.15
                ctas.append(cta(
                    k if rng.random() < 0.93 else rng.choice([ARMED, k + 1, (k - 1) & U64]), smid,
                    t0=rng.randrange(1 << 20), t1=rng.randrange(1 << 20), cycles=rng.choice([0, 100, 1000, rng.randrange(1 << 36)]),
                    mismatches=rng.randrange(1, 1 << 20) if bad and rng.random() < 0.6 else 0,
                    fold_mismatches=rng.randrange(1, 256) if bad else 0, fold=rng.randrange(1 << 64),
                    nsmid=257 if unsupported and rng.random() < 0.05 else rng.choice([132, 132, 256])))
            per_round.append(ctas)
        rr = covered_rounds(per_round)
        if rng.random() < 0.1:                             # a bitmap that says more or fewer SMs than published
            rr = [(ctas, [rng.randrange(1 << 64) for _ in range(4)]) for ctas, _ in rr]
        rounds.append(rr)
        its.append(rng.choice([1, 2, 4, 16, 256]))
        c = rng.choice([0, 0, 0, 1, 3, 17]) if rng.random() < 0.97 else rng.choice([records_cap, records_cap + 1, 10 ** 7])
        claims.append(c)
        recs = []
        for _ in range(min(c, records_cap)):
            f = dict(leg=leg, smid=rng.choice(pool), row=rng.randrange(128), col=rng.randrange(256),
                     expected=rng.randrange(-(1 << 31), 1 << 31))
            if precision:
                f["actual_bits"] = rng.randrange(1 << 64)
            else:
                f["actual"] = rng.randrange(-(1 << 31), 1 << 31)
            recs.append(f)
        records.append(recs)
    return sm_call(n_legs, grid, k, rounds, legs=legs, iterations=its, claims=claims, records=records)


@pytest.mark.parametrize("probe", ["compute", "precision"])
def test_random_calls_equal_the_restatement(cro, probe):
    precision = probe == "precision"
    p = cro.SM_LEGS_PRECISION if precision else cro.SM_LEGS_COMPUTE
    n_legs = cro.PRECISION_LEGS if precision else cro.COMPUTE_LEGS
    rng = random.Random(20261016 + precision)
    seen = set()
    for _ in range(500):
        r, _, _ = check_sm(cro, p, random_sm_call(rng, n_legs, cro.COMPUTE_RECORDS, precision))
        seen.add((r["status"], r["verdict"]))
    assert seen >= {(cro.OK, cro.COMPUTE_NONE), (cro.ERR_CHECKSUM, cro.COMPUTE_SM), (cro.ERR_CHECKSUM, cro.COMPUTE_ALL),
                    (cro.ERR_UNSUPPORTED, cro.COMPUTE_NONE)}, seen


# ---- SRAM: hand-built cases ------------------------------------------------------------------------------------------
def net_round(k, smids, cluster, per_block=None):
    """One network round: block j on SM smids[j], with per_block[j]'s fields."""
    return [sram_cta(k, s, block=j, rank=j % cluster, **(per_block or {}).get(j, {})) for j, s in enumerate(smids)]


def test_a_write_record_names_its_writer_through_the_rounds_block_map(cro, coracle):
    """Cluster 4, two network rounds with different block maps.  Block 5 (rank 1 of cluster 1) reads Q wrong in D3: its
    writer is rank 0 (prev), block 4, and the record came from round 1, so the writer is round 1's SM at block 4."""
    k, C = 21, 4
    r0 = net_round(k, [10, 11, 12, 13, 14, 15, 16, 17], C)
    r1 = net_round(k, [20, 21, 22, 23, 24, 25, 26, 27], C, {5: dict(count=[0, 0, 0, 1, 0, 0])})
    rec = sram_record(3, smid=25, peer_block=4, round=1, word=9)
    call = sram_call(k, 16, 8, C, [[], [r0, r1]], legs=2, claims=(0, 1), records=([], [rec]))
    r, sms, faults = check_sram(cro, coracle, call)
    (f,) = faults
    assert (f["direction"], f["smid"], f["peer_smid"], f["element"]) == (cro.SRAM_DIR_WRITE, 25, 24, 3)
    assert r["bad_pairs"] == 1 and r["bad_pair"][0] == (24, 25, cro.SRAM_DIR_WRITE) and r["verdict"] == cro.SRAM_LINK
    assert r["leg"][1]["sms_covered"] == 16 and r["leg"][1]["complete"] == 1 and r["leg"][1]["cluster"] == C
    # the same record from round 0 names round 0's SM
    call["records"][1] = [sram_record(3, smid=15, peer_block=4, round=0, word=9)]
    assert check_sram(cro, coracle, call)[2][0]["peer_smid"] == 14


def test_a_silent_block_or_a_record_out_of_range_names_no_peer(cro, coracle):
    k, C = 8, 2
    r0 = net_round(k, [1, 2, 3, 4], C)
    r0[2]["stamp"] = ARMED                                 # block 2 did not publish
    recs = [sram_record(1, smid=4, peer_block=2, round=0),           # silent owner
            sram_record(1, smid=1, peer_block=4, round=0, word=6),   # block past the round's grid
            sram_record(3, smid=2, peer_block=0, round=1, word=7)]   # a round that never ran
    call = sram_call(k, 4, 4, C, [[], [r0]], legs=2, claims=(0, 3), records=([], recs))
    r, _, faults = check_sram(cro, coracle, call)
    assert [f["peer_smid"] for f in faults] == [SILENT] * 3
    assert r["verdict"] == cro.SRAM_ALL and r["leg"][1]["unpublished"] == 1
    assert r["bad_pairs"] == 3 and r["bad_pair"][:3] == [(1, 0xFFFF, 1), (4, 0xFFFF, 1), (0xFFFF, 2, 2)]


def test_pairs_with_an_end_that_failed_locally_are_dropped(cro, coracle):
    k, C = 30, 2
    local = [sram_cta(k, s) for s in range(4)]
    call0 = sram_call(k, 4, 4, C, [], claims=(1, 3))
    fold = local_fold(coracle, call0)
    for c in local:
        c.update(fold_x=fold[0], fold_s=fold[1], fold_w=fold[2])
    local[1]["count"] = [0, 0, 4, 0, 0, 0]                 # SM 1 fails the local leg (an earlier iteration)
    net = net_round(k, [0, 1, 2, 3], C)
    recs = [sram_record(1, smid=0, peer_block=1),          # 0 read 1: 1 failed locally, dropped
            sram_record(3, smid=0, peer_block=1),          # 1 wrote 0: dropped
            sram_record(1, smid=2, peer_block=3)]          # 2 read 3: kept
    call = dict(call0, rounds=[[local], [net]], records=[[sram_record(2, smid=1)], recs])
    r, sms, _ = check_sram(cro, coracle, call)
    assert r["bad_sms"] == 1 and r["bad_sm"][0] == 1 and sms[1]["leg"][0]["mark"] == cro.SRAM_INTERMITTENT
    assert r["bad_pairs"] == 1 and r["bad_pair"][0] == (2, 3, cro.SRAM_DIR_READ)
    assert r["verdict"] == cro.SRAM_SM                     # sm before link


def test_pairs_are_ordered_and_capped(cro, coracle):
    k, C = 40, 8
    smids = list(range(100, 116))
    net = net_round(k, smids, C)
    rng = random.Random(9)
    recs = []
    for _ in range(30):
        b = rng.randrange(16)
        recs.append(sram_record(rng.choice([1, 3]), smid=smids[b], peer_block=rng.randrange(16), word=rng.randrange(64)))
    call = sram_call(k, 16, 16, C, [[], [net]], legs=2, claims=(0, len(recs)), records=([], recs))
    r, _, faults = check_sram(cro, coracle, call)
    pairs = sorted({(f["direction"], f["smid"], f["peer_smid"]) if f["direction"] == 1 else
                    (f["direction"], f["peer_smid"], f["smid"]) for f in faults})
    assert r["bad_pairs"] == len(pairs) >= 9
    assert r["bad_pair"] == [(a, o, d) for d, a, o in pairs[:cro.SRAM_MAX_PAIRS]]


def test_verdict_precedence_all_then_sm_then_link(cro, coracle):
    k, C = 50, 2
    base = sram_call(k, 2, 2, C, [], claims=(0, 1))
    fold = local_fold(coracle, base)
    good = lambda s, **kw: sram_cta(k, s, fold=fold, **kw)
    link = [sram_record(1, smid=0, peer_block=1)]
    reader = {0: dict(count=[0, 1, 0, 0, 0, 0])}
    cases = [
        ([good(0), good(1)], cro.SRAM_LINK),
        ([good(0, last=1, count=[0, 1, 0, 0, 0, 0]), good(1)], cro.SRAM_SM),
        ([good(0, last=1, count=[0, 1, 0, 0, 0, 0]), good(1, count=[0, 0, 0, 0, 0, 1])], cro.SRAM_ALL),
        ([good(0), sram_cta(k, 1, fold=(fold[0] ^ 1, fold[1], fold[2]))], cro.SRAM_SM),        # only the fold
        ([good(0), dict(good(1), stamp=ARMED)], cro.SRAM_ALL),
    ]
    for local, verdict in cases:
        call = dict(base, rounds=[[local], [net_round(k, [0, 1], C, reader)]], records=[[], link])
        r, sms, _ = check_sram(cro, coracle, call)
        assert r["verdict"] == verdict and r["status"] == cro.ERR_CHECKSUM, (local, r["verdict"])
    r, sms, _ = check_sram(cro, coracle, dict(base, rounds=[[cases[0][0]], [net_round(k, [0, 1], C)]], claims=[0, 0]))
    assert r["verdict"] == cro.SRAM_NONE and r["status"] == cro.OK and r["leg"][0]["fold_xor"] == fold[0]


def test_sram_marks_and_the_fold_over_rounds(cro, coracle):
    k = 60
    base = sram_call(k, 3, 2, 2, [], legs=1)
    fold = local_fold(coracle, base)
    r0 = [sram_cta(k, 7, fold=(1, 2, 3)), sram_cta(k, 5, fold=fold, count=[0, 0, 0, 2, 0, 0], last=2), sram_cta(ARMED, 1)]
    r1 = [sram_cta(k, 5, fold=fold), sram_cta(k, 3, fold=(4, 5, 6)), sram_cta(k, 3, fold=fold)]
    r, sms, _ = check_sram(cro, coracle, dict(base, rounds=[[r0, r1], []]))
    L = r["leg"][0]
    assert (L["fold_xor"], L["fold_sum"], L["fold_wsum"]) == (4, 5, 6)   # SM 3's first CTA
    assert [s["leg"][0]["mark"] for s in sms] == [cro.SRAM_INTERMITTENT, cro.SRAM_PERSISTENT, cro.SRAM_INTERMITTENT]
    assert L["fold_mismatches"] == 2 and L["sms_covered"] == 3 and L["complete"] == 1 and L["rounds"] == 2


def test_sram_nsmid_beyond_the_result_fails_with_a_blank_result(cro, coracle):
    k = 70
    call = sram_call(k, 2, 2, 2, [[[sram_cta(k, 0), sram_cta(k, 1, count=[0, 1, 0, 0, 0, 0])]],
                                  [net_round(k, [0, 1], 2, {1: dict(nsmid=300)})]], claims=(0, 1),
                     records=([], [sram_record(1, smid=0, peer_block=1)]))
    r, sms, faults = check_sram(cro, coracle, call)
    assert r["status"] == cro.ERR_UNSUPPORTED and not sms and not faults and r["bad_pairs"] == 0
    assert (r["seed"], r["call"], r["sm_count"], r["legs"], r["bytes_per_sm"]) == (0x1234, k, 2, 3, 8 * 64)


# ---- SRAM: seeded sweep ----------------------------------------------------------------------------------------------
def random_sram_call(rng, coracle):
    cluster = rng.choice([2, 4, 8])
    sm_count = rng.choice([2, 4, 8, 16, 40])
    net_grid = cluster * rng.randint(1, max(1, sm_count // cluster))
    k = rng.randrange(1 << 40)
    call = sram_call(k, sm_count, net_grid, cluster, [[], []], legs=rng.choice([0, 0, 1, 2]),
                     n_words=rng.choice([32, 64, 96]), iterations=rng.choice([1, 2, 3, 64]), seed=rng.randrange(1 << 64))
    fold = local_fold(coracle, call)
    pool = rng.sample(range(256), rng.choice([sm_count, sm_count + 5, max(1, sm_count // 2)]))
    unsupported = rng.random() < 0.03
    n_rounds = [rng.choice([1, 1, 2, 4]) if rng.random() < 0.95 else 0 for _ in range(2)]
    for leg in range(2):
        grid = net_grid if leg else sm_count
        for _ in range(n_rounds[leg]):
            ctas = []
            for j in range(grid):
                bad = rng.random() < 0.1
                count = [rng.randrange(1, 9) if bad and rng.random() < 0.5 else 0 for _ in range(6)]
                ctas.append(sram_cta(
                    k if rng.random() < 0.95 else rng.choice([ARMED, k + 1]), rng.choice(pool), block=j,
                    rank=j % cluster if leg else 0, count=count, last=rng.choice([0, sum(count)]) if bad else 0,
                    fold=fold if leg or rng.random() < 0.9 else tuple(rng.randrange(1 << 64) for _ in range(3)),
                    t0=rng.randrange(1 << 20), t1=rng.randrange(1 << 20), cycles=rng.randrange(1 << 30),
                    nsmid=300 if unsupported and rng.random() < 0.05 else 132))
            call["rounds"][leg].append(ctas)
        c = rng.choice([0, 0, 1, 2, 5, 12]) if rng.random() < 0.97 else rng.choice([4096, 4097, 10 ** 6])
        call["claims"][leg] = c
        for _ in range(min(c, 4096)):
            el = rng.randrange(1, 6) if leg == 0 else rng.choice([1, 3])
            call["records"][leg].append(sram_record(
                el, smid=rng.choice(pool), peer_block=rng.randrange(net_grid + 2), round=rng.randrange(n_rounds[leg] + 1),
                word=rng.randrange(call["n_words"]), iteration=rng.randrange(call["iterations"]),
                expected=rng.randrange(1 << 64), actual=rng.randrange(1 << 64)))
    return call


def test_random_sram_calls_equal_the_restatement(cro, coracle):
    rng = random.Random(20261017)
    seen, capped = set(), 0
    for _ in range(500):
        r, _, _ = check_sram(cro, coracle, random_sram_call(rng, coracle))
        seen.add(r["verdict"] if r["status"] != cro.ERR_UNSUPPORTED else "unsupported")
        capped += r["bad_pairs"] > cro.SRAM_MAX_PAIRS
    assert seen == {cro.SRAM_NONE, cro.SRAM_SM, cro.SRAM_LINK, cro.SRAM_ALL, "unsupported"}, seen
    assert capped > 0


# ---- the C ABI -------------------------------------------------------------------------------------------------------
FIELDS = {
    "cro_sm_cta": ("SmCta", ["stamp", "t0", "t1", "cycles", "mismatches", "fold_mismatches", "fold", "smid", "nsmid"]),
    "cro_sram_cta": ("SramCta", ["stamp", "t0", "t1", "cycles", "count", "last", "fold_x", "fold_s", "fold_w", "smid",
                                 "nsmid", "rank", "block"]),
    "cro_sram_record": ("SramRecord", ["element", "iteration", "smid", "peer_block", "round", "word", "expected", "actual"]),
}


def test_ctypes_layout_of_the_mirrors_matches_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    for k in ("CRO_SM_LEGS_COMPUTE", "CRO_SM_LEGS_PRECISION"):
        src.append('printf("const %s %%d\\n", (int)(%s));' % (k, k))
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
    assert (cro.SM_LEGS_COMPUTE, cro.SM_LEGS_PRECISION) == (got[("const", "CRO_SM_LEGS_COMPUTE")],
                                                              got[("const", "CRO_SM_LEGS_PRECISION")])


def test_sm_legs_hook_refuses_bad_arguments(cro):
    lib, u32, u64 = cro.lib, ctypes.c_uint32, ctypes.c_uint64
    its, rounds, claims = (u32 * 7)(*[1] * 7), (u32 * 7)(), (u64 * 7)()
    ctas, bits = (cro.SmCta * 4)(), (u64 * 16)()
    recs = (cro.PrecisionFault * 4)()
    r, sms, faults = cro.PrecisionResult(), (cro.PrecisionSm * 4)(), (cro.PrecisionFault * 4)()
    ns, n = ctypes.c_int(-1), ctypes.c_int(-1)

    def call(**kw):
        a = dict(probe=cro.SM_LEGS_PRECISION, legs=0, its=its, grid=2, k=0, rounds=rounds, ctas=ctas, bits=bits,
                 claims=claims, recs=recs, out=ctypes.byref(r), sms=sms, sms_cap=4, ns=ctypes.byref(ns), faults=faults,
                 cap=4, n=ctypes.byref(n))
        a.update(kw)
        return lib.cro_selftest_sm_legs_classify(*a.values())
    assert call() == cro.OK and (ns.value, n.value) == (0, 0)
    for kw in (dict(probe=2), dict(probe=-1), dict(legs=0x80), dict(its=None), dict(rounds=None), dict(claims=None),
               dict(grid=0), dict(out=None), dict(ns=None), dict(n=None), dict(sms_cap=-1), dict(cap=-1),
               dict(sms=None), dict(faults=None), dict(its=(u32 * 7)(1, 1, 0, 1, 1, 1, 1))):
        assert call(**kw) == cro.ERR_INVALID_ARG, kw
    assert call(its=(u32 * 7)(1, 1, 0, 1, 1, 1, 1), legs=0x7B) == cro.OK      # leg 2 not run: its count is not read
    rounds[3] = 1
    assert call(ctas=None) == cro.ERR_INVALID_ARG and call(bits=None) == cro.ERR_INVALID_ARG
    claims[0] = 2
    assert call(recs=None) == cro.ERR_INVALID_ARG
    assert call(recs=None, legs=0x7E) == cro.OK                              # leg 0 not run: its claims are not read
    rounds[3], claims[0] = 0, 0
    assert call(ctas=None, bits=None, recs=None, sms=None, sms_cap=0, faults=None, cap=0) == cro.OK


def test_sram_hook_refuses_bad_arguments(cro):
    lib, u32, u64 = cro.lib, ctypes.c_uint32, ctypes.c_uint64
    rounds, claims = (u32 * 2)(), (u64 * 2)()
    ctas, recs = (cro.SramCta * 8)(), (cro.SramRecord * 4)()
    r, sms, faults = cro.SramResult(), (cro.SramSm * 4)(), (cro.SramFault * 4)()
    ns, n = ctypes.c_int(-1), ctypes.c_int(-1)

    def call(**kw):
        a = dict(legs=0, its=2, n_words=32, seed=1, cluster=2, sm_count=4, net_grid=4, k=0, rounds=rounds, ctas=ctas,
                 claims=claims, recs=recs, out=ctypes.byref(r), sms=sms, sms_cap=4, ns=ctypes.byref(ns), faults=faults,
                 cap=4, n=ctypes.byref(n))
        a.update(kw)
        return lib.cro_selftest_sram_classify(*a.values())
    assert call() == cro.OK
    for kw in (dict(legs=4), dict(its=0), dict(its=cro.SRAM_MAX_ITERATIONS + 1), dict(cluster=3), dict(cluster=16),
               dict(sm_count=0), dict(net_grid=0), dict(net_grid=6, cluster=4), dict(rounds=None), dict(claims=None),
               dict(out=None), dict(ns=None), dict(n=None), dict(sms_cap=-1), dict(cap=-1), dict(sms=None),
               dict(faults=None)):
        assert call(**kw) == cro.ERR_INVALID_ARG, kw
    assert call(legs=1, net_grid=0) == cro.OK                # no network leg: its grid is not read
    rounds[1] = 1
    assert call(ctas=None) == cro.ERR_INVALID_ARG and call(ctas=None, legs=1) == cro.OK
    claims[0] = 1
    assert call(recs=None) == cro.ERR_INVALID_ARG and call(recs=None, legs=2) == cro.OK
