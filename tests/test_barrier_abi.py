"""The barrier probe without a GPU: the ctypes mirrors against the header as gcc lays it out, cro_barrier_expected
against oracle/barrier.py, the injection predictions, the classification (timeouts and LINK pairs included) and the
emitter against the restatement, the helper's argv and frame through a stand-in, and the kernels as ptxas and
cuobjdump built them (every form in its leg's loop; no call, local memory or spill)."""
import ctypes
import importlib.util
import json
import os
import random
import re
import shutil
import stat
import subprocess
import sys
import tempfile
import time
from collections import Counter

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
LIB = os.path.join(ROOT, "composable-resource-operator_b200", "libcroprobe.so")
CLI = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
U = "GPU-5ca90000-0000-0000-0000-000000000006"

FIELDS = {
    "cro_barrier_opts": ("BarrierOpts", ["iterations", "legs", "max_rounds", "deadline_ms", "cluster", "test_inject_leg",
                                         "test_inject_sm", "test_inject_warp", "test_inject_lane", "test_inject_op",
                                         "test_inject_iteration", "reserved", "test_inject_mask"]),
    "cro_barrier_result": ("BarrierResult", ["status", "verdict", "seed", "call", "sm_count", "nsmid", "cuda_error", "legs",
                                             "iterations", "rounds", "sms_covered", "complete", "ctas", "unpublished",
                                             "threads_unpublished", "failed_sms", "bad_sms", "failed_legs", "bad_sm", "recorded",
                                             "sms_listed", "cluster", "mismatches", "ops_checked", "fold_mismatches", "leg_ns",
                                             "fold", "expect", "timeouts", "cluster_sms", "bad_pairs", "bad_pair", "ns", "timer_ns",
                                             "wall_ns", "helper_ns", "table_ns"]),
    "cro_barrier_sm": ("BarrierSm", ["smid", "mark", "failed_legs", "ctas", "mismatches", "fold_mismatches", "ns", "cycles"]),
    "cro_barrier_row": ("BarrierRow", ["form", "bar", "count", "warps", "producers", "phases", "held", "arriver", "expect", "pred",
                                       "next_rank", "slot_init", "slot_expect"]),
    "cro_barrier_fault": ("BarrierFault", ["leg", "op", "iteration", "smid", "warp", "lane", "kind", "bar", "phase", "slot",
                                           "peer_smid", "reserved", "expected", "actual"]),
    "cro_barrier_thread": ("BarrierThread", ["stamp", "count", "last", "fold_x", "fold_s", "fold_w"]),
    "cro_barrier_cta": ("BarrierCta", ["stamp", "t0", "t1", "cycles", "smid", "nsmid", "block", "reserved"]),
    "cro_barrier_pair": ("BarrierPair", ["smid", "peer_smid"]),
}
CONSTANTS = ["CRO_BARRIER_LEG_BAR", "CRO_BARRIER_LEG_MBAR", "CRO_BARRIER_LEG_CLUSTER", "CRO_BARRIER_LEGS", "CRO_BARRIER_ALL_LEGS",
             "CRO_BARRIER_THREADS", "CRO_BARRIER_WARPS", "CRO_BARRIER_THREAD_RECORDS", "CRO_BARRIER_RECORDS", "CRO_BARRIER_MAX_SMS",
             "CRO_BARRIER_MAX_ITERATIONS", "CRO_BARRIER_MAX_ROUNDS", "CRO_BARRIER_MAX_PAIRS", "CRO_BARRIER_BAR_OPS",
             "CRO_BARRIER_MBAR_OPS", "CRO_BARRIER_CLUSTER_OPS", "CRO_BARRIER_MAX_OPS", "CRO_BARRIER_WAIT_NS",
             "CRO_BARRIER_FORM_POPC", "CRO_BARRIER_FORM_ARRIVE", "CRO_BARRIER_FORM_TICKET", "CRO_BARRIER_FORM_TX",
             "CRO_BARRIER_FORM_CBAR", "CRO_BARRIER_FORM_ST_V4", "CRO_BARRIER_FORM_RED_ADD", "CRO_BARRIER_FORM_RED_DEC",
             "CRO_BARRIER_KIND_VALUE", "CRO_BARRIER_KIND_EARLY", "CRO_BARRIER_KIND_TICKET", "CRO_BARRIER_KIND_TIMEOUT",
             "CRO_BARRIER_NONE", "CRO_BARRIER_SM", "CRO_BARRIER_ALL", "CRO_BARRIER_LINK", "CRO_BARRIER_PERSISTENT",
             "CRO_BARRIER_INTERMITTENT"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    import barrier
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    for k in CONSTANTS:
        src.append('printf("const %s %%lld\\n", (long long)(%s));' % (k, k))
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
        assert [f for f, *_ in cls._fields_] == fields, cname
        for f in fields:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k
    assert cro.BARRIER_OPS == barrier.OPS


# ---- the table against oracle/barrier.py ----------------------------------------------------------------------------
SEEDS = [0, 1, 0x1234_5678_9ABC_DEF0, (1 << 64) - 1, 0xD1B54A32D192ED03, 1 << 52, 0x8000_0000_0000_0001, 0x0F0F_F0F0_3C3C_C3C3]


def as_dict(x):
    d = {}
    for k, _ in x._fields_:
        v = getattr(x, k)
        d[k] = list(v) if hasattr(v, "_length_") else v
    return d


@pytest.mark.parametrize("seed", SEEDS)
def test_table_equals_the_restatement(cro, seed):
    import barrier
    for leg in range(cro.BARRIER_LEGS):
        for cluster in ((2, 4, 8) if leg == cro.BARRIER_LEG_CLUSTER else (2,)):
            rows, words = cro.barrier_expected(leg, seed, cluster)
            for r, (R, w) in enumerate(barrier.table(leg, seed, cluster)):
                assert as_dict(rows[r]) == R, (leg, r)
                assert [[words[(r * 256 + t) * 2], words[(r * 256 + t) * 2 + 1]] for t in range(256)] == w, (leg, r)


def test_table_invariants(cro):
    """Every row keeps its barrier legal: counts are whole warps, the ARRIVE producers and consumers are disjoint, the
    MBAR init counts equal the arrivals a phase makes, the held thread takes part, and the async byte totals are exact."""
    import barrier
    for seed in SEEDS[:4]:
        rows, words = cro.barrier_expected(0, seed)
        assert sorted({r.bar for r in rows}) == list(range(16))
        assert sorted({r.count for r in rows if r.form != barrier.ARRIVE}) == list(range(32, 257, 32))
        for r in rows:
            assert r.count % 32 == 0 and r.count == 32 * bin(r.warps | r.producers).count("1") and not (r.warps & r.producers)
        rows, words = cro.barrier_expected(1, seed)
        for i, r in enumerate(rows):
            part = barrier.members(r.warps)
            mine = [words[(i * 256 + t) * 2] for t in range(256)]
            if r.form == barrier.COUNT:
                assert r.count == sum(mine[t] for t in part) and r.held in part and r.phases >= 2
            if r.form == barrier.DROP:
                assert r.count == len(part) and r.held in part and mine[r.held] == 0
            if r.form == barrier.TX:
                assert r.count == 1 and r.expect == sum(mine[t] for t in part) < (1 << 20) and r.held in part
            if r.form == barrier.TICKET:
                assert r.count == len(part) + 1
        rows, _ = cro.barrier_expected(2, seed)
        assert [r.form for r in rows] == [barrier.CBAR, barrier.CBAR] + list(range(barrier.ST_B32, barrier.RED_DEC + 1))


GRID = [(0, 7, 0, 0, 1), (0, 7, 7, 31, 1 << 40), (0, 48, 3, 5, 1), (0, 16, 0, 0, 2), (1, 0, 0, 0, 1), (1, 2, 7, 31, 1 << 9),
        (1, 6, 4, 4, 3), (2, 0, 0, 0, 1), (2, 5, 7, 31, 1 << 63), (2, 12, 0, 0, 1), (2, 12, 7, 31, 1)]


@pytest.mark.parametrize("leg,op,w,l,mask", GRID)
def test_injection_predictions(cro, leg, op, w, l, mask):
    """An injection makes one record per check of the row the thread makes, each the clean value XOR the mask; a
    thread that checks nothing in the row makes none."""
    import barrier
    seed = random.Random(leg * 100 + op).randrange(1 << 64)
    R, words = barrier.row(leg, seed, op)
    got = barrier.injected(leg, seed, op, w, l, mask)
    t = 32 * w + l
    assert all(a == e ^ mask and a != e for _k, _b, _p, _s, e, a in got)
    if R["form"] in (barrier.POPC, barrier.AND, barrier.OR):
        assert len(got) == (R["warps"] >> w & 1)
    elif R["form"] == barrier.ARRIVE:
        assert len(got) == (len(barrier.members(R["producers"])) if R["warps"] >> w & 1 else 0)
    elif leg == barrier.MBAR:
        assert len(got) == R["phases"] * (5 if R["form"] == barrier.TICKET and R["warps"] >> w & 1 else 3)
    elif R["form"] >= barrier.RED_ADD:
        assert len(got) == 1 + (t < R["arriver"])
    else:
        assert len(got) in (2, 3)


# ---- the classification against the restatement -------------------------------------------------------------------
def make_call(cro, rng, case):
    import barrier
    legs = rng.choice([0x7, 1, 0x4, 0x6]) if case not in ("overflow", "link", "short", "capped") else \
        {"overflow": 0x7, "link": 0x5, "short": 0x5, "capped": 0x6}[case]
    sm_count, iterations, call = rng.choice([(3, 1, 0), (2, 4, 3), (4, 2, 9)]) if case not in ("overflow", "capped") else \
        (3, 1, 0) if case == "overflow" else (4, 1, 0)
    if case == "link":
        sm_count = 4
    cluster = rng.choice([2, 4, 8])
    seed = rng.randrange(1 << 64)
    r0, _, _ = cro.selftest_barrier_classify(legs, iterations, seed, cluster, 1, 0, [])
    expect = {leg: tuple(r0.expect[leg]) for leg in range(3) if legs >> leg & 1}
    n_rounds = rng.choice([1, 2])
    smids = rng.sample(range(sm_count + 4), sm_count)
    rounds = {}
    for leg in expect:
        rounds[leg] = []
        for _ in range(n_rounds):
            ctas, thr, recs = [], [], []
            for j in range(sm_count):
                c = cro.BarrierCta()
                c.stamp, c.t0, c.t1, c.cycles = call, 1000 + j, 2000 + rng.randrange(99), rng.randrange(1 << 30)
                c.smid, c.nsmid, c.block = smids[j] if rng.random() < 0.9 or case == "link" else rng.choice(smids), 140, j
                ctas.append(c)
                for q in range(256):
                    t = cro.BarrierThread()
                    t.stamp = call
                    if q == 0:
                        t.fold_x, t.fold_s, t.fold_w = expect[leg]
                    thr.append(t)
                    for _k in range(4):
                        f = cro.BarrierFault()
                        f.leg, f.op, f.iteration, f.smid = leg, rng.randrange(barrier.OPS[leg]), rng.randrange(iterations), c.smid
                        f.warp, f.lane, f.kind, f.bar = q >> 5, q & 31, rng.randrange(4), rng.randrange(24)
                        f.phase, f.slot = rng.randrange(8), rng.randrange(256)
                        f.peer_smid = rng.choice(smids) if leg == 2 else c.smid
                        f.expected, f.actual = rng.randrange(1 << 64), rng.randrange(1 << 64)
                        recs.append(f)
            rounds[leg].append((ctas, thr, recs))
    flat = [rnd for leg in sorted(rounds) for rnd in rounds[leg]]
    if case in ("one", "every", "overflow", "timeout"):
        for ctas, thr, _ in (flat if case in ("every", "overflow") else [rng.choice(flat)]):
            for j in (range(sm_count) if case in ("every", "overflow") else [rng.randrange(sm_count)]):
                for q in (range(256) if case in ("every", "overflow") else [rng.randrange(256)]):
                    t = thr[j * 256 + q]
                    t.count = rng.randrange(1, 7) if case != "overflow" else 40
                    t.last = rng.choice([0, t.count])
    if case == "link":
        ctas, thr, _ = rounds[2][0]
        for q in (3, 200):
            thr[q].count, thr[q].last = 2, 2
    if case == "short":      # the clusters reach one SM fewer than the CTA-local leg
        for ctas, _, _ in rounds[2]:
            ctas[-1].smid = ctas[0].smid
    if case == "capped":     # MBAR records fill the 4096 cap; the CLUSTER pairs still count
        for ctas, thr, _ in rounds[1]:
            for t in thr:
                t.count, t.last = 4, 4
        ctas, thr, _ = rounds[2][0]
        thr[7].count = thr[7].last = 1
    if case == "fold":
        rng.choice(flat)[1][rng.randrange(sm_count * 256)].fold_w ^= 1
    if case == "silent":
        ctas, thr, _ = rng.choice(flat)
        if rng.random() < 0.5:
            rng.choice(ctas).stamp = (1 << 64) - 1
        else:
            rng.choice(thr).stamp = (1 << 64) - 1
    if case == "nsmid":
        rng.choice(rng.choice(flat)[0]).nsmid = 300
    return dict(legs=legs, seed=seed, call=call, iterations=iterations, cluster=cluster, sm_count=sm_count, rounds=rounds,
                expect=expect)


def test_closed_form_is_the_restatements_fold(cro):
    import barrier
    seed = 0x1234_5678_9ABC_DEF0
    for cluster in (2, 8):
        r, _, _ = cro.selftest_barrier_classify(cro.BARRIER_ALL_LEGS, 3, seed, cluster, 1, 0, [])
        for leg in range(cro.BARRIER_LEGS):
            assert tuple(r.expect[leg]) == barrier.fold(leg, seed, cluster), leg


@pytest.mark.parametrize("case", ["clean", "one", "every", "fold", "silent", "overflow", "nsmid", "timeout", "link", "short", "capped"])
def test_classification_equals_the_restatement(cro, case):
    import barrier
    rng = random.Random(sum(map(ord, case)) + 7)
    for _ in range(2):
        c = make_call(cro, rng, case)
        legs_in_order = [c["rounds"][leg] for leg in sorted(c["rounds"])]
        r, sms, faults = cro.selftest_barrier_classify(c["legs"], c["iterations"], c["seed"], c["cluster"], c["sm_count"], c["call"],
                                                       legs_in_order, cap=cro.BARRIER_RECORDS + 8)
        want, wsms, wrecs = barrier.classify(
            dict(c, rounds={leg: [([as_dict(x) for x in a], [as_dict(x) for x in b], [as_dict(x) for x in d])
                                  for a, b, d in rr] for leg, rr in c["rounds"].items()}), c["expect"])
        assert r.status == want["status"], case
        if case == "nsmid":
            assert r.status == cro.ERR_UNSUPPORTED and not sms and not faults
            continue
        for k in ("verdict", "seed", "call", "sm_count", "legs", "nsmid", "iterations", "rounds", "sms_covered", "complete", "ctas",
                  "unpublished", "threads_unpublished", "failed_sms", "bad_sms", "failed_legs", "timer_ns", "timeouts", "bad_pairs",
                  "cluster_sms"):
            assert getattr(r, k) == want[k], (case, k, getattr(r, k), want[k])
        assert list(r.bad_sm[:min(r.bad_sms, 16)]) == want["bad_sm"]
        assert [(p.smid, p.peer_smid) for p in r.bad_pair[:min(r.bad_pairs, 16)]] == want["bad_pair"]
        assert list(r.mismatches) == want["mismatches"] and list(r.ops_checked) == want["ops_checked"]
        assert list(r.fold_mismatches) == want["fold_mismatches"]
        assert [tuple(f) for f in r.fold] == [tuple(f) for f in want["fold"]]
        assert [as_dict(s) for s in sms] == wsms
        assert [as_dict(f) for f in faults] == wrecs and r.recorded == len(wrecs)
        if case == "every":
            assert r.verdict == cro.BARRIER_ALL
        if case == "silent":
            assert r.verdict == cro.BARRIER_ALL and r.unpublished + r.threads_unpublished == 1
        if case == "overflow":
            assert r.recorded == cro.BARRIER_RECORDS and sum(r.mismatches) > cro.BARRIER_RECORDS
        if case == "link":
            assert r.verdict == cro.BARRIER_LINK and r.bad_pairs >= 1 and r.bad_sms == 1
        if case == "short":
            assert r.sms_covered == c["sm_count"] and r.complete == 1 and r.cluster_sms == c["sm_count"] - 1
        if case == "capped":
            assert r.recorded == cro.BARRIER_RECORDS and all(f.leg == 1 for f in faults) and r.bad_pairs >= 1
        if case == "timeout":
            assert r.timeouts == sum(1 for f in faults if f.kind == cro.BARRIER_KIND_TIMEOUT) or r.recorded == cro.BARRIER_RECORDS


def test_null_arguments_are_refused(cro):
    r, sms, faults = cro.BarrierResult(), (cro.BarrierSm * 4)(), (cro.BarrierFault * 4)()
    ks, k = ctypes.c_int(), ctypes.c_int()
    rows, words = (cro.BarrierRow * 64)(), (ctypes.c_uint64 * (64 * 512))()
    assert cro.lib.cro_emit_barrier_annotations_json(None, None, 0, None) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_barrier(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_barrier_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                          ctypes.byref(k)) == cro.ERR_INVALID_ARG
    for leg, cl, ro, wo in ((3, 2, rows, words), (-1, 2, rows, words), (0, 3, rows, words), (0, 16, rows, words),
                            (0, 2, None, words), (0, 2, rows, None)):
        assert cro.lib.cro_barrier_expected(leg, 0, cl, ro, wo) == cro.ERR_INVALID_ARG
    for legs, it, cl, n in ((0, 1, 2, 1), (0x8, 1, 2, 1), (1, 0, 2, 1), (1, cro.BARRIER_MAX_ITERATIONS + 1, 2, 1), (1, 1, 2, 0),
                            (1, 1, 5, 1)):
        assert cro.lib.cro_selftest_barrier_classify(legs, it, 0, cl, n, 0, 0, None, None, None, ctypes.byref(r), sms, 4,
                                                     ctypes.byref(ks), faults, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the emitter -----------------------------------------------------------------------------------------------------
def test_emitter_equals_the_restatement(cro):
    import barrier
    rng = random.Random(20261019)
    for _ in range(400):
        r = cro.BarrierResult()
        r.status = rng.choice([0, -6, -6, -4, -1, -10])
        r.verdict = rng.choice([0, 1, 2, 3, 3, 4])
        r.cuda_error = rng.choice([0, 214, 700])
        r.sm_count, r.sms_covered = 132, rng.choice([132, 131, 0])
        r.bad_sms = rng.choice([0, 1, 5, 16, 17, 132])
        for i in range(16):
            r.bad_sm[i] = rng.randrange(256)
            r.bad_pair[i].smid, r.bad_pair[i].peer_smid = rng.randrange(256), rng.randrange(256)
        r.bad_pairs = rng.choice([0, 1, 3, 16, 40])
        r.failed_legs = rng.randrange(8)
        r.iterations = rng.choice([1, 3, 4096])
        d = {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sms_covered": r.sms_covered,
             "sm_count": r.sm_count, "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm[:min(r.bad_sms, 16)]),
             "failed_legs": r.failed_legs, "iterations": r.iterations, "bad_pairs": r.bad_pairs,
             "bad_pair": [(p.smid, p.peer_smid) for p in r.bad_pair[:min(r.bad_pairs, 16)]]}
        assert cro.emit_barrier_annotations_json(r).encode() == barrier.annotations_json(d), d


def test_emitter_spells_the_keys(cro):
    r = cro.BarrierResult()
    r.status, r.verdict, r.sm_count, r.sms_covered, r.bad_sms, r.failed_legs, r.iterations = -6, 3, 132, 132, 1, 0x4, 3
    r.bad_sm[0], r.bad_pairs = 7, 1
    r.bad_pair[0].smid, r.bad_pair[0].peer_smid = 7, 40
    assert json.loads(cro.emit_barrier_annotations_json(r)) == {
        "cohdi.io/probe-barrier-verdict": "link", "cohdi.io/probe-barrier-sms": "132/132", "cohdi.io/probe-barrier-bad-sms": "7",
        "cohdi.io/probe-barrier-legs": "cluster", "cohdi.io/probe-barrier-iterations": "3",
        "cohdi.io/probe-barrier-bad-pairs": "7>40"}


# ---- the helper wire and the helper through a stand-in --------------------------------------------------------------
def test_wire_table_covers_the_options_and_round_trips(tmp_path):
    spec = importlib.util.spec_from_file_location("helper_wire_program", os.path.join(HERE, "test_helper_wire.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    body = ('    { const size_t at[] = {offsetof(cro_barrier_opts, deadline_ms), offsetof(cro_barrier_opts, reserved)}, '
            'size[] = {sizeof(int32_t), sizeof(uint32_t)}; check("barrier", &cro_wire_barrier, sizeof(cro_barrier_opts), at, size, 2); }')
    src = tmp_path / "wire.c"
    src.write_text(mod.PROGRAM.replace("@BODY@", body))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    assert "argc barrier-raw 16" in out.stdout


def test_cli_takes_exactly_its_argument_count():
    run = lambda k: subprocess.run([CLI, "barrier-raw", U] + ["0"] * (k - 3), capture_output=True, timeout=60).returncode
    assert run(15) == 64 and run(17) == 64
    assert run(16) != 64


def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


HELPER = """
import os, struct, sys
assert sys.argv[1] == "barrier-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 16, sys.argv
open(%(log)r, "a").write(" ".join(sys.argv[1:]) + "\\n")
seed_base, iters, legs, rounds, cluster, leg, sm, warp, lane, op, iteration, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(488)
struct.pack_into("<iIQQII", r, 0, -6, 1, 1234, 0, 132, 132)
struct.pack_into("<iIII", r, 32, 0, legs or 7, iters, 3)
struct.pack_into("<IIIIIIII", r, 48, 132, 1, 396, 0, 0, 1, 1, 1 << leg)
struct.pack_into("<H", r, 80, sm)
struct.pack_into("<QII", r, 112, n, %(listed)d, cluster or 2)
struct.pack_into("<Q", r, 128 + 8 * leg, n)
sms = bytearray(256 * 64)
struct.pack_into("<IIII", sms, 0, 3, 0, 0, 3)
struct.pack_into("<IIII", sms, 64, sm, 1, 1 << leg, 3)
faults = b"".join(struct.pack("<12I2Q", leg, op, iteration, sm, warp, lane + j, 1, 4, 0, 2, sm, 0, 0, mask) for j in range(n))
sys.stdout.buffer.write(bytes(r) + bytes(sms) + faults + b"%(extra)s")
sys.exit(1)
"""


def helper(tmp_path, listed=2, extra=""):
    log = str(tmp_path / "argv.log")
    return fake_helper(tmp_path, HELPER % {"log": log, "listed": listed, "extra": extra}), log


def test_helper_argv_frame_and_fresh_seed_bases(cro, tmp_path, monkeypatch):
    path, log = helper(tmp_path)
    monkeypatch.setenv("CRO_HELPER_PATH", path)
    r, sms, faults = cro.probe_barrier_uuid(None, U, iterations=3, legs=0x3, cluster=4, inject=(1, 9, 2, 17, 5, 2, 1 << 40))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.BARRIER_SM and r.seed == 1234 and r.failed_legs == 1 << 1
    assert list(r.bad_sm[:r.bad_sms]) == [9] and r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2 and r.cluster == 4
    assert [s.smid for s in sms] == [3, 9] and sms[1].mark == cro.BARRIER_PERSISTENT
    assert [(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, f.kind, f.bar, f.slot, f.actual) for f in faults] == \
        [(1, 5, 2, 9, 2, 17 + j, 1, 4, 2, 1 << 40) for j in range(3)]
    r, sms, faults = cro.probe_barrier_uuid(None, U, cap=2)
    assert len(faults) == 2 and r.recorded == 2
    a, b = (ln.split() for ln in open(log).read().split("\n")[:2])
    assert a[0] == "barrier-raw" and a[1] == U and a[3:] == ["3", "3", "0", "4", "1", "9", "2", "17", "5", "2", str(1 << 40), "256"]
    assert b[3:] == ["0"] * 11 + ["2"]
    assert a[2] != b[2] and int(a[2]) & 0xFF == 0 and int(b[2]) & 0xFF == 0, (a[2], b[2])


def test_malformed_helper_frames_and_exit_3_are_errors(cro, tmp_path, monkeypatch):
    for listed, extra in ((2, "x"), (cro.BARRIER_MAX_SMS + 1, "")):
        path, _ = helper(tmp_path, listed, extra)
        monkeypatch.setenv("CRO_HELPER_PATH", path)
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_barrier_uuid(None, U)
        assert e.value.code == cro.ERR_EXEC and "barrier helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_barrier_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    """The in-process form cannot bound a wedged bar.sync or barrier.cluster.wait; the helper form's deadline can."""
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_barrier_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "barrier helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


BAD_OPTIONS = [dict(iterations=65537), dict(max_rounds=65), dict(legs=0x8), dict(cluster=3), dict(cluster=16),
               dict(inject=(3, 0, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 0, 1)),
               dict(inject=(0, -2, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 8, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 32, 0, 0, 1)),
               dict(inject=(0, 0, 0, 0, 64, 0, 1)), dict(inject=(1, 0, 0, 0, 8, 0, 1)), dict(inject=(2, 0, 0, 0, 17, 0, 1)),
               dict(inject=(0, 0, 0, 0, 0, 3, 1), iterations=3), dict(inject=(2, 0, 0, 0, 0, 0, 1), legs=1)]


def test_bad_options_are_refused_before_any_spawn(cro, tmp_path, monkeypatch):
    marker = tmp_path / "spawned"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('1')\n" % str(marker)))
    for kw in BAD_OPTIONS + [dict(deadline_ms=-1)]:
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_barrier_uuid(None, U, **kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert not marker.exists()


# ---- the kernels as the compiler built them -------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")
# Each leg's native forms as ptxas emits them for this build (PTX form: SASS, DESIGN.md "The barrier probe").
FORMS = {0: {"BAR.RED.POPC.DEFER_BLOCKING", "BAR.RED.AND.DEFER_BLOCKING", "BAR.RED.OR.DEFER_BLOCKING", "BAR.SYNC.DEFER_BLOCKING",
             "BAR.ARV"},
         1: {"SYNCS.EXCH.64", "SYNCS.ARRIVE.TRANS64.A1T0", "SYNCS.ARRIVE.TRANS64.ART0", "SYNCS.ARRIVE.TRANS64.OPTOUT.A1T0",
             "SYNCS.ARRIVE.TRANS64.RED.A0TX", "SYNCS.ARRIVE.TRANS64.TMASK.ART0", "SYNCS.PHASECHK.TRANS64",
             "SYNCS.PHASECHK.TRANS64.TRYWAIT", "SYNCS.ARRIVE.TRANS64"},
         2: {"STAS", "STAS.64", "STAS.128", "REDAS.ADD", "REDAS.ADD.64", "REDAS.MIN", "REDAS.MAX", "REDAS.MIN.S32", "REDAS.MAX.S32",
             "REDAS.AND", "REDAS.OR", "REDAS.XOR", "REDAS.INC", "REDAS.DEC", "UCGABAR_ARV", "UCGABAR_WAIT",
             "SYNCS.PHASECHK.TRANS64.TRYWAIT", "SYNCS.ARRIVE.TRANS64"}}
# The forms only one leg may issue.
OWN = {0: ("BAR.RED", "BAR.ARV"), 1: ("SYNCS.ARRIVE.TRANS64.A1T0", "SYNCS.ARRIVE.TRANS64.OPTOUT", "SYNCS.ARRIVE.TRANS64.RED",
                                      "SYNCS.PHASECHK.TRANS64 ", "SYNCS.ARRIVE.TRANS64.TMASK"),
       2: ("STAS", "REDAS", "UCGABAR")}


def sass():
    kernels, cur = {}, None
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", LIB], text=True).splitlines():
        if "Function : " in ln:
            m = re.search(r"barrier_kernelILj(\d)E", ln)
            cur = int(m.group(1)) if m else None
            if cur is not None:
                kernels[cur] = []
            continue
        m = INSN.search(ln)
        if cur is not None and m:
            kernels[cur].append((int(m.group(1), 16), m.group(2), ln))
    return kernels


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_each_leg_issues_its_forms_inside_the_loop_and_no_other_legs():
    kernels = sass()
    assert sorted(kernels) == [0, 1, 2]
    for leg, ins in kernels.items():
        # the iteration loop: from the first %clock64 read to the second
        clocks = [a for a, op, _ in ins if op.startswith("CS2R")]
        first, last = min(clocks), max(clocks)
        inside = Counter(op for a, op, _ in ins if first <= a <= last)
        assert FORMS[leg] <= set(inside), (leg, FORMS[leg] - set(inside))
        ops = Counter(op for _a, op, _ in ins)
        for other, names in OWN.items():
            if other != leg:
                assert not [op for op in ops if (op + " ").startswith(names)], (leg, other)
        assert not [op for op in ops if op.startswith(("CALL", "LDL", "STL"))], (leg, ops)
        # the report path, after the loop's last %clock64: plain stores and fences only (the CLUSTER leg's exit barrier,
        # a CTA bar.sync and the cluster arrive / wait as ptxas lowers it, comes before it)
        tail = [op for a, op, _ in ins if a > last]
        end = [i for i, op in enumerate(tail) if op.startswith(("UCGABAR_WAIT", "BAR.SYNC"))] if leg == 2 else []
        tail = tail[end[-1] + 1:] if end else tail
        assert not [op for op in tail if op.startswith(("BAR", "VOTE", "ATOM", "RED", "SYNCS", "SHFL", "MATCH"))], (leg, tail)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_the_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c",
                                             os.path.join(CSRC, "barrier_kernels.cu"), "-o", os.path.join(d, "a.o")],
                           capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    assert len(re.findall(r"Compiling entry function '\S*barrier_kernel", text)) == 3, text
    assert text.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == 3, text
