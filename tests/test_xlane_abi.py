"""The cross-lane probe without a GPU: the ctypes mirrors against the header as gcc lays it out, cro_xlane_expected and
the injection predictions against oracle/xlane.py, the classification and the emitter against the restatement, the
helper's argv and frame through a stand-in, and the kernels as ptxas and cuobjdump built them (each instantiation
issues its own leg's cross-lane forms and no other leg's; no global atomics, calls, local memory or spills)."""
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
U = "GPU-5ca90000-0000-0000-0000-000000000004"

FIELDS = {
    "cro_xlane_opts": ("XlaneOpts", ["iterations", "legs", "max_rounds", "deadline_ms", "test_inject_leg", "test_inject_sm",
                                     "test_inject_warp", "test_inject_lane", "test_inject_op", "test_inject_iteration",
                                     "test_inject_mask"]),
    "cro_xlane_result": ("XlaneResult", ["status", "verdict", "seed", "call", "sm_count", "nsmid", "cuda_error", "legs",
                                         "iterations", "rounds", "sms_covered", "complete", "ctas", "unpublished",
                                         "threads_unpublished", "failed_sms", "bad_sms", "failed_legs", "bad_sm", "recorded",
                                         "sms_listed", "reserved", "mismatches", "ops_checked", "fold_mismatches", "leg_ns",
                                         "fold", "expect", "ns", "timer_ns", "wall_ns", "helper_ns"]),
    "cro_xlane_sm": ("XlaneSm", ["smid", "mark", "failed_legs", "ctas", "mismatches", "fold_mismatches", "ns", "cycles"]),
    "cro_xlane_fault": ("XlaneFault", ["leg", "op", "iteration", "smid", "warp", "lane", "peer", "reserved", "expected", "actual"]),
    "cro_xlane_thread": ("XlaneThread", ["stamp", "count", "last", "fold_x", "fold_s", "fold_w"]),
    "cro_xlane_cta": ("XlaneCta", ["stamp", "t0", "t1", "cycles", "smid", "nsmid", "block", "reserved"]),
}
CONSTANTS = ["CRO_XLANE_LEG_SHFL", "CRO_XLANE_LEG_VOTE", "CRO_XLANE_LEG_MATCH", "CRO_XLANE_LEG_REDUX", "CRO_XLANE_LEG_ATOMS",
             "CRO_XLANE_LEGS", "CRO_XLANE_ALL_LEGS", "CRO_XLANE_THREADS", "CRO_XLANE_WARPS", "CRO_XLANE_THREAD_RECORDS",
             "CRO_XLANE_RECORDS", "CRO_XLANE_MAX_SMS", "CRO_XLANE_MAX_ITERATIONS", "CRO_XLANE_MAX_ROUNDS", "CRO_XLANE_SHFL_OPS",
             "CRO_XLANE_VOTE_OPS", "CRO_XLANE_MATCH_OPS", "CRO_XLANE_REDUX_OPS", "CRO_XLANE_ATOMS_OPS", "CRO_XLANE_MAX_OPS",
             "CRO_XLANE_NONE", "CRO_XLANE_SM", "CRO_XLANE_ALL", "CRO_XLANE_PERSISTENT", "CRO_XLANE_INTERMITTENT"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
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
    assert cro.XLANE_OPS == [got[("const", "CRO_XLANE_%s_OPS" % n)] for n in ("SHFL", "VOTE", "MATCH", "REDUX", "ATOMS")]


# ---- the answers against oracle/xlane.py ----------------------------------------------------------------------------
SEEDS = [0, 1, 0x1234_5678_9ABC_DEF0, (1 << 64) - 1, 0xD1B54A32D192ED03, 1 << 54, 0x8000_0000_0000_0001, 0x0F0F_F0F0_3C3C_C3C3]


@pytest.mark.parametrize("seed", SEEDS)
def test_expected_equals_the_restatement(cro, seed):
    import xlane
    it = seed % 5
    for leg in range(cro.XLANE_LEGS):
        for w in range(cro.XLANE_WARPS):
            assert cro.xlane_expected(leg, seed, it, w) == xlane.expected(leg, seed, it, w), (leg, w)


def test_expected_covers_the_edges_it_claims(cro):
    import xlane
    e = [cro.xlane_expected(xlane.SHFL, 99, 0, 3)[op * 32:(op + 1) * 32] for op in range(xlane.OPS[xlane.SHFL])]
    # up at width 32 by 1: lane 0 keeps its own value with the predicate clear; every other lane reads lane - 1
    assert e[32][0] >> 32 == 0 and all(e[32][l] >> 32 == 1 for l in range(1, 32))
    assert e[32][0] & xlane.U32 == xlane.shfl_operand(xlane.iteration_seed(99, 0), 32, 3, 0)
    v = cro.xlane_expected(xlane.VOTE, 99, 0, 3)
    assert v[0] == 0 and v[4 * 32] == xlane.U32 and v[(2 + 7) * 4 * 32] == 1 << 7 and v[(34 + 7) * 4 * 32] == xlane.U32 ^ (1 << 7)
    m = cro.xlane_expected(xlane.MATCH, 99, 0, 3)
    assert m[0] == xlane.U32 and m[32] == (1 << 33) - 1 and m[3 * 4 * 32 + 5] == 1 << 5
    r = cro.xlane_expected(xlane.REDUX, 99, 0, 3)
    assert r[(0 * 32 + 4) * 9 * 32 + 2 * 32] == 0 and r[(1 * 32 + 4) * 9 * 32 + 3 * 32] == xlane.U32
    assert r[(2 * 32 + 4) * 9 * 32 + 4 * 32] == 0x80000000 and r[(3 * 32 + 4) * 9 * 32 + 5 * 32] == 0x7FFFFFFF


def test_the_closed_form_folds_the_last_iteration(cro):
    import xlane
    seed = 0x1234_5678_9ABC_DEF0
    r, _, _ = cro.selftest_xlane_classify(cro.XLANE_ALL_LEGS, 3, seed, 1, 0, [])
    for leg in range(cro.XLANE_LEGS):
        assert tuple(r.expect[leg]) == xlane.fold(leg, seed, 3), leg


# ---- what an injection does -----------------------------------------------------------------------------------------
# Ops whose result the injected operand changes wherever the lane sits: shuffles (where some lane reads the injected
# one), ballots and the all-clear / all-set vote rows, matches over one class, sums and xors, and the shared atomics
# whose final word or presence slots follow every operand.
GRID = [(0, op) for op in (0, 5, 31, 32, 40, 80, 88, 89, 100, 145, 146, 160, 176)] + \
       [(1, op) for op in (0, 1, 3, 4, 6, 7, 8, 264, 280, 380)] + \
       [(2, op) for op in (0, 1, 2, 3)] + \
       [(3, op) for op in (0, 1, 8, 9, 17, 130 * 9, 130 * 9 + 1, 130 * 9 + 8, 143 * 9 + 8)] + \
       [(4, op) for op in (0, 1, 2, 3, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57,
                           58, 59)]


@pytest.mark.parametrize("leg,op", GRID)
def test_injection_predictions_are_exact_and_nonempty(cro, leg, op):
    """Every prediction is nonempty, names the lanes the ISA says, and its raw bits are the restated op on the changed
    operand (for SHFL: exactly the lanes whose source is the injected lane, each naming it as peer)."""
    import xlane
    rng = random.Random(leg * 1000 + op)
    seed = rng.randrange(1 << 64)
    for w, l in ((0, 0), (7, 31), (3, 17)):
        mask = (1 << 40) | 1 if leg in (2,) else 1 if leg == 1 else 1 << rng.randrange(32) if leg != 4 else 1 << 3
        if leg == 4 and xlane.KINDS[op // 4] in xlane.WIDE:
            mask = 1 << 35
        p = xlane.injected(leg, seed, 2, op, w, l, mask)
        read = leg != xlane.SHFL or any(xlane.shfl_source(op, x)[0] == l for x in range(32))
        assert bool(p) == read, (leg, op, w, l)
        clean = {k: e for k, (e, _a, _p) in p.items()}
        for (pw, pl), (e, a, peer) in p.items():
            assert e != a
            if leg == xlane.SHFL:
                assert pw == w and peer == l and a == e ^ (mask & xlane.U32)
            else:
                assert peer == xlane.NO_PEER
            if leg != xlane.ATOMS:
                assert e == cro.xlane_expected(leg, seed, 2, pw)[op * 32 + pl] == clean[(pw, pl)]
        if leg == xlane.SHFL:
            assert sorted(pl for _w, pl in p) == sorted(x for x in range(32) if xlane.shfl_source(op, x)[0] == l)
        if leg == xlane.REDUX and op % 9 in (0, 1, 8):
            assert len(p) == 32                                     # a sum or xor fails on every lane of the warp
        if leg == xlane.ATOMS and xlane.KINDS[op // 4].startswith("exch"):
            assert list(p) == [(w, l)]                              # only the injected thread's value goes missing


# ---- the classification against oracle/xlane.py --------------------------------------------------------------------
def as_dict(x):
    return {k: getattr(x, k) for k, _ in x._fields_}


def make_call(cro, rng, case):
    import xlane
    legs = rng.choice([0x1F, 1, 0x14, 0x3]) if case != "overflow" else 0x1F
    sm_count, iterations, call = rng.choice([(3, 1, 0), (2, 4, 3), (1, 2, 9)]) if case != "overflow" else (3, 1, 0)
    seed = rng.randrange(1 << 64)
    expect = {leg: xlane.fold(leg, seed, iterations) for leg in range(5) if legs >> leg & 1}
    n_rounds = rng.choice([1, 2])
    smids = rng.sample(range(sm_count + 4), sm_count)
    rounds = {}
    for leg in expect:
        rounds[leg] = []
        for _ in range(n_rounds):
            ctas, thr, recs = [], [], []
            for j in range(sm_count):
                c = cro.XlaneCta()
                c.stamp, c.t0, c.t1, c.cycles = call, 1000 + j, 2000 + rng.randrange(99), rng.randrange(1 << 30)
                c.smid, c.nsmid, c.block = smids[j] if rng.random() < 0.9 else rng.choice(smids), 140, j
                ctas.append(c)
                for q in range(256):
                    t = cro.XlaneThread()
                    t.stamp = call
                    if q == 0:
                        t.fold_x, t.fold_s, t.fold_w = expect[leg]
                    thr.append(t)
                    for _k in range(4):
                        f = cro.XlaneFault()
                        f.leg, f.op, f.iteration, f.smid = leg, rng.randrange(xlane.OPS[leg]), rng.randrange(iterations), c.smid
                        f.warp, f.lane, f.peer = q >> 5, q & 31, rng.randrange(1 << 32)
                        f.expected, f.actual = rng.randrange(1 << 64), rng.randrange(1 << 64)
                        recs.append(f)
            rounds[leg].append((ctas, thr, recs))
    flat = [rnd for leg in sorted(rounds) for rnd in rounds[leg]]
    if case in ("one", "every", "overflow"):
        for ctas, thr, _ in (flat if case != "one" else [rng.choice(flat)]):
            for j in (range(sm_count) if case != "one" else [rng.randrange(sm_count)]):
                for q in (range(256) if case != "one" else [rng.randrange(256)]):
                    t = thr[j * 256 + q]
                    t.count = rng.randrange(1, 7) if case != "overflow" else 40
                    t.last = rng.choice([0, t.count])
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
    return dict(legs=legs, seed=seed, call=call, iterations=iterations, sm_count=sm_count, rounds=rounds, expect=expect)


@pytest.mark.parametrize("case", ["clean", "one", "every", "fold", "silent", "overflow", "nsmid"])
def test_classification_equals_the_restatement(cro, case):
    import xlane
    rng = random.Random(sum(map(ord, case)))
    for _ in range(3):
        c = make_call(cro, rng, case)
        legs_in_order = [c["rounds"][leg] for leg in sorted(c["rounds"])]
        r, sms, faults = cro.selftest_xlane_classify(c["legs"], c["iterations"], c["seed"], c["sm_count"], c["call"],
                                                     legs_in_order, cap=cro.XLANE_RECORDS + 8)
        want, wsms, wrecs = xlane.classify(
            dict(c, rounds={leg: [([as_dict(x) for x in a], [as_dict(x) for x in b], [as_dict(x) for x in d])
                                  for a, b, d in rr] for leg, rr in c["rounds"].items()}), c["expect"])
        assert r.status == want["status"], case
        if case == "nsmid":
            assert r.status == cro.ERR_UNSUPPORTED and not sms and not faults
            continue
        for k in ("verdict", "seed", "call", "sm_count", "legs", "nsmid", "iterations", "rounds", "sms_covered", "complete", "ctas",
                  "unpublished", "threads_unpublished", "failed_sms", "bad_sms", "failed_legs", "timer_ns"):
            assert getattr(r, k) == want[k], (case, k, getattr(r, k), want[k])
        assert list(r.bad_sm[:min(r.bad_sms, 16)]) == want["bad_sm"]
        assert list(r.mismatches) == want["mismatches"] and list(r.ops_checked) == want["ops_checked"]
        assert list(r.fold_mismatches) == want["fold_mismatches"]
        assert [tuple(f) for f in r.fold] == [tuple(f) for f in want["fold"]]
        assert [{k: (list(v) if k == "mismatches" else v) for k, v in as_dict(s).items()} for s in sms] == wsms
        assert len(sms) == r.sms_listed
        assert [as_dict(f) for f in faults] == wrecs and r.recorded == len(wrecs)
        if case == "every":
            assert r.verdict == cro.XLANE_ALL
        if case == "silent":
            assert r.verdict == cro.XLANE_ALL and r.unpublished + r.threads_unpublished == 1
        if case == "overflow":
            assert r.recorded == cro.XLANE_RECORDS and sum(r.mismatches) > cro.XLANE_RECORDS


def test_null_arguments_are_refused(cro):
    r, sms, faults = cro.XlaneResult(), (cro.XlaneSm * 4)(), (cro.XlaneFault * 4)()
    ks, k = ctypes.c_int(), ctypes.c_int()
    out = (ctypes.c_uint64 * (cro.XLANE_MAX_OPS * 32))()
    assert cro.lib.cro_emit_xlane_annotations_json(None, None, 0, None) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_xlane(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_xlane_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                        ctypes.byref(k)) == cro.ERR_INVALID_ARG
    for leg, w, o in ((5, 0, out), (-1, 0, out), (0, 8, out), (0, -1, out), (0, 0, None)):
        assert cro.lib.cro_xlane_expected(leg, 0, 0, w, o) == cro.ERR_INVALID_ARG
    for legs, it, n in ((0, 1, 1), (0x20, 1, 1), (1, 0, 1), (1, cro.XLANE_MAX_ITERATIONS + 1, 1), (1, 1, 0)):
        assert cro.lib.cro_selftest_xlane_classify(legs, it, 0, n, 0, 0, None, None, None, ctypes.byref(r), sms, 4,
                                                   ctypes.byref(ks), faults, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the emitter against oracle/xlane.py ----------------------------------------------------------------------------
def crafted(cro):
    rng = random.Random(20261017)
    for _ in range(400):
        r = cro.XlaneResult()
        r.status = rng.choice([0, -6, -6, -4, -1, -10])
        r.verdict = rng.choice([0, 1, 2, 3])
        r.cuda_error = rng.choice([0, 214, 700])
        r.sm_count, r.sms_covered = 132, rng.choice([132, 131, 0])
        r.bad_sms = rng.choice([0, 1, 5, 16, 17, 132])
        for i in range(16):
            r.bad_sm[i] = rng.randrange(256)
        r.failed_legs = rng.randrange(32)
        r.iterations = rng.choice([1, 3, 4096])
        yield r


def test_emitter_equals_the_restatement(cro):
    import xlane
    for r in crafted(cro):
        d = {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sms_covered": r.sms_covered,
             "sm_count": r.sm_count, "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm[:min(r.bad_sms, 16)]),
             "failed_legs": r.failed_legs, "iterations": r.iterations}
        assert cro.emit_xlane_annotations_json(r).encode() == xlane.annotations_json(d), d


def test_emitter_spells_the_keys(cro):
    r = cro.XlaneResult()
    r.status, r.verdict, r.sm_count, r.sms_covered, r.bad_sms, r.failed_legs, r.iterations = -6, 1, 132, 132, 2, 0x12, 3
    r.bad_sm[0], r.bad_sm[1] = 7, 40
    assert json.loads(cro.emit_xlane_annotations_json(r)) == {
        "cohdi.io/probe-xlane-verdict": "sm", "cohdi.io/probe-xlane-sms": "132/132", "cohdi.io/probe-xlane-bad-sms": "7,40",
        "cohdi.io/probe-xlane-legs": "vote,atoms", "cohdi.io/probe-xlane-iterations": "3"}


# ---- the helper wire and the helper through a stand-in --------------------------------------------------------------
def test_wire_table_covers_the_options_and_round_trips(tmp_path):
    spec = importlib.util.spec_from_file_location("helper_wire_program", os.path.join(HERE, "test_helper_wire.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    body = ('    { const size_t at[] = {offsetof(cro_xlane_opts, deadline_ms)}, size[] = {sizeof(int32_t)}; '
            'check("xlane", &cro_wire_xlane, sizeof(cro_xlane_opts), at, size, 1); }')
    src = tmp_path / "wire.c"
    src.write_text(mod.PROGRAM.replace("@BODY@", body))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    assert "argc xlane-raw 15" in out.stdout


def test_cli_takes_exactly_its_argument_count():
    run = lambda k: subprocess.run([CLI, "xlane-raw", U] + ["0"] * (k - 3), capture_output=True, timeout=60).returncode
    assert run(14) == 64 and run(16) == 64
    assert run(15) != 64


def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


HELPER = """
import os, struct, sys
assert sys.argv[1] == "xlane-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 15, sys.argv
open(%(log)r, "a").write(" ".join(sys.argv[1:]) + "\\n")
seed_base, iters, legs, rounds, leg, sm, warp, lane, op, iteration, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(560)
struct.pack_into("<iIQQII", r, 0, -6, 1, 1234, 0, 132, 132)
struct.pack_into("<iIII", r, 32, 0, legs or 31, iters, 5)
struct.pack_into("<IIIIIIII", r, 48, 132, 1, 660, 0, 0, 1, 1, 1 << leg)
struct.pack_into("<H", r, 80, sm)
struct.pack_into("<QI", r, 112, n, %(listed)d)
struct.pack_into("<Q", r, 128 + 8 * leg, n)
sms = bytearray(256 * 80)
struct.pack_into("<IIII", sms, 0, 3, 0, 0, 5)
struct.pack_into("<IIII", sms, 80, sm, 1, 1 << leg, 5)
faults = b"".join(struct.pack("<8IQQ", leg, op, iteration, sm, warp, lane + j, lane, 0, 5, 5 ^ mask) for j in range(n))
sys.stdout.buffer.write(bytes(r) + bytes(sms) + faults + b"%(extra)s")
sys.exit(1)
"""


def helper(tmp_path, listed=2, extra=""):
    log = str(tmp_path / "argv.log")
    return fake_helper(tmp_path, HELPER % {"log": log, "listed": listed, "extra": extra}), log


def test_helper_argv_frame_and_fresh_seed_bases(cro, tmp_path, monkeypatch):
    path, log = helper(tmp_path)
    monkeypatch.setenv("CRO_HELPER_PATH", path)
    r, sms, faults = cro.probe_xlane_uuid(None, U, iterations=3, legs=0x9, inject=(3, 9, 2, 17, 100, 2, 1 << 40))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.XLANE_SM and r.seed == 1234 and r.failed_legs == 1 << 3
    assert list(r.bad_sm[:r.bad_sms]) == [9] and r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2
    assert [s.smid for s in sms] == [3, 9] and sms[1].mark == cro.XLANE_PERSISTENT
    assert [(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, f.peer, f.expected, f.actual) for f in faults] == \
        [(3, 100, 2, 9, 2, 17 + j, 17, 5, 5 ^ (1 << 40)) for j in range(3)]
    r, sms, faults = cro.probe_xlane_uuid(None, U, cap=2)
    assert len(faults) == 2 and r.recorded == 2
    a, b = (ln.split() for ln in open(log).read().split("\n")[:2])
    assert a[0] == "xlane-raw" and a[1] == U and a[3:] == ["3", "9", "0", "3", "9", "2", "17", "100", "2", str(1 << 40), "256"]
    assert b[3:] == ["0"] * 10 + ["2"]
    assert a[2] != b[2] and int(a[2]) & 0xFF == 0 and int(b[2]) & 0xFF == 0, (a[2], b[2])


def test_malformed_helper_frames_are_errors(cro, tmp_path, monkeypatch):
    for listed, extra in ((2, "x"), (cro.XLANE_MAX_SMS + 1, "")):
        path, _ = helper(tmp_path, listed, extra)
        monkeypatch.setenv("CRO_HELPER_PATH", path)
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_xlane_uuid(None, U)
        assert e.value.code == cro.ERR_EXEC and "cross-lane helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.stdout.buffer.write(b'short')\nsys.exit(1)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_xlane_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_xlane_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_xlane_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "cross-lane helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


def test_bad_options_are_refused_before_any_spawn(cro, tmp_path, monkeypatch):
    marker = tmp_path / "spawned"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('1')\n" % str(marker)))
    calls = [dict(iterations=cro.XLANE_MAX_ITERATIONS + 1), dict(max_rounds=cro.XLANE_MAX_ROUNDS + 1), dict(legs=0x20),
             dict(deadline_ms=-1), dict(inject=(5, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 0, 1)),
             dict(inject=(0, 0, 8, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 32, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 177, 0, 1)),
             dict(inject=(4, 0, 0, 0, 5, 0, 1)), dict(inject=(0, 0, 0, 0, 0, 3, 1), iterations=3),
             dict(inject=(2, 0, 0, 0, 0, 0, 1), legs=1)]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_xlane_uuid(None, U, **kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert not marker.exists()


# ---- the kernels as the compiler built them -------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]
INSN = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")
CLASSES = {0: "SHFL", 1: "VOTE", 2: "MATCH", 3: "REDUX", 4: "ATOMS"}
FORMS = {0: {"SHFL.IDX", "SHFL.UP", "SHFL.DOWN", "SHFL.BFLY"},
         1: {"VOTE.ANY", "VOTE.ALL", "VOTE.EQ"},
         2: {"MATCH.ANY", "MATCH.ALL", "MATCH.ANY.U64", "MATCH.ALL.U64"},
         3: {"REDUX.SUM", "REDUX.SUM.S32", "REDUX.MIN", "REDUX.MAX", "REDUX.MIN.S32", "REDUX.MAX.S32", "REDUX", "REDUX.OR",
             "REDUX.XOR"},
         4: {"ATOMS.ADD", "ATOMS.INC", "ATOMS.DEC", "ATOMS.MIN", "ATOMS.MAX", "ATOMS.MIN.S32", "ATOMS.MAX.S32", "ATOMS.AND",
             "ATOMS.OR", "ATOMS.XOR", "ATOMS.EXCH", "ATOMS.EXCH.64", "ATOMS.CAS", "ATOMS.CAS.64", "ATOMS.CAST.SPIN.64"}}


def class_of(op):
    head = op.split(".")[0]
    return {"VOTEU": "VOTE"}.get(head, head)


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_each_leg_issues_its_forms_and_no_other_legs():
    kernels, cur = {}, None
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", LIB], text=True).splitlines():
        if "Function : " in ln:
            m = re.search(r"xlane_kernelILj(\d)E", ln)
            cur = int(m.group(1)) if m else None
            if cur is not None:
                kernels[cur] = Counter()
            continue
        m = INSN.search(ln)
        if cur is not None and m:
            kernels[cur][m.group(1)] += 1
    assert sorted(kernels) == [0, 1, 2, 3, 4]
    for leg, ops in kernels.items():
        assert FORMS[leg] <= set(ops), (leg, FORMS[leg] - set(ops))
        assert ops["VOTE.ANY"] >= 2 if leg == 1 else True           # ballot (VOTE.ANY R) and any (VOTE.ANY P)
        others = {op for op in ops if class_of(op) in {"SHFL", "VOTE", "MATCH", "REDUX", "ELECT", "ATOMS"}
                  and class_of(op) != CLASSES[leg]}
        assert not others, (leg, others)
        assert not [op for op in ops if class_of(op) in ("ATOMG", "RED", "CALL", "LDL", "STL")], (leg, ops)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_the_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "xlane_kernels.cu"), "-o",
                                             os.path.join(d, "x.o")], capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    assert len(re.findall(r"Compiling entry function '\S*xlane_kernel", text)) == 5, text
    assert text.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == 5, text
