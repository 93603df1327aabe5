"""The ALU probe without a GPU: the ctypes mirrors against the header as gcc lays it out, cro_alu_expected (operands
and exact results) against oracle/alu.py, hand-worked rounding cases, the round-to-nearest rows against numpy, the
injection predictions, the classification and the emitter against the restatement, the helper's argv and frame
through a stand-in, and the kernels as ptxas and cuobjdump built them (every form in its leg's loop; no call, local
memory, spill, MMA or another leg's form)."""
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

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
LIB = os.path.join(ROOT, "composable-resource-operator_b200", "libcroprobe.so")
CLI = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
U = "GPU-5ca90000-0000-0000-0000-000000000005"

FIELDS = {
    "cro_alu_opts": ("AluOpts", ["iterations", "legs", "max_rounds", "deadline_ms", "test_inject_leg", "test_inject_sm",
                                 "test_inject_warp", "test_inject_lane", "test_inject_op", "test_inject_iteration",
                                 "test_inject_operand", "reserved", "test_inject_mask"]),
    "cro_alu_result": ("AluResult", ["status", "verdict", "seed", "call", "sm_count", "nsmid", "cuda_error", "legs", "iterations",
                                     "rounds", "sms_covered", "complete", "ctas", "unpublished", "threads_unpublished",
                                     "failed_sms", "bad_sms", "failed_legs", "bad_sm", "recorded", "sms_listed", "reserved",
                                     "mismatches", "ops_checked", "fold_mismatches", "leg_ns", "fold", "expect", "ns",
                                     "timer_ns", "wall_ns", "helper_ns", "table_ns"]),
    "cro_alu_sm": ("AluSm", ["smid", "mark", "failed_legs", "ctas", "mismatches", "fold_mismatches", "ns", "cycles"]),
    "cro_alu_record": ("AluRecord", [("in_", "in"), "out", "reserved"]),
    "cro_alu_fault": ("AluFault", ["leg", "op", "iteration", "smid", "warp", "lane", "reserved", ("in_", "in"), "expected",
                                   "actual"]),
    "cro_alu_thread": ("AluThread", ["stamp", "count", "last", "fold_x", "fold_s", "fold_w"]),
    "cro_alu_cta": ("AluCta", ["stamp", "t0", "t1", "cycles", "smid", "nsmid", "block", "reserved"]),
}
CONSTANTS = ["CRO_ALU_LEG_LOGIC", "CRO_ALU_LEG_SHIFT", "CRO_ALU_LEG_IADD", "CRO_ALU_LEG_IMUL", "CRO_ALU_LEG_FLOAT", "CRO_ALU_LEGS",
             "CRO_ALU_ALL_LEGS", "CRO_ALU_THREADS", "CRO_ALU_WARPS", "CRO_ALU_THREAD_RECORDS", "CRO_ALU_RECORDS", "CRO_ALU_MAX_SMS",
             "CRO_ALU_MAX_ITERATIONS", "CRO_ALU_MAX_ROUNDS", "CRO_ALU_LOGIC_OPS", "CRO_ALU_SHIFT_OPS", "CRO_ALU_IADD_OPS",
             "CRO_ALU_IMUL_OPS", "CRO_ALU_FLOAT_OPS", "CRO_ALU_MAX_OPS", "CRO_ALU_NONE", "CRO_ALU_SM", "CRO_ALU_ALL",
             "CRO_ALU_PERSISTENT", "CRO_ALU_INTERMITTENT"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    import alu
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            c = f[1] if isinstance(f, tuple) else f
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, c, cname, c))
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
        names = [f[0] if isinstance(f, tuple) else f for f in fields]
        assert [f for f, *_ in cls._fields_] == names, cname
        for f in fields:
            py_name, c_name = f if isinstance(f, tuple) else (f, f)
            assert getattr(cls, py_name).offset == got[(cname, c_name)], (cname, f)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k
    assert cro.ALU_OPS == alu.OPS == [got[("const", "CRO_ALU_%s_OPS" % n)] for n in ("LOGIC", "SHIFT", "IADD", "IMUL", "FLOAT")]


# ---- the table against oracle/alu.py --------------------------------------------------------------------------------
SEEDS = [0, 1, 0x1234_5678_9ABC_DEF0, (1 << 64) - 1, 0xD1B54A32D192ED03, 1 << 53, 0x8000_0000_0000_0001, 0x0F0F_F0F0_3C3C_C3C3]


@pytest.mark.parametrize("seed", SEEDS)
def test_table_equals_the_restatement(cro, seed):
    """Operands and exact results of every (leg, op, lane) of two warps per seed, all eight warps over the eight."""
    import alu
    for leg in range(cro.ALU_LEGS):
        for w in (SEEDS.index(seed), 7 - SEEDS.index(seed)):
            got = cro.alu_expected(leg, seed, w)
            for i, (x, out) in enumerate(alu.expected(leg, seed, w)):
                r = got[i]
                assert list(r.in_) == x and tuple(r.out) == tuple(out), (leg, w, i // 32, i % 32)


def f32(v):
    return int(np.array(v, dtype=np.float32).view(np.uint32))


def f64(v):
    return int(np.array(v, dtype=np.float64).view(np.uint64))


# (form, a, b, c, expected) of hand-worked f32 cases per mode: ties to even, the overflow boundary, subnormal results
# and the sign of an exact zero.
ONE, HALF_ULP = f32(1.0), f32(2.0 ** -24)
HAND = [
    (0, ONE, HALF_ULP, 0, ONE),                       # 1 + 2^-24: a tie, to even
    (0, f32(1.0 + 2 ** -23), HALF_ULP, 0, f32(1.0 + 2 ** -22)),   # odd, the tie goes up
    (1, f32(1.0 + 2 ** -23), HALF_ULP, 0, f32(1.0 + 2 ** -23)),
    (2, f32(-1.0), f32(-(2.0 ** -30)), 0, f32(-(1.0 + 2 ** -23))),   # rm of a negative inexact sum goes away from 0
    (3, ONE, f32(2.0 ** -30), 0, f32(1.0 + 2 ** -23)),
    (0, 0x7F7FFFFF, f32(2.0 ** 103), 0, 0x7F800000),  # FLT_MAX + half an ulp: rn to infinity
    (1, 0x7F7FFFFF, 0x7F7FFFFF, 0, 0x7F7FFFFF),       # rz never overflows to infinity
    (2, 0x7F7FFFFF, 0x7F7FFFFF, 0, 0x7F7FFFFF),
    (3, 0x7F7FFFFF, 0x7F7FFFFF, 0, 0x7F800000),
    (2, 0xFF7FFFFF, 0xFF7FFFFF, 0, 0xFF800000),
    (3, 0xFF7FFFFF, 0xFF7FFFFF, 0, 0xFF7FFFFF),
    (0, ONE, f32(-1.0), 0, 0),                        # cancellation: +0 but -0 rounding down
    (1, ONE, f32(-1.0), 0, 0),
    (2, ONE, f32(-1.0), 0, 0x80000000),
    (3, ONE, f32(-1.0), 0, 0),
    (0, 0x80000000, 0x80000000, 0, 0x80000000),
    (8, 0x00000001, f32(0.5), 0, 0),                  # min subnormal / 2: a tie to the even 0
    (8, 0x00000003, f32(0.5), 0, 0x00000002),         # 1.5 ulp: up to even
    (9, 0x00000003, f32(0.5), 0, 0x00000001),
    (11, 0x00000001, 0x00000001, 0, 0x00000001),      # rp of a positive underflow: the smallest subnormal
    (10, 0x80000001, 0x00000001, 0, 0x80000001),
    (8, 0x00800000, f32(0.5), 0, 0x00400000),         # min normal / 2: exactly subnormal
    (14, ONE, ONE, f32(-1.0), 0x80000000),            # fma 1 * 1 - 1 rounding down: -0
    (12, f32(1.0 + 2 ** -12), f32(1.0 - 2 ** -12), f32(-1.0), f32(-(2.0 ** -24))),   # fma keeps the low bits
]


@pytest.mark.parametrize("case", HAND)
def test_hand_worked_rounding(case):
    import alu
    f, a, b, c, want = case
    assert alu.result(alu.FLOAT, f, [a, b, c, 0])[0] == want, case


def test_hand_worked_rounding_in_the_table_builder(cro):
    """The library's builder agrees with the hand-worked cases wherever the table holds the same operands, and every
    rounding decision the cases name appears in the FLOAT leg of some seed."""
    import alu
    for f, a, b, c, want in HAND:
        assert alu.result(alu.FLOAT, f, [a, b, c, 0])[0] == want
    seen = Counter()
    for seed in SEEDS[:2]:
        for w in range(cro.ALU_WARPS):
            for i, r in enumerate(cro.alu_expected(alu.FLOAT, seed, w)):
                f = i // 32 // alu.ROWS[alu.FLOAT]
                if f < 16:
                    out = r.out[0]
                    seen["zero"] += out & 0x7FFFFFFF == 0
                    seen["negzero"] += out == 0x80000000
                    seen["sub"] += 0 < out & 0x7FFFFFFF < 0x00800000
                    seen["inf"] += out & 0x7FFFFFFF == 0x7F800000
                    seen["max"] += out & 0x7FFFFFFF == 0x7F7FFFFF
    assert all(seen[k] > 0 for k in ("zero", "negzero", "sub", "inf", "max")), seen


def test_round_to_nearest_rows_match_numpy(cro):
    import alu
    for seed in SEEDS[:3]:
        for w in (0, 5):
            recs = cro.alu_expected(alu.FLOAT, seed, w)
            for i, r in enumerate(recs):
                f = i // 32 // alu.ROWS[alu.FLOAT]
                if f in (0, 4, 8):
                    a, b = np.array([r.in_[0], r.in_[1]], dtype=np.uint32).view(np.float32)
                    with np.errstate(all="ignore"):
                        v = {0: a + b, 4: a - b, 8: a * b}[f]
                    assert f32(v) == r.out[0], (f, hex(r.in_[0]), hex(r.in_[1]))
                elif f == 12:
                    a, b, c = (np.float64(x) for x in np.array(list(r.in_[:3]), dtype=np.uint32).view(np.float32))
                    # a * b is exact in binary64; + c then one rounding to binary32 is double rounding only on ties
                    exact = alu.value(alu.F32, r.in_[0]) * alu.value(alu.F32, r.in_[1]) + alu.value(alu.F32, r.in_[2])
                    if exact == float(a * b + c) and abs(exact) < 3e38:
                        assert f32(np.float32(a * b + c)) == r.out[0] or exact == 0


# ---- what an injection does -----------------------------------------------------------------------------------------
# (leg, form, operand, mask, changes): masks the op ignores predict no record.
GRID = [(0, 0xF0, 1, 1 << 5, False),          # LUT 0xF0 is a: b does not matter
        (0, 0xF0, 0, 1 << 5, True), (0, 0x96, 2, 1 << 31, True), (0, 0x00, 0, 0xFFFF, False), (0, 0xFF, 2, 1, False),
        (0, 258, 0, 1, True), (0, 259, 1, 1, False), (0, 260, 0, 1 << 40, True),
        (1, 12, 0, 1 << 32, False),           # prmt reads a 32-bit a
        (1, 13, 2, 1 << 8, False),            # the mode forms read only c[1:0]
        (1, 4, 0, 1, None), (1, 8, 0, 1 << 63, None), (1, 0, 1, 1 << 3, None),
        (2, 0, 0, 1, True), (2, 1, 3, 1 << 63, True), (2, 48, 2, 1, True), (2, 14, 2, 1, False),
        (3, 0, 2, 1, False), (3, 6, 2, 1, True), (3, 13, 0, 1 << 7, None), (3, 12, 1, 1 << 40, True),
        (4, 0, 2, 1, False), (4, 12, 2, 1 << 31, None), (4, 16, 0, 1, None), (4, 31, 0, 1 << 22, None)]


@pytest.mark.parametrize("leg,form,operand,mask,changes", GRID)
def test_injection_predictions(cro, leg, form, operand, mask, changes):
    """Every prediction names the table's operands and expected result and the restated op on the changed operand;
    where the form ignores the changed bits there is none."""
    import alu
    rng = random.Random(leg * 1000 + form)
    seed = rng.randrange(1 << 64)
    any_record = False
    for row in range(alu.ROWS[leg]):
        op = form * alu.ROWS[leg] + row
        for w, l in ((0, 0), (7, 31), (3, 17)):
            p = alu.injected(leg, seed, op, w, l, operand, mask)
            r = cro.alu_expected(leg, seed, w)[op * 32 + l]
            if p is None:
                continue
            any_record = True
            x, e, a = p
            assert x == list(r.in_) and e == tuple(r.out) and a != e
            y = list(x)
            y[operand] ^= mask
            assert a == alu.result(leg, form, y)
    if changes is not None:
        assert any_record == changes, (leg, form, operand, mask)


# ---- the classification against the restatement -------------------------------------------------------------------
def as_dict(x):
    d = {}
    for k, _ in x._fields_:
        v = getattr(x, k)
        d[k] = list(v) if hasattr(v, "_length_") else v
    return d


def make_call(cro, rng, case):
    import alu
    legs = rng.choice([0x1F, 1, 0x14, 0x3]) if case != "overflow" else 0x1F
    sm_count, iterations, call = rng.choice([(3, 1, 0), (2, 4, 3), (1, 2, 9)]) if case != "overflow" else (3, 1, 0)
    seed = rng.randrange(1 << 64)
    r0, _, _ = cro.selftest_alu_classify(legs, iterations, seed, 1, 0, [])
    expect = {leg: tuple(r0.expect[leg]) for leg in range(5) if legs >> leg & 1}
    n_rounds = rng.choice([1, 2])
    smids = rng.sample(range(sm_count + 4), sm_count)
    rounds = {}
    for leg in expect:
        rounds[leg] = []
        for _ in range(n_rounds):
            ctas, thr, recs = [], [], []
            for j in range(sm_count):
                c = cro.AluCta()
                c.stamp, c.t0, c.t1, c.cycles = call, 1000 + j, 2000 + rng.randrange(99), rng.randrange(1 << 30)
                c.smid, c.nsmid, c.block = smids[j] if rng.random() < 0.9 else rng.choice(smids), 140, j
                ctas.append(c)
                for q in range(256):
                    t = cro.AluThread()
                    t.stamp = call
                    if q == 0:
                        t.fold_x, t.fold_s, t.fold_w = expect[leg]
                    thr.append(t)
                    for _k in range(4):
                        f = cro.AluFault()
                        f.leg, f.op, f.iteration, f.smid = leg, rng.randrange(alu.OPS[leg]), rng.randrange(iterations), c.smid
                        f.warp, f.lane = q >> 5, q & 31
                        for i in range(4):
                            f.in_[i] = rng.randrange(1 << 64)
                        for i in range(3):
                            f.expected[i], f.actual[i] = rng.randrange(1 << 64), rng.randrange(1 << 64)
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


def test_closed_form_is_the_restatements_fold(cro):
    import alu
    seed = 0x1234_5678_9ABC_DEF0
    r, _, _ = cro.selftest_alu_classify(cro.ALU_ALL_LEGS, 3, seed, 1, 0, [])
    for leg in range(cro.ALU_LEGS):
        assert tuple(r.expect[leg]) == alu.fold(leg, seed), leg


@pytest.mark.parametrize("case", ["clean", "one", "every", "fold", "silent", "overflow", "nsmid"])
def test_classification_equals_the_restatement(cro, case):
    import alu
    rng = random.Random(sum(map(ord, case)) + 1)
    for _ in range(2):
        c = make_call(cro, rng, case)
        legs_in_order = [c["rounds"][leg] for leg in sorted(c["rounds"])]
        r, sms, faults = cro.selftest_alu_classify(c["legs"], c["iterations"], c["seed"], c["sm_count"], c["call"], legs_in_order,
                                                   cap=cro.ALU_RECORDS + 8)
        want, wsms, wrecs = alu.classify(
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
        assert [as_dict(s) for s in sms] == wsms
        assert [as_dict(f) for f in faults] == wrecs and r.recorded == len(wrecs)
        if case == "every":
            assert r.verdict == cro.ALU_ALL
        if case == "silent":
            assert r.verdict == cro.ALU_ALL and r.unpublished + r.threads_unpublished == 1
        if case == "overflow":
            assert r.recorded == cro.ALU_RECORDS and sum(r.mismatches) > cro.ALU_RECORDS


def test_null_arguments_are_refused(cro):
    r, sms, faults = cro.AluResult(), (cro.AluSm * 4)(), (cro.AluFault * 4)()
    ks, k = ctypes.c_int(), ctypes.c_int()
    out = (cro.AluRecord * (cro.ALU_MAX_OPS * 32))()
    assert cro.lib.cro_emit_alu_annotations_json(None, None, 0, None) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_alu(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_alu_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    for leg, w, o in ((5, 0, out), (-1, 0, out), (0, 8, out), (0, -1, out), (0, 0, None)):
        assert cro.lib.cro_alu_expected(leg, 0, w, o) == cro.ERR_INVALID_ARG
    for legs, it, n in ((0, 1, 1), (0x20, 1, 1), (1, 0, 1), (1, cro.ALU_MAX_ITERATIONS + 1, 1), (1, 1, 0)):
        assert cro.lib.cro_selftest_alu_classify(legs, it, 0, n, 0, 0, None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks),
                                                 faults, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the emitter -----------------------------------------------------------------------------------------------------
def test_emitter_equals_the_restatement(cro):
    import alu
    rng = random.Random(20261018)
    for _ in range(400):
        r = cro.AluResult()
        r.status = rng.choice([0, -6, -6, -4, -1, -10])
        r.verdict = rng.choice([0, 1, 2, 3])
        r.cuda_error = rng.choice([0, 214, 700])
        r.sm_count, r.sms_covered = 132, rng.choice([132, 131, 0])
        r.bad_sms = rng.choice([0, 1, 5, 16, 17, 132])
        for i in range(16):
            r.bad_sm[i] = rng.randrange(256)
        r.failed_legs = rng.randrange(32)
        r.iterations = rng.choice([1, 3, 4096])
        d = {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sms_covered": r.sms_covered,
             "sm_count": r.sm_count, "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm[:min(r.bad_sms, 16)]),
             "failed_legs": r.failed_legs, "iterations": r.iterations}
        assert cro.emit_alu_annotations_json(r).encode() == alu.annotations_json(d), d


def test_emitter_spells_the_keys(cro):
    r = cro.AluResult()
    r.status, r.verdict, r.sm_count, r.sms_covered, r.bad_sms, r.failed_legs, r.iterations = -6, 1, 132, 132, 2, 0x12, 3
    r.bad_sm[0], r.bad_sm[1] = 7, 40
    assert json.loads(cro.emit_alu_annotations_json(r)) == {
        "cohdi.io/probe-alu-verdict": "sm", "cohdi.io/probe-alu-sms": "132/132", "cohdi.io/probe-alu-bad-sms": "7,40",
        "cohdi.io/probe-alu-legs": "shift,float", "cohdi.io/probe-alu-iterations": "3"}


# ---- the helper wire and the helper through a stand-in --------------------------------------------------------------
def test_wire_table_covers_the_options_and_round_trips(tmp_path):
    spec = importlib.util.spec_from_file_location("helper_wire_program", os.path.join(HERE, "test_helper_wire.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    body = ('    { const size_t at[] = {offsetof(cro_alu_opts, deadline_ms), offsetof(cro_alu_opts, reserved)}, '
            'size[] = {sizeof(int32_t), sizeof(uint32_t)}; check("alu", &cro_wire_alu, sizeof(cro_alu_opts), at, size, 2); }')
    src = tmp_path / "wire.c"
    src.write_text(mod.PROGRAM.replace("@BODY@", body))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    assert "argc alu-raw 16" in out.stdout


def test_cli_takes_exactly_its_argument_count():
    run = lambda k: subprocess.run([CLI, "alu-raw", U] + ["0"] * (k - 3), capture_output=True, timeout=60).returncode
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
assert sys.argv[1] == "alu-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 16, sys.argv
open(%(log)r, "a").write(" ".join(sys.argv[1:]) + "\\n")
seed_base, iters, legs, rounds, leg, sm, warp, lane, op, iteration, operand, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(568)
struct.pack_into("<iIQQII", r, 0, -6, 1, 1234, 0, 132, 132)
struct.pack_into("<iIII", r, 32, 0, legs or 31, iters, 5)
struct.pack_into("<IIIIIIII", r, 48, 132, 1, 660, 0, 0, 1, 1, 1 << leg)
struct.pack_into("<H", r, 80, sm)
struct.pack_into("<QI", r, 112, n, %(listed)d)
struct.pack_into("<Q", r, 128 + 8 * leg, n)
sms = bytearray(256 * 80)
struct.pack_into("<IIII", sms, 0, 3, 0, 0, 5)
struct.pack_into("<IIII", sms, 80, sm, 1, 1 << leg, 5)
faults = b"".join(struct.pack("<8I4Q3Q3Q", leg, op, iteration, sm, warp, lane + j, 0, 0, 1, 2, 3, 4, 5, 0, 0, 5 ^ mask, 0, 0)
                  for j in range(n))
sys.stdout.buffer.write(bytes(r) + bytes(sms) + faults + b"%(extra)s")
sys.exit(1)
"""


def helper(tmp_path, listed=2, extra=""):
    log = str(tmp_path / "argv.log")
    return fake_helper(tmp_path, HELPER % {"log": log, "listed": listed, "extra": extra}), log


def test_helper_argv_frame_and_fresh_seed_bases(cro, tmp_path, monkeypatch):
    path, log = helper(tmp_path)
    monkeypatch.setenv("CRO_HELPER_PATH", path)
    r, sms, faults = cro.probe_alu_uuid(None, U, iterations=3, legs=0x9, inject=(3, 9, 2, 17, 40, 2, 1, 1 << 40))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.ALU_SM and r.seed == 1234 and r.failed_legs == 1 << 3
    assert list(r.bad_sm[:r.bad_sms]) == [9] and r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2
    assert [s.smid for s in sms] == [3, 9] and sms[1].mark == cro.ALU_PERSISTENT
    assert [(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, list(f.in_), f.expected[0], f.actual[0]) for f in faults] == \
        [(3, 40, 2, 9, 2, 17 + j, [1, 2, 3, 4], 5, 5 ^ (1 << 40)) for j in range(3)]
    r, sms, faults = cro.probe_alu_uuid(None, U, cap=2)
    assert len(faults) == 2 and r.recorded == 2
    a, b = (ln.split() for ln in open(log).read().split("\n")[:2])
    assert a[0] == "alu-raw" and a[1] == U and a[3:] == ["3", "9", "0", "3", "9", "2", "17", "40", "2", "1", str(1 << 40), "256"]
    assert b[3:] == ["0"] * 11 + ["2"]
    assert a[2] != b[2] and int(a[2]) & 0xFF == 0 and int(b[2]) & 0xFF == 0, (a[2], b[2])


def test_malformed_helper_frames_and_exit_3_are_errors(cro, tmp_path, monkeypatch):
    for listed, extra in ((2, "x"), (cro.ALU_MAX_SMS + 1, "")):
        path, _ = helper(tmp_path, listed, extra)
        monkeypatch.setenv("CRO_HELPER_PATH", path)
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_alu_uuid(None, U)
        assert e.value.code == cro.ERR_EXEC and "ALU helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_alu_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_alu_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "ALU helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


BAD_OPTIONS = [dict(iterations=65537), dict(max_rounds=65), dict(legs=0x20), dict(inject=(5, 0, 0, 0, 0, 0, 0, 1)),
               dict(inject=(-1, 0, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 0, 0, 1)), dict(inject=(0, -2, 0, 0, 0, 0, 0, 1)),
               dict(inject=(0, 0, 8, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 32, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 538, 0, 0, 1)),
               dict(inject=(1, 0, 0, 0, 76, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 0, 0, 4, 1)),
               dict(inject=(0, 0, 0, 0, 0, 3, 0, 1), iterations=3), dict(inject=(2, 0, 0, 0, 0, 0, 0, 1), legs=1)]


def test_bad_options_are_refused_before_any_spawn(cro, tmp_path, monkeypatch):
    marker = tmp_path / "spawned"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('1')\n" % str(marker)))
    for kw in BAD_OPTIONS + [dict(deadline_ms=-1)]:
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_alu_uuid(None, U, **kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert not marker.exists()


# ---- the kernels as the compiler built them -------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")
# Each leg's native forms as ptxas emits them for this build (setp's lt / le come out as gt / ge with the operands
# swapped; the carry chains as IADD3 with IADD3.X or IMAD.X).
FORMS = {0: {"LOP3.LUT", "BMSK", "BMSK.W", "BREV", "POPC", "FLO.U32", "FLO", "FLO.U32.SH", "FLO.SH", "SGXT", "SGXT.U32",
             "SGXT.W", "SGXT.W.U32"},
         1: {"SHF.L.W.U32.HI", "SHF.R.W.U32", "SHF.R.S64", "SHF.R.U64", "PRMT", "PRMT.F4E", "PRMT.B4E", "PRMT.RC8", "PRMT.ECL",
             "PRMT.ECR", "PRMT.RC16"},
         2: {"ISETP.GE.AND", "SEL", "VIMNMX", "VIMNMX.U32", "VIMNMX.RELU", "VIMNMX.S16", "VIMNMX.U16", "VIMNMX3", "VIMNMX3.U32",
             "VIMNMX3.RELU", "VIMNMX3.S16", "VIMNMX3.U16", "VIADDMNMX", "VIADDMNMX.U32", "VIADDMNMX.RELU", "VIADDMNMX.S16",
             "VIADDMNMX.U16", "VABSDIFF", "VABSDIFF.U32"},
         3: {"IMAD.HI", "IMAD.HI.U32", "IMAD.WIDE", "IMAD.WIDE.U32", "IMAD.X", "IDP.4A.U8.U8", "IDP.4A.U8.S8", "IDP.4A.S8.U8",
             "IDP.4A.S8.S8", "IDP.2A.LO.U16.U8", "IDP.2A.LO.U16.S8", "IDP.2A.LO.S16.U8", "IDP.2A.LO.S16.S8", "IDP.2A.HI.U16.U8",
             "IDP.2A.HI.U16.S8", "IDP.2A.HI.S16.U8", "IDP.2A.HI.S16.S8"},
         4: {"FADD", "FADD.RZ", "FADD.RM", "FADD.RP", "FMUL", "FMUL.RZ", "FMUL.RM", "FMUL.RP", "FFMA", "FFMA.RZ", "FFMA.RM",
             "FFMA.RP", "DADD.RZ", "DADD.RM", "DADD.RP", "DMUL.RZ", "DMUL.RM", "DMUL.RP", "DFMA.RZ", "DFMA.RM", "DFMA.RP", "FMNMX",
             "FMNMX.NAN", "FMNMX.XORSIGN", "FSETP.NE.AND", "FSETP.GT.AND", "FSETP.GE.AND", "FSETP.NEU.AND", "FSETP.GTU.AND",
             "FSETP.GEU.AND", "FSETP.NAN.AND"}}
# The forms only one leg may issue (address arithmetic and compares use LOP3, IADD3, IMAD, ISETP and SHF everywhere).
OWN = {0: ("BMSK", "BREV", "POPC", "FLO", "SGXT"), 1: ("PRMT", "SHF.L.W", "SHF.R.W", "SHF.R.S64"),
       2: ("VIMNMX", "VIADDMNMX", "VABSDIFF"), 3: ("IMAD.HI", "IDP"), 4: ("FADD", "FMUL", "FFMA", "DADD", "DMUL", "DFMA", "FMNMX", "FSETP")}


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_each_leg_issues_its_forms_inside_the_loop_and_no_other_legs():
    kernels, cur = {}, None
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", LIB], text=True).splitlines():
        if "Function : " in ln:
            m = re.search(r"alu_kernelILj(\d)E", ln)
            cur = int(m.group(1)) if m else None
            if cur is not None:
                kernels[cur] = []
            continue
        m = INSN.search(ln)
        if cur is not None and m:
            kernels[cur].append((int(m.group(1), 16), m.group(2), ln))
    assert sorted(kernels) == [0, 1, 2, 3, 4]
    for leg, ins in kernels.items():
        # the iteration loop: from the first table load to the backward branch that closes it
        loads = [a for a, op, _ in ins if op.startswith("LDG")]
        first, last = min(loads), max(a for a, op, _ in ins if op == "BRA")
        inside = Counter(op for a, op, _ in ins if first <= a <= last)
        assert FORMS[leg] <= set(inside), (leg, FORMS[leg] - set(inside))
        ops = Counter(op for _a, op, _ in ins)
        for other, names in OWN.items():
            if other != leg:
                assert not [op for op in ops if op.startswith(names)], (leg, other, [op for op in ops if op.startswith(names)])
        assert not [op for op in ops if op.startswith(("CALL", "LDL", "STL", "HMMA", "IMMA", "DMMA", "HGMMA", "IGMMA", "QGMMA"))], \
            (leg, ops)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_the_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-I" + os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c",
                                             os.path.join(CSRC, "alu_kernels.cu"), "-o", os.path.join(d, "a.o")],
                           capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    assert len(re.findall(r"Compiling entry function '\S*alu_kernel", text)) == 5, text
    assert text.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == 5, text
