"""The SM compute probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the operands and answers
of the library, the C oracle and numpy against each other, the exactness bound on real data, the annotation emitter
against oracle/compute.py, and the tensor-core instructions in the library's SASS."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = [0, 1, 0x00C0FFEE00000000 + (1 << 61), (1 << 64) - 1, 0xD1B54A32D192ED03, 0x0123456789ABCDEF,
         0x8000000000000000, 0x00C0FFEE00000003 + (1 << 61) + 5 * 0xD1B54A32D192ED03]

FIELDS = {
    "cro_compute_opts": ("ComputeOpts", ["iterations", "alu_iterations", "legs", "max_rounds", "test_inject_leg",
                                         "test_inject_sm", "test_inject_iteration", "test_inject_row", "test_inject_col",
                                         "test_inject_mask"]),
    "cro_compute_leg": ("ComputeLeg", ["iterations", "rounds", "ops", "ns", "timer_ns", "sms_covered", "complete",
                                       "mismatches", "fold_mismatches", "recorded", "failed_sms", "unpublished", "ctas",
                                       "slowest_sm", "slow_permille", "reserved", "fold", "expect_fold"]),
    "cro_compute_result": ("ComputeResult", ["status", "verdict", "seed", "call", "sm_count", "legs", "host_ref_ns", "nsmid",
                                             "bad_sms", "bad_sm", "leg"]),
    "cro_compute_sm_leg": ("ComputeSmLeg", ["mismatches", "fold_mismatches", "ns", "cycles", "ctas", "mark"]),
    "cro_compute_sm": ("ComputeSm", ["smid", "reserved", "leg"]),
    "cro_compute_fault": ("ComputeFault", ["leg", "smid", "row", "col", "expected", "actual"]),
}
CONSTANTS = ["CRO_COMPUTE_M", "CRO_COMPUTE_N", "CRO_COMPUTE_K", "CRO_COMPUTE_LEG_S8", "CRO_COMPUTE_LEG_BF16",
             "CRO_COMPUTE_LEG_E4M3", "CRO_COMPUTE_LEG_FFMA", "CRO_COMPUTE_LEG_IMAD", "CRO_COMPUTE_LEGS",
             "CRO_COMPUTE_ALL_LEGS", "CRO_COMPUTE_ANSWER_S8", "CRO_COMPUTE_ANSWER_SMALL", "CRO_COMPUTE_RECORDS",
             "CRO_COMPUTE_MAX_SMS", "CRO_COMPUTE_MAX_ITERATIONS", "CRO_COMPUTE_MAX_ALU_ITERATIONS", "CRO_COMPUTE_MAX_ROUNDS",
             "CRO_COMPUTE_NONE", "CRO_COMPUTE_SM", "CRO_COMPUTE_ALL", "CRO_COMPUTE_PERSISTENT", "CRO_COMPUTE_INTERMITTENT"]


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
        for f in fields:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k


@pytest.fixture(scope="module")
def c_oracle(_built):
    import compute
    return compute.CComputeOracle()


def test_operands_agree_between_the_c_oracle_and_numpy(c_oracle):
    import compute
    rng = random.Random(7)
    for seed in SEEDS:
        for answer in (compute.S8, compute.SMALL):
            a, b = compute.operands(answer, seed)
            for _ in range(64):
                m, k, n = rng.randrange(128), rng.randrange(256), rng.randrange(256)
                assert c_oracle.operand(answer, seed, m * 256 + k) == a[m, k]
                assert c_oracle.operand(answer, seed, 32768 + k * 256 + n) == b[k, n]
            if answer == compute.SMALL:
                assert a.min() >= -4 and a.max() <= 3
            else:
                assert a.min() >= -128 and a.max() <= 127


@pytest.mark.parametrize("seed", SEEDS)
def test_answers_agree_between_library_c_oracle_and_numpy(cro, c_oracle, seed):
    import compute
    for answer in (cro.COMPUTE_ANSWER_S8, cro.COMPUTE_ANSWER_SMALL):
        want = compute.answer(answer, seed)
        assert (c_oracle.answer(answer, seed) == want).all()
        assert (np.array(cro.compute_expected(answer, seed)).reshape(128, 256) == want).all()
    assert np.abs(compute.answer(compute.S8, seed)).max() <= 256 * 128 * 128


def test_compute_expected_refuses_an_unknown_answer(cro):
    out = (ctypes.c_int32 * (128 * 256))()
    assert cro.lib.cro_compute_expected(2, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_compute_expected(0, 0, None) == cro.ERR_INVALID_ARG


@pytest.mark.parametrize("seed", SEEDS[:3])
def test_small_int_partial_sums_stay_within_2_to_the_12(seed):
    import compute
    assert compute.max_partial_sum(compute.SMALL, seed) <= 4096


def test_the_fragment_covers_the_tile_once():
    import compute
    rows, cols = compute.fragment()
    assert sorted(zip(rows.ravel().tolist(), cols.ravel().tolist())) == [(m, n) for m in range(128) for n in range(256)]


# ---- the emitter against oracle/compute.py --------------------------------------------------------------------------
def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "sm_count": r.sm_count, "legs": r.legs, "bad_sms": r.bad_sms,
            "bad_sm": list(r.bad_sm),
            "leg": [{"ops": L.ops, "ns": L.ns, "sms_covered": L.sms_covered, "mismatches": L.mismatches,
                     "fold_mismatches": L.fold_mismatches, "unpublished": L.unpublished, "slowest_sm": L.slowest_sm,
                     "slow_permille": L.slow_permille} for L in r.leg]}


def make_result(cro, rng, **kw):
    r = cro.ComputeResult()
    r.status = kw.get("status", 0)
    r.verdict = kw.get("verdict", 0)
    r.sm_count = kw.get("sm_count", rng.choice([132, 114, 1, 256]))
    r.legs = kw.get("legs", rng.choice([0x1F, 0x1F, 0x07, 0x18, 0x01, rng.randrange(0, 32)]))
    n_bad = kw.get("bad_sms", rng.choice([0, 0, 1, 3, 16, 17, 132]))
    r.bad_sms = n_bad
    ids = sorted(rng.sample(range(256), min(n_bad, 16)))
    for i, x in enumerate(ids):
        r.bad_sm[i] = x
    for i in range(5):
        L = r.leg[i]
        L.ops = rng.choice([0, rng.randrange(0, 1 << 50)])
        L.ns = kw.get("ns", rng.choice([0, 1, rng.randrange(1, 1 << 32)]))
        L.sms_covered = kw.get("covered", rng.choice([r.sm_count, r.sm_count, rng.randrange(0, r.sm_count + 1)]))
        L.mismatches = rng.choice([0, 0, 0, 1, rng.randrange(0, 1 << 40)])
        L.fold_mismatches = rng.choice([0, 0, 0, 1, 256])
        L.unpublished = rng.choice([0, 0, 0, 0, 1])
        L.slowest_sm = rng.randrange(0, 256)
        L.slow_permille = rng.choice([0, 1000, rng.randrange(1000, 3000)])
    return r


def crafted(cro):
    rng = random.Random(20261015)
    yield make_result(cro, rng, ns=0, bad_sms=0)                                                  # zero ns everywhere
    yield make_result(cro, rng, legs=0)                                                            # no leg ran
    for st, v in [(0, 0), (cro.ERR_CHECKSUM, cro.COMPUTE_SM), (cro.ERR_CHECKSUM, cro.COMPUTE_ALL),
                  (cro.ERR_CHECKSUM, cro.COMPUTE_NONE), (cro.ERR_CUDA, 0), (cro.ERR_INVALID_ARG, 0), (cro.ERR_UNSUPPORTED, 0)]:
        yield make_result(cro, rng, status=st, verdict=v)
    for n in (0, 1, 15, 16, 17, 200):                                                             # empty and truncated lists
        yield make_result(cro, rng, status=cro.ERR_CHECKSUM, verdict=cro.COMPUTE_SM, bad_sms=n)
    yield make_result(cro, rng, covered=0)                                                         # incomplete coverage
    for _ in range(400):
        yield make_result(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM]), verdict=rng.choice([0, 1, 2]))


def test_emitter_equals_the_restatement(cro):
    import compute
    seen = set()
    for r in crafted(cro):
        got = cro.emit_compute_annotations_json(r).encode()
        want = compute.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(compute.annotations(as_dict(r))["cohdi.io/probe-compute-verdict"])
    assert seen == {"ok", "sm", "all", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.ComputeResult()
    r.status, r.verdict, r.sm_count, r.legs, r.bad_sms = cro.ERR_CHECKSUM, cro.COMPUTE_SM, 132, 0x1F, 2
    r.bad_sm[0], r.bad_sm[1] = 7, 131
    for i in range(5):
        r.leg[i].sms_covered = 132
        r.leg[i].ops, r.leg[i].ns = 3 * 10 ** 12, 10 ** 7
    r.leg[1].sms_covered = 130
    r.leg[3].fold_mismatches = 1
    r.leg[4].slowest_sm, r.leg[4].slow_permille = 9, 1234
    import json
    ann = json.loads(cro.emit_compute_annotations_json(r))
    p = "cohdi.io/probe-compute-"
    assert ann == {p + "verdict": "sm", p + "sms": "130/132", p + "bad-sms": "7,131", p + "failed-legs": "ffma",
                   p + "s8-gops": "300000", p + "bf16-gflops": "300000", p + "e4m3-gflops": "300000",
                   p + "slowest-sm": "9 1234"}


def test_emitter_rejects_a_null_result(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_compute_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_probe_compute_without_a_context_is_refused(cro):
    r = cro.ComputeResult()
    n, n_sms = ctypes.c_int(-1), ctypes.c_int(-1)
    sms = (cro.ComputeSm * 4)()
    faults = (cro.ComputeFault * 4)()
    assert cro.lib.cro_probe_compute(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(n_sms), faults, 4,
                                     ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not installed")
def test_the_library_issues_every_tensor_core_flavour(cro):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.check_output([tool, "-sass", cro.LIB_PATH], text=True)
    for op in ("IGMMA", "HGMMA", "QGMMA"):
        assert op in sass, op
