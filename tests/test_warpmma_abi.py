"""The SM warp-MMA probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the library's answers
against the compute and precision probes' and oracle/warpmma.py, the exactness of the substitution's predicted rows,
the annotation emitter and the classification against the restatements, the helper form through a stand-in helper,
and the instructions and register use of its kernels."""
import ctypes
import json
import os
import random
import re
import shutil
import stat
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
SEEDS = [0, 1, 0x00C0FFEE00000000 + (1 << 55), (1 << 64) - 1, 0xD1B54A32D192ED03, 0x0123456789ABCDEF,
         0x8000000000000000, 0x00C0FFEE00000003 + (1 << 55) + 5 * 0xD1B54A32D192ED03]
U = "GPU-5ca90000-0000-0000-0000-000000000004"
RESULT, SM, FAULT, MAX_SMS = 704, 248, 24, 256
U64 = (1 << 64) - 1
STRIDE = 0xD1B54A32D192ED03
# the substitutions tests/test_warpmma_probe.py makes: (leg, row, k-step) on the first and on the last covered SM
ADDR_CASES = [(0, 93, 3), (0, 6, 15), (1, 93, 0), (1, 6, 31), (2, 93, 17), (2, 6, 30), (3, 93, 1), (3, 6, 26),
              (4, 93, 8), (4, 6, 21)]

FIELDS = {
    "cro_warpmma_opts": ("WarpMmaOpts", ["iterations", "legs", "max_rounds", "test_inject_leg", "test_inject_sm",
                                         "test_inject_iteration", "test_inject_row", "test_inject_col", "test_inject_mask",
                                         "test_addr", "test_addr_leg", "test_addr_sm", "test_addr_iteration", "test_addr_row",
                                         "test_addr_kstep"]),
    "cro_warpmma_result": ("WarpMmaResult", ["status", "verdict", "seed", "call", "sm_count", "legs", "host_ref_ns", "nsmid",
                                             "bad_sms", "bad_sm", "leg"]),
    "cro_warpmma_sm": ("WarpMmaSm", ["smid", "reserved", "leg"]),
    "cro_warpmma_fault": ("WarpMmaFault", ["leg", "smid", "row", "col", "expected", "actual_bits"]),
}
CONSTANTS = ["CRO_WARPMMA_LEG_S8", "CRO_WARPMMA_LEG_F16", "CRO_WARPMMA_LEG_BF16", "CRO_WARPMMA_LEG_TF32",
             "CRO_WARPMMA_LEG_F16ACC", "CRO_WARPMMA_LEG_MOVE", "CRO_WARPMMA_LEGS", "CRO_WARPMMA_ALL_LEGS",
             "CRO_WARPMMA_ANSWER_S8", "CRO_WARPMMA_ANSWER_SMALL", "CRO_WARPMMA_ANSWER_SMALL128", "CRO_WARPMMA_ANSWER_NARROW",
             "CRO_WARPMMA_ANSWER_MOVE", "CRO_WARPMMA_ANSWERS", "CRO_WARPMMA_M", "CRO_WARPMMA_N", "CRO_WARPMMA_K",
             "CRO_WARPMMA_TF32_K", "CRO_WARPMMA_RECORDS", "CRO_WARPMMA_MAX_SMS", "CRO_WARPMMA_MAX_ITERATIONS",
             "CRO_WARPMMA_MAX_ROUNDS", "CRO_SM_LEGS_WARPMMA"]


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
    assert got[("cro_warpmma_result", "sizeof")] == RESULT and got[("cro_warpmma_sm", "sizeof")] == SM
    assert got[("cro_warpmma_fault", "sizeof")] == FAULT and got[("cro_warpmma_opts", "sizeof")] == 64


def tile(values):
    return np.array(values, dtype=np.int64).reshape(128, 256)


@pytest.mark.parametrize("seed", SEEDS)
def test_answers_are_the_compute_and_precision_probes_and_the_block_transposed_tile(cro, seed):
    import warpmma
    got = [tile(cro.warpmma_expected(a, seed)) for a in range(cro.WARPMMA_ANSWERS)]
    assert (got[0] == tile(cro.compute_expected(cro.COMPUTE_ANSWER_S8, seed))).all()
    assert (got[1] == tile(cro.compute_expected(cro.COMPUTE_ANSWER_SMALL, seed))).all()
    assert (got[2] == tile(cro.precision_expected(cro.PRECISION_ANSWER_SMALL128, seed))).all()
    assert (got[3] == tile(cro.precision_expected(cro.PRECISION_ANSWER_NARROW, seed))).all()
    from oracle import pattern_word
    s = np.array([(pattern_word(seed, e // 4) >> (16 * (e % 4))) & 0xFFFF for e in range(128 * 256)]).reshape(128, 256)
    blocks = s.reshape(16, 8, 32, 8).transpose(0, 2, 1, 3)               # [a][b][i][j] = S[8a + i][8b + j]
    want = np.swapaxes(blocks, 2, 3).transpose(0, 2, 1, 3).reshape(128, 256)
    assert (got[4] == want).all() and (got[4] == warpmma.answer(warpmma.MOVE, seed)).all()
    for a in range(4):
        assert (got[a] == warpmma.answer(a, seed)).all(), a


def test_warpmma_expected_refuses_an_unknown_answer(cro):
    out = (ctypes.c_int32 * (128 * 256))()
    assert cro.lib.cro_warpmma_expected(5, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_warpmma_expected(-1, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_warpmma_expected(0, 0, None) == cro.ERR_INVALID_ARG


def gpu_seeds():
    """The operand seeds of the GPU test's in-process calls: seed_base | minor + 2^55 + k * stride for its first calls."""
    return [((0x00C0FFEE00000000 | minor) + (1 << 55) + k * STRIDE) & U64 for minor in range(8) for k in range(48)]


def test_substituted_rows_are_exact_and_differ_from_the_clean_row():
    """The predicted row of every substitution the GPU test makes is exact in its leg's accumulator (every partial sum
    within 2^24 in f32, 2^31 in int32, 2048 in f16) and differs from the clean row in at least one column, at every
    seed those calls can have."""
    import warpmma
    bound = {0: (1 << 31) - 1, 1: 1 << 24, 2: 1 << 24, 3: 1 << 24, 4: 2048}
    for seed in gpu_seeds()[::7] + SEEDS:
        for leg, row, kstep in ADDR_CASES:
            a = warpmma.LEG_ANSWER[leg]
            assert warpmma.substituted_partial_bound(leg, seed, row, kstep) <= bound[leg], (leg, seed)
            good, bad = warpmma.answer(a, seed), warpmma.substituted_row(leg, seed, row, kstep)
            assert (bad != good[row]).any(), (leg, row, kstep, hex(seed))


def test_the_predicted_row_is_the_product_with_the_substituted_segment():
    import warpmma
    seed = SEEDS[5]
    for leg, row, kstep in ADDR_CASES:
        a, b = warpmma.operands(warpmma.LEG_ANSWER[leg], seed)
        per = 16 // warpmma.LEG_ELEM[leg]
        a2 = a.copy()
        a2[row, kstep * per:(kstep + 1) * per] = a[row ^ 1, kstep * per:(kstep + 1) * per]
        full = a2 @ b
        assert (full[row] == warpmma.substituted_row(leg, seed, row, kstep)).all()
        assert (np.delete(full, row, axis=0) == np.delete(a @ b, row, axis=0)).all()
        assert warpmma.k_steps(leg) == (16 if leg == 0 else 32)


def test_the_fold_of_an_answer_is_its_encoding_weighted_by_position():
    import warpmma
    t = np.array([[0, -1], [2, 65535]], dtype=np.int64)
    w = [2 * e + 1 for e in range(4)]
    assert warpmma.cta_fold(0, t) == sum((int(v) & 0xFFFFFFFF) * x for v, x in zip(t.ravel(), w)) % (1 << 64)
    assert warpmma.cta_fold(5, t) == sum((int(v) & 0xFFFF) * x for v, x in zip(t.ravel(), w)) % (1 << 64)
    small = np.array([[0, -1], [2, -3]], dtype=np.int64)
    assert warpmma.cta_fold(1, small) == sum(int(np.float32(v).view(np.uint32)) * x for v, x in zip(small.ravel(), w))
    assert warpmma.cta_fold(4, small) == sum(int(np.float16(v).view(np.uint16)) * x for v, x in zip(small.ravel(), w))
    assert warpmma.value_bits(4, -3) == 0xC200 and warpmma.value_bits(5, 0xBEEF) == 0xBEEF


# ---- the emitter against oracle/warpmma.py ---------------------------------------------------------------------------
def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "sm_count": r.sm_count, "legs": r.legs, "bad_sms": r.bad_sms,
            "bad_sm": list(r.bad_sm),
            "leg": [{"ops": L.ops, "ns": L.ns, "sms_covered": L.sms_covered, "mismatches": L.mismatches,
                     "fold_mismatches": L.fold_mismatches, "unpublished": L.unpublished, "slowest_sm": L.slowest_sm,
                     "slow_permille": L.slow_permille} for L in r.leg]}


def make_result(cro, rng, **kw):
    r = cro.WarpMmaResult()
    r.status = kw.get("status", 0)
    r.verdict = kw.get("verdict", 0)
    r.sm_count = kw.get("sm_count", rng.choice([132, 114, 1, 256]))
    r.legs = kw.get("legs", rng.choice([0x3F, 0x3F, 0x03, 0x3C, 0x20, rng.randrange(0, 64)]))
    n_bad = kw.get("bad_sms", rng.choice([0, 0, 1, 3, 16, 17, 132]))
    r.bad_sms = n_bad
    for i, x in enumerate(sorted(rng.sample(range(256), min(n_bad, 16)))):
        r.bad_sm[i] = x
    for i in range(6):
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
    rng = random.Random(20261017)
    yield make_result(cro, rng, ns=0, bad_sms=0)
    yield make_result(cro, rng, legs=0)
    for st, v in [(0, 0), (cro.ERR_CHECKSUM, cro.COMPUTE_SM), (cro.ERR_CHECKSUM, cro.COMPUTE_ALL),
                  (cro.ERR_CHECKSUM, cro.COMPUTE_NONE), (cro.ERR_CUDA, 0), (cro.ERR_INVALID_ARG, 0), (cro.ERR_UNSUPPORTED, 0)]:
        yield make_result(cro, rng, status=st, verdict=v)
    for n in (0, 1, 15, 16, 17, 200):
        yield make_result(cro, rng, status=cro.ERR_CHECKSUM, verdict=cro.COMPUTE_SM, bad_sms=n)
    yield make_result(cro, rng, covered=0)
    for _ in range(400):
        yield make_result(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM]), verdict=rng.choice([0, 1, 2]))


def test_emitter_equals_the_restatement(cro):
    import warpmma
    seen = set()
    for r in crafted(cro):
        got = cro.emit_warpmma_annotations_json(r).encode()
        want = warpmma.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(warpmma.annotations(as_dict(r))["cohdi.io/probe-warpmma-verdict"])
    assert seen == {"ok", "sm", "all", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.WarpMmaResult()
    r.status, r.verdict, r.sm_count, r.legs, r.bad_sms = cro.ERR_CHECKSUM, cro.COMPUTE_SM, 132, 0x3F, 2
    r.bad_sm[0], r.bad_sm[1] = 7, 131
    for i in range(6):
        r.leg[i].sms_covered = 132
        r.leg[i].ops, r.leg[i].ns = 3 * 10 ** 12, 10 ** 7
    r.leg[2].sms_covered = 130
    r.leg[5].fold_mismatches = 1
    r.leg[1].mismatches = 1
    r.leg[5].ops = 7 * 10 ** 9
    r.leg[4].slowest_sm, r.leg[4].slow_permille = 9, 1234
    ann = json.loads(cro.emit_warpmma_annotations_json(r))
    p = "cohdi.io/probe-warpmma-"
    assert ann == {p + "verdict": "sm", p + "sms": "130/132", p + "bad-sms": "7,131", p + "failed-legs": "f16,move",
                   p + "s8-gops": "300000", p + "f16-gflops": "300000", p + "bf16-gflops": "300000",
                   p + "tf32-gflops": "300000", p + "f16acc-gflops": "300000", p + "move-gelems": "700",
                   p + "slowest-sm": "9 1234"}


def test_emitter_rejects_a_null_result(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_warpmma_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_probe_warpmma_without_a_context_is_refused(cro):
    r = cro.WarpMmaResult()
    n, n_sms = ctypes.c_int(-1), ctypes.c_int(-1)
    sms = (cro.WarpMmaSm * 4)()
    faults = (cro.WarpMmaFault * 4)()
    assert cro.lib.cro_probe_warpmma(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(n_sms), faults, 4,
                                     ctypes.byref(n)) == cro.ERR_INVALID_ARG


# ---- the classification against oracle/warpmma.py --------------------------------------------------------------------
def plain(x):
    if isinstance(x, ctypes.Structure):
        return {f: plain(getattr(x, f)) for f, _ in x._fields_}
    if isinstance(x, ctypes.Array):
        return [plain(v) for v in x]
    return x


def bitmap(smids):
    w = [0, 0, 0, 0]
    for s in smids:
        w[s // 64] |= 1 << (s % 64)
    return w


def random_call(rng):
    grid = rng.choice([1, 2, 3, 5, 8, 16, 33])
    k = rng.randrange(1 << 40)
    pool = rng.sample(range(256), rng.choice([1, max(1, grid // 2), grid, grid + 3]))
    unsupported = rng.random() < 0.03
    rounds, claims, records, its = [], [], [], []
    for leg in range(6):
        per_round, seen = [], set()
        for _ in range(rng.choice([0, 1, 2, 3]) if rng.random() < 0.1 else rng.choice([1, 1, 2, 4])):
            ctas = []
            for _ in range(grid):
                bad = rng.random() < 0.15
                ctas.append(dict(stamp=k if rng.random() < 0.93 else rng.choice([U64, k + 1]), t0=rng.randrange(1 << 20),
                                 t1=rng.randrange(1 << 20), cycles=rng.choice([0, 100, rng.randrange(1 << 36)]),
                                 mismatches=rng.randrange(1, 1 << 20) if bad and rng.random() < 0.6 else 0,
                                 fold_mismatches=rng.randrange(1, 256) if bad else 0, fold=rng.randrange(1 << 64),
                                 smid=rng.choice(pool), nsmid=257 if unsupported and rng.random() < 0.05 else 132))
            seen |= {c["smid"] for c in ctas if c["stamp"] == k}
            per_round.append((ctas, bitmap(seen)))
        rounds.append(per_round)
        its.append(rng.choice([1, 2, 4, 256]))
        c = rng.choice([0, 0, 0, 1, 3, 17]) if rng.random() < 0.97 else rng.choice([4096, 4097, 10 ** 7])
        claims.append(c)
        records.append([dict(leg=leg, smid=rng.choice(pool), row=rng.randrange(128), col=rng.randrange(256),
                             expected=rng.randrange(-(1 << 31), 1 << 31), actual_bits=rng.randrange(1 << 32))
                        for _ in range(min(c, 4096))])
    return {"legs": rng.choice([0, 0, rng.randrange(1, 64)]), "iterations": its, "grid": grid, "call": k, "rounds": rounds,
            "claims": claims, "records": records}


def test_classification_equals_the_restatement(cro):
    import warpmma
    rng = random.Random(20261017)
    seen = set()
    for _ in range(300):
        call = random_call(rng)
        rounds = [[([cro.SmCta(**c) for c in ctas], bits) for ctas, bits in call["rounds"][l]] for l in range(6)]
        recs = [[cro.WarpMmaFault(**f) for f in call["records"][l]] for l in range(6)]
        r, sms, faults = cro.selftest_sm_legs_classify(cro.SM_LEGS_WARPMMA, call["iterations"], call["grid"], call["call"],
                                                       rounds, call["claims"], recs, legs=call["legs"])
        want = warpmma.classify(call)
        assert plain(r) == want[0]
        assert [plain(s) for s in sms] == want[1]
        full = lambda f: sorted(f.items())
        assert sorted((plain(f) for f in faults), key=full) == sorted(want[2], key=full)
        seen.add((r.status, r.verdict))
    assert seen >= {(cro.OK, cro.COMPUTE_NONE), (cro.ERR_CHECKSUM, cro.COMPUTE_SM), (cro.ERR_CHECKSUM, cro.COMPUTE_ALL),
                    (cro.ERR_UNSUPPORTED, cro.COMPUTE_NONE)}, seen


# ---- the helper form through a stand-in ---------------------------------------------------------------------------
# It leaves its argv and CUDA_VISIBLE_DEVICES in <dir>/argv.json and writes a result whose bytes come from
# random.Random(<seed>) with the given status, two per-SM entries and min(cap, 3) records.
FAKE = r"""
import json, os, random, struct, sys
d = os.path.dirname(os.path.abspath(sys.argv[0]))
open(os.path.join(d, "argv.json"), "w").write(json.dumps({"argv": sys.argv[1:], "cvd": os.environ.get("CUDA_VISIBLE_DEVICES")}))
cfg = json.loads(%r)
rng = random.Random(cfg["seed"])
blob = lambda k: bytes(rng.randrange(256) for _ in range(k))
assert sys.argv[1] == "warpmma-raw" and len(sys.argv) == 20, sys.argv
n = min(int(sys.argv[-1]), 3)
r = bytearray(blob(%d))
struct.pack_into("<i", r, 0, cfg["status"])
out = bytes(r) + struct.pack("<QQ", cfg.get("n_sms", 2), n) + blob(2 * %d) + bytes((%d - 2) * %d) + blob(%d * n)
out += cfg.get("extra", "").encode()
open(os.path.join(d, "out.bin"), "wb").write(out)
sys.stdout.buffer.write(out)
sys.exit(0 if cfg["status"] == 0 else 1)
"""


def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


def fake(tmp_path, monkeypatch, status=0, seed=1, **cfg):
    cfg.update(status=status, seed=seed)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, FAKE % (json.dumps(cfg), RESULT, SM, MAX_SMS, SM, FAULT)))


def seen(tmp_path):
    with open(os.path.join(str(tmp_path), "argv.json")) as f:
        return json.load(f)


def test_argv_carries_every_option(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_warpmma_uuid(None, U, iterations=9, legs=0b101101, max_rounds=11, inject=(0, 131, 8, -1, 63, 1 << 31),
                           addr=(3, -1, 7, 127, 31), cap=6)
    s = seen(tmp_path)
    assert s["cvd"] == U
    argv = s["argv"]
    assert argv[:2] == ["warpmma-raw", U] and len(argv) == 19
    assert int(argv[2]) and int(argv[2]) & 0xFF == 0
    assert argv[3:] == [str(v) for v in (9, 0b101101, 11, 0, 131, 8, -1, 63, 1 << 31, 1, 3, -1, 7, 127, 31, 6)]
    cro.probe_warpmma_uuid(None, U)
    assert seen(tmp_path)["argv"][3:] == ["0", str(cro.WARPMMA_ALL_LEGS)] + ["0"] * 13 + ["256"]


def test_each_call_passes_a_new_seed_base(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    bases = []
    for _ in range(3):
        cro.probe_warpmma_uuid(None, U)
        bases.append(int(seen(tmp_path)["argv"][2]))
    assert len(set(bases)) == len(bases) and all(b and b & 0xFF == 0 for b in bases), [hex(b) for b in bases]


def test_result_sms_and_faults_come_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, seed=12)
    r, sms, faults, ns = cro.probe_warpmma_uuid(None, U)
    with open(os.path.join(str(tmp_path), "out.bin"), "rb") as f:
        out = f.read()
    head = RESULT + 16 + MAX_SMS * SM
    assert r.status == cro.ERR_CHECKSUM and ns > 0 and bytes(r) == out[:RESULT]
    assert len(sms) == 2 and b"".join(bytes(s) for s in sms) == out[RESULT + 16:RESULT + 16 + 2 * SM]
    assert len(faults) == 3 and b"".join(bytes(f) for f in faults) == out[head:]
    fake(tmp_path, monkeypatch, status=cro.OK)
    assert cro.probe_warpmma_uuid(None, U)[0].status == cro.OK


@pytest.mark.parametrize("how", [dict(extra="x"), dict(n_sms=MAX_SMS + 1)], ids=["one-more", "n_sms"])
def test_malformed_output_is_loud(cro, tmp_path, monkeypatch, how):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, **how)
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_warpmma_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "warpmma helper for %s failed" % U in str(e.value)


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    import time
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_warpmma_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "warpmma helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


REFUSED = [dict(legs=0x40), dict(iterations=65537), dict(max_rounds=65),
           dict(inject=(6, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 1)),
           dict(inject=(0, -2, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)),
           dict(inject=(0, 0, 0, -2, 0, 1)), dict(inject=(2, 0, 3, 0, 0, 1), iterations=3),
           dict(inject=(2, 0, 0, 0, 0, 1 << 32)), dict(inject=(4, 0, 0, 0, 0, 1 << 16)), dict(inject=(5, 0, 0, 0, 0, 1 << 16)),
           dict(addr=(5, 0, 0, 0, 0)), dict(addr=(6, 0, 0, 0, 0)), dict(addr=(-1, 0, 0, 0, 0)),
           dict(addr=(0, 256, 0, 0, 0)), dict(addr=(0, -2, 0, 0, 0)), dict(addr=(0, 0, 256, 0, 0)),
           dict(addr=(0, 0, 0, 128, 0)), dict(addr=(0, 0, 0, 0, 16)), dict(addr=(1, 0, 0, 0, 32)),
           dict(addr=(2, 0, 0, 0, 32)), dict(addr=(3, 0, 0, 0, 32)), dict(addr=(4, 0, 0, 0, 32))]


@pytest.mark.parametrize("kw", REFUSED, ids=[json.dumps(k) for k in REFUSED])
def test_arguments_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_warpmma_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "): warpmma probe: legs must be" in str(e.value)
    assert not marker.exists()


def test_an_addr_flag_other_than_one_is_refused(cro, tmp_path, monkeypatch):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    o = cro.WarpMmaOpts()
    o.test_addr = 2
    r = cro.WarpMmaResult()
    sms, faults = (cro.WarpMmaSm * 4)(), (cro.WarpMmaFault * 4)()
    n, n_sms, ns = ctypes.c_int(), ctypes.c_int(), ctypes.c_uint64()
    assert cro.lib.cro_probe_warpmma_uuid(None, U.encode(), ctypes.byref(o), 0, ctypes.byref(r), sms, 4,
                                          ctypes.byref(n_sms), faults, 4, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert not marker.exists()


def test_the_largest_legal_options_do_reach_the_helper(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_warpmma_uuid(None, U, iterations=65536, max_rounds=64, inject=(3, 255, 65535, 127, 255, (1 << 32) - 1),
                           addr=(4, 255, 65535, 127, 31))
    assert seen(tmp_path)["argv"][3:] == [str(v) for v in (65536, cro.WARPMMA_ALL_LEGS, 64, 3, 255, 65535, 127, 255,
                                                           (1 << 32) - 1, 1, 4, 255, 65535, 127, 31, 256)]
    cro.probe_warpmma_uuid(None, U, inject=(5, 0, 0, 0, 0, 0xFFFF), addr=(0, 0, 0, 0, 15))
    assert seen(tmp_path)["argv"][6:] == [str(v) for v in (5, 0, 0, 0, 0, 0xFFFF, 1, 0, 0, 0, 0, 15, 256)]


@pytest.mark.parametrize("argv", [["warpmma-raw", U, "0"], ["warpmma-raw", U] + ["0"] * 18, ["warpmma-raw"]],
                         ids=["short", "long", "bare"])
def test_cli_refuses_a_wrong_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64


def test_a_helper_that_cannot_see_the_gpu_is_no_device(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_warpmma_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wire_table_covers_the_options_and_round_trips(tmp_path):
    """cro_wire_warpmma against cro_warpmma_opts: every byte of the struct on argv exactly once, every field formatted
    as its own type prints and parsed back byte for byte, and 20 arguments in all."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("helper_wire_program", os.path.join(ROOT, "tests", "test_helper_wire.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    body = ('    { const size_t at[] = {0}, size[] = {0}; '
            'check("warpmma", &cro_wire_warpmma, sizeof(cro_warpmma_opts), at, size, 0); }')
    src = tmp_path / "wire.c"
    src.write_text(mod.PROGRAM.replace("@BODY@", body))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    assert "argc warpmma-raw 20" in out.stdout


# ---- the kernels ----------------------------------------------------------------------------------------------------
def _tool(name):
    return shutil.which(name) or ("/usr/local/cuda/bin/" + name if os.path.exists("/usr/local/cuda/bin/" + name) else None)


FORMS = {0: ["IMMA.16832.S8.S8 "], 1: ["HMMA.16816.F32 "], 2: ["HMMA.16816.F32.BF16 "], 3: ["HMMA.1688.F32.TF32 "],
         4: ["HMMA.16816.F16 "],
         5: ["LDSM.16.M88.4 ", "MOVM.16.MT88 ", "STSM.16.MT88.4 ", "LDSM.16.MT88.4 ", "STSM.16.M88.4 "]}
MMA_OPS = ("HMMA", "IMMA", "DMMA", "BMMA")
CONVERSIONS = ("F2F", "F2I", "I2F", "I2I", "F2FP", "I2FP", "FRND")


@pytest.fixture(scope="module")
def kernels(cro):
    """{leg: [(address, opcode, operands)]} of the library's warp-MMA kernels."""
    sass = subprocess.check_output([_tool("cuobjdump"), "-sass", cro.LIB_PATH], text=True)
    out = {}
    for blk in sass.split("Function : ")[1:]:
        m = re.search(r"warpmma_kernelILj(\d)E", blk.split("\n")[0])
        if m:
            out[int(m.group(1))] = [(int(a, 16), op, rest) for a, op, rest in re.findall(
                r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);", blk)]
    return out


@pytest.mark.skipif(_tool("cuobjdump") is None, reason="cuobjdump is not installed")
def test_each_leg_issues_its_native_forms_and_nothing_emulated(kernels):
    assert sorted(kernels) == list(range(6))
    for leg, ins in kernels.items():
        text = "\n".join(op + " " + rest for _, op, rest in ins)
        for form in FORMS[leg]:
            assert form in text, (leg, form)
        assert "LDSM.16.M88.4 " in text, leg
        if leg in (1, 2, 4):
            assert "LDSM.16.MT88.4 " in text, leg
        mma = {op for _, op, _ in ins if op.startswith(MMA_OPS)}
        assert mma == ({FORMS[leg][0].split()[0]} if leg < 5 else set()), (leg, mma)
        ops = {op for _, op, _ in ins}
        for bad in ("CALL", "HGMMA", "IGMMA", "QGMMA", "LDL", "STL"):
            assert not any(op.startswith(bad) for op in ops), (leg, bad)


@pytest.mark.skipif(_tool("cuobjdump") is None, reason="cuobjdump is not installed")
def test_the_iteration_loop_feeds_the_mma_from_ldsm_only(kernels):
    """Inside each arithmetic leg's iteration loop (the outermost backward branch around its MMAs) the only shared loads
    are LDSM and nothing converts a number: a build that fed an MMA from LDS, or emulated a form, fails here."""
    for leg in range(5):
        ins = kernels[leg]
        loops = []
        for a, op, rest in ins:
            t = re.search(r"0x([0-9a-f]+)", rest)
            if op.startswith("BRA") and t and int(t.group(1), 16) < a:
                loops.append((int(t.group(1), 16), a))
        mma = [a for a, op, _ in ins if op.startswith(MMA_OPS)]
        lo, hi = max((l for l in loops if l[0] <= min(mma) and l[1] >= max(mma)), key=lambda l: l[1] - l[0])
        body = Counter(op for a, op, _ in ins if lo <= a <= hi)
        assert body[FORMS[leg][0].split()[0]] == 32, (leg, body)      # one k-step of 32 n-tiles, rolled
        loads = {op for op in body if op.startswith("LD") and not op.startswith(("LDG", "LDC"))}
        assert loads == {"LDSM.16.M88.4"} | ({"LDSM.16.MT88.4"} if leg in (1, 2, 4) else set()), (leg, loads)
        assert not [op for op in body if op.startswith(CONVERSIONS)], leg


@pytest.mark.skipif(_tool("nvcc") is None, reason="nvcc is not installed")
def test_no_warpmma_kernel_spills(tmp_path):
    out = subprocess.run([_tool("nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(CSRC, "warpmma_kernels.cu"), "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True, check=True).stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", out)
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len([e for e in entries if "warpmma_kernel" in e]) == 6 and len(spills) == 6, out
    assert all(s == ("0", "0", "0") for s in spills), out
    assert all(int(r) <= 255 for r in re.findall(r"Used (\d+) registers", out)), out
