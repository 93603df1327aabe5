"""The SM sparse probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the library's answers
against oracle/sparse.py and the sparse structure of their operands, the exactness bound on real data, the annotation
emitter and the classification against the restatements, the helper form through a stand-in helper, and the
instructions and register use of its kernels."""
import ctypes
import json
import os
import random
import re
import shutil
import stat
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
SEEDS = [0, 1, 0x00C0FFEE00000000 + (1 << 57), (1 << 64) - 1, 0xD1B54A32D192ED03, 0x0123456789ABCDEF,
         0x8000000000000000, 0x00C0FFEE00000003 + (1 << 57) + 5 * 0xD1B54A32D192ED03]
U = "GPU-5ca90000-0000-0000-0000-000000000003"
RESULT, SM, FAULT, MAX_SMS = 704, 248, 24, 256
U64 = (1 << 64) - 1

FIELDS = {
    "cro_sparse_opts": ("SparseOpts", ["iterations", "legs", "max_rounds", "test_inject_leg", "test_inject_sm",
                                       "test_inject_iteration", "test_inject_row", "test_inject_col", "test_inject_mask",
                                       "test_meta", "test_meta_leg", "test_meta_sm", "test_meta_iteration", "test_meta_row",
                                       "test_meta_group"]),
    "cro_sparse_result": ("SparseResult", ["status", "verdict", "seed", "call", "sm_count", "legs", "host_ref_ns", "nsmid",
                                           "bad_sms", "bad_sm", "leg"]),
    "cro_sparse_sm": ("SparseSm", ["smid", "reserved", "leg"]),
    "cro_sparse_fault": ("SparseFault", ["leg", "smid", "row", "col", "expected", "actual_bits"]),
}
CONSTANTS = ["CRO_SPARSE_LEG_S8", "CRO_SPARSE_LEG_E4M3", "CRO_SPARSE_LEG_E5M2", "CRO_SPARSE_LEG_BF16", "CRO_SPARSE_LEG_F16",
             "CRO_SPARSE_LEG_TF32", "CRO_SPARSE_LEGS", "CRO_SPARSE_ALL_LEGS", "CRO_SPARSE_ANSWER_S8", "CRO_SPARSE_ANSWER_SMALL",
             "CRO_SPARSE_ANSWER_SMALL256", "CRO_SPARSE_ANSWER_SMALL128", "CRO_SPARSE_ANSWERS", "CRO_SPARSE_M", "CRO_SPARSE_N",
             "CRO_SPARSE_K", "CRO_SPARSE_K16", "CRO_SPARSE_TF32_K", "CRO_SPARSE_RECORDS", "CRO_SPARSE_MAX_SMS",
             "CRO_SPARSE_MAX_ITERATIONS", "CRO_SPARSE_MAX_ROUNDS", "CRO_SM_LEGS_SPARSE"]


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
    assert got[("cro_sparse_result", "sizeof")] == RESULT and got[("cro_sparse_sm", "sizeof")] == SM
    assert got[("cro_sparse_fault", "sizeof")] == FAULT and got[("cro_sparse_opts", "sizeof")] == 64


@pytest.mark.parametrize("seed", SEEDS)
def test_answers_agree_between_library_and_numpy(cro, seed):
    import sparse
    for a in range(cro.SPARSE_ANSWERS):
        assert (np.array(cro.sparse_expected(a, seed)).reshape(128, 256) == sparse.answer(a, seed)).all(), a


@pytest.mark.parametrize("seed", SEEDS)
def test_the_logical_a_is_sparse_with_every_pair_and_no_zero_kept_value(seed):
    import sparse
    for a in range(4):
        ac, b, pair = sparse.operands(a, seed)
        g, p = sparse.GROUP[a], len(sparse.pairs(a))
        assert (ac != 0).all() and b.shape == (sparse.K[a], 256)
        la = sparse.logical_a(a, seed).reshape(128, -1, g)
        kept = 2 if g == 4 else 1
        assert ((la != 0).sum(axis=2) == kept).all(), a             # 2:4 (TF32: 1:2), exactly where the pair says
        for m in range(128):
            assert set(pair[m].tolist()) == set(range(p)), (a, m)    # every pair in every row
        assert (la.reshape(128, -1) != 0).sum() == ac.size
        lo, hi = (-128, 127) if a == sparse.S8 else (-4, 4)
        assert ac.min() >= lo and ac.max() <= hi and b.min() >= lo and b.max() <= min(hi, 127 if a == sparse.S8 else 3)


def test_sparse_expected_refuses_an_unknown_answer(cro):
    out = (ctypes.c_int32 * (128 * 256))()
    assert cro.lib.cro_sparse_expected(4, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_sparse_expected(-1, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_sparse_expected(0, 0, None) == cro.ERR_INVALID_ARG


@pytest.mark.parametrize("seed", SEEDS)
def test_every_partial_sum_stays_exact_in_its_accumulator(seed):
    """K/2 kept products of at most 2^14 (s8) or 16 (small-int): int32 for S8, f32's 24 bits for the rest, and every
    value a small-int leg reads is exact in e4m3, e5m2, bf16, f16 and tf32."""
    import sparse
    bound = {sparse.S8: 256 * 128 * 128, sparse.SMALL: 256 * 16, sparse.SMALL256: 128 * 16, sparse.SMALL128: 64 * 16}
    for a, b in bound.items():
        assert sparse.abs_sum(a, seed).max() <= b, a
    assert bound[sparse.S8] < 1 << 31 and max(bound[a] for a in (1, 2, 3)) <= 1 << 12
    assert all(float(np.float32(v)) == v for v in range(-4096, 4097))
    import torch
    small = torch.arange(-4, 5, dtype=torch.float32)
    for dt in (torch.float8_e4m3fn, torch.float8_e5m2, torch.bfloat16, torch.float16):
        assert torch.equal(small.to(dt).to(torch.float32), small), dt
    f32 = small.numpy().view(np.uint32)
    assert (f32 & 0x1FFF == 0).all()                                 # tf32 keeps the top 19 bits of an f32


def test_a_substitution_changes_only_its_row():
    import sparse
    for a, (row, group) in ((0, (5, 127)), (1, (0, 0)), (2, (127, 63)), (3, (64, 33))):
        good, bad = sparse.answer(a, SEEDS[5]), sparse.substituted(a, SEEDS[5], row, group)
        diff = np.nonzero((good != bad).any(axis=1))[0].tolist()
        assert diff == [row], (a, diff)


@pytest.mark.parametrize("seed", SEEDS[:4])
def test_the_unselected_thread_pairs_register_gives_a_wrong_answer_in_every_row(seed):
    """In the 16- and 32-bit legs the thread pair a selector does not name holds every pair advanced by one: an
    instruction that read it would compute this answer, wrong in every row, so a clean call pins the selector mapping."""
    import sparse
    for a in (sparse.SMALL256, sparse.SMALL128):
        _, b, pair = sparse.operands(a, seed)
        other = sparse.logical_a(a, seed, (pair + 1) % len(sparse.pairs(a))) @ b
        assert (other != sparse.answer(a, seed)).any(axis=1).all(), a


def test_the_fold_of_an_answer_is_its_encoding_weighted_by_position():
    import sparse
    tile = np.array([[0, -1], [2, -3]], dtype=np.int64)
    want32 = sum(int(np.float32(v).view(np.uint32)) * (2 * e + 1) for e, v in enumerate(tile.ravel())) % (1 << 64)
    wanti = sum((int(v) & 0xFFFFFFFF) * (2 * e + 1) for e, v in enumerate(tile.ravel())) % (1 << 64)
    assert sparse.cta_fold(1, tile) == want32 and sparse.cta_fold(0, tile) == wanti
    assert int(sparse.encode(3, np.array([0], dtype=np.int64))[0]) == 0


# ---- the emitter against oracle/sparse.py ---------------------------------------------------------------------------
def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "sm_count": r.sm_count, "legs": r.legs, "bad_sms": r.bad_sms,
            "bad_sm": list(r.bad_sm),
            "leg": [{"ops": L.ops, "ns": L.ns, "sms_covered": L.sms_covered, "mismatches": L.mismatches,
                     "fold_mismatches": L.fold_mismatches, "unpublished": L.unpublished, "slowest_sm": L.slowest_sm,
                     "slow_permille": L.slow_permille} for L in r.leg]}


def make_result(cro, rng, **kw):
    r = cro.SparseResult()
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
    import sparse
    seen = set()
    for r in crafted(cro):
        got = cro.emit_sparse_annotations_json(r).encode()
        want = sparse.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(sparse.annotations(as_dict(r))["cohdi.io/probe-sparse-verdict"])
    assert seen == {"ok", "sm", "all", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.SparseResult()
    r.status, r.verdict, r.sm_count, r.legs, r.bad_sms = cro.ERR_CHECKSUM, cro.COMPUTE_SM, 132, 0x3F, 2
    r.bad_sm[0], r.bad_sm[1] = 7, 131
    for i in range(6):
        r.leg[i].sms_covered = 132
        r.leg[i].ops, r.leg[i].ns = 3 * 10 ** 12, 10 ** 7
    r.leg[2].sms_covered = 130
    r.leg[5].fold_mismatches = 1
    r.leg[1].mismatches = 1
    r.leg[4].slowest_sm, r.leg[4].slow_permille = 9, 1234
    ann = json.loads(cro.emit_sparse_annotations_json(r))
    p = "cohdi.io/probe-sparse-"
    assert ann == {p + "verdict": "sm", p + "sms": "130/132", p + "bad-sms": "7,131", p + "failed-legs": "e4m3,tf32",
                   p + "s8-gops": "300000", p + "e4m3-gflops": "300000", p + "e5m2-gflops": "300000",
                   p + "bf16-gflops": "300000", p + "f16-gflops": "300000", p + "tf32-gflops": "300000",
                   p + "slowest-sm": "9 1234"}


def test_emitter_rejects_a_null_result(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_sparse_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_probe_sparse_without_a_context_is_refused(cro):
    r = cro.SparseResult()
    n, n_sms = ctypes.c_int(-1), ctypes.c_int(-1)
    sms = (cro.SparseSm * 4)()
    faults = (cro.SparseFault * 4)()
    assert cro.lib.cro_probe_sparse(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(n_sms), faults, 4,
                                    ctypes.byref(n)) == cro.ERR_INVALID_ARG


# ---- the classification against oracle/sparse.py --------------------------------------------------------------------
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
    import sparse
    rng = random.Random(20261017)
    seen = set()
    for _ in range(300):
        call = random_call(rng)
        rounds = [[([cro.SmCta(**c) for c in ctas], bits) for ctas, bits in call["rounds"][l]] for l in range(6)]
        recs = [[cro.SparseFault(**f) for f in call["records"][l]] for l in range(6)]
        r, sms, faults = cro.selftest_sm_legs_classify(cro.SM_LEGS_SPARSE, call["iterations"], call["grid"], call["call"],
                                                       rounds, call["claims"], recs, legs=call["legs"])
        want = sparse.classify(call)
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
assert sys.argv[1] == "sparse-raw" and len(sys.argv) == 20, sys.argv
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
    cro.probe_sparse_uuid(None, U, iterations=9, legs=0b101101, max_rounds=11, inject=(0, 131, 8, -1, 63, 1 << 31),
                          meta=(5, -1, 7, 127, 63), cap=6)
    s = seen(tmp_path)
    assert s["cvd"] == U
    argv = s["argv"]
    assert argv[:2] == ["sparse-raw", U] and len(argv) == 19
    assert int(argv[2]) and int(argv[2]) & 0xFF == 0
    assert argv[3:] == [str(v) for v in (9, 0b101101, 11, 0, 131, 8, -1, 63, 1 << 31, 1, 5, -1, 7, 127, 63, 6)]
    cro.probe_sparse_uuid(None, U)
    assert seen(tmp_path)["argv"][3:] == ["0", str(cro.SPARSE_ALL_LEGS)] + ["0"] * 13 + ["256"]


def test_each_call_passes_a_new_seed_base(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    bases = []
    for _ in range(3):
        cro.probe_sparse_uuid(None, U)
        bases.append(int(seen(tmp_path)["argv"][2]))
    assert len(set(bases)) == len(bases) and all(b and b & 0xFF == 0 for b in bases), [hex(b) for b in bases]


def test_result_sms_and_faults_come_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, seed=12)
    r, sms, faults, ns = cro.probe_sparse_uuid(None, U)
    with open(os.path.join(str(tmp_path), "out.bin"), "rb") as f:
        out = f.read()
    head = RESULT + 16 + MAX_SMS * SM
    assert r.status == cro.ERR_CHECKSUM and ns > 0 and bytes(r) == out[:RESULT]
    assert len(sms) == 2 and b"".join(bytes(s) for s in sms) == out[RESULT + 16:RESULT + 16 + 2 * SM]
    assert len(faults) == 3 and b"".join(bytes(f) for f in faults) == out[head:]
    fake(tmp_path, monkeypatch, status=cro.OK)
    assert cro.probe_sparse_uuid(None, U)[0].status == cro.OK


@pytest.mark.parametrize("how", [dict(extra="x"), dict(n_sms=MAX_SMS + 1)], ids=["one-more", "n_sms"])
def test_malformed_output_is_loud(cro, tmp_path, monkeypatch, how):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, **how)
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sparse_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "sparse helper for %s failed" % U in str(e.value)


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    import time
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sparse_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "sparse helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


REFUSED = [dict(legs=0x40), dict(iterations=65537), dict(max_rounds=65),
           dict(inject=(6, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 1)),
           dict(inject=(0, -2, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)),
           dict(inject=(0, 0, 0, -2, 0, 1)), dict(inject=(2, 0, 3, 0, 0, 1), iterations=3),
           dict(inject=(2, 0, 0, 0, 0, 1 << 32)), dict(meta=(6, 0, 0, 0, 0)), dict(meta=(-1, 0, 0, 0, 0)),
           dict(meta=(0, 256, 0, 0, 0)), dict(meta=(0, -2, 0, 0, 0)), dict(meta=(0, 0, 256, 0, 0)),
           dict(meta=(0, 0, 0, 128, 0)), dict(meta=(0, 0, 0, 0, 128)), dict(meta=(3, 0, 0, 0, 64)),
           dict(meta=(4, 0, 0, 0, 64)), dict(meta=(5, 0, 0, 0, 64))]


@pytest.mark.parametrize("kw", REFUSED, ids=[json.dumps(k) for k in REFUSED])
def test_arguments_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sparse_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "): sparse probe: legs must be" in str(e.value)
    assert not marker.exists()


def test_a_meta_flag_other_than_one_is_refused(cro, tmp_path, monkeypatch):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    o = cro.SparseOpts()
    o.test_meta = 2
    r = cro.SparseResult()
    sms, faults = (cro.SparseSm * 4)(), (cro.SparseFault * 4)()
    n, n_sms, ns = ctypes.c_int(), ctypes.c_int(), ctypes.c_uint64()
    assert cro.lib.cro_probe_sparse_uuid(None, U.encode(), ctypes.byref(o), 0, ctypes.byref(r), sms, 4, ctypes.byref(n_sms),
                                         faults, 4, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert not marker.exists()


def test_the_largest_legal_options_do_reach_the_helper(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_sparse_uuid(None, U, iterations=65536, max_rounds=64, inject=(5, 255, 65535, 127, 255, (1 << 32) - 1),
                          meta=(0, 255, 65535, 127, 127))
    assert seen(tmp_path)["argv"][3:] == [str(v) for v in (65536, cro.SPARSE_ALL_LEGS, 64, 5, 255, 65535, 127, 255,
                                                           (1 << 32) - 1, 1, 0, 255, 65535, 127, 127, 256)]


@pytest.mark.parametrize("argv", [["sparse-raw", U, "0"], ["sparse-raw", U] + ["0"] * 18, ["sparse-raw"]],
                         ids=["short", "long", "bare"])
def test_cli_refuses_a_wrong_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64


# ---- the kernels ----------------------------------------------------------------------------------------------------
def _tool(name):
    return shutil.which(name) or ("/usr/local/cuda/bin/" + name if os.path.exists("/usr/local/cuda/bin/" + name) else None)


@pytest.mark.skipif(_tool("cuobjdump") is None, reason="cuobjdump is not installed")
def test_the_library_issues_every_sparse_instruction(cro):
    sass = subprocess.check_output([_tool("cuobjdump"), "-sass", cro.LIB_PATH], text=True)
    for op in ("IGMMA.SP.64x256x64.S8.S8", "QGMMA.SP.64x256x64.F32.E4M3.E4M3", "QGMMA.SP.64x256x64.F32.E5M2.E5M2",
               "HGMMA.SP.64x256x32.F32.BF16", "HGMMA.SP.64x256x16.F32.TF32"):
        assert op in sass, op
    f16 = [blk for blk in sass.split("Function : ") if blk.startswith("_ZN3cro") and "sparse_kernelILj4E" in blk.split("\n")[0]]
    assert len(f16) == 1 and "HGMMA.SP.64x256x32.F32 " in f16[0] and ".BF16" not in f16[0]
    for leg in (3, 4, 5):           # both selectors in every iteration
        blk = [b for b in sass.split("Function : ") if b.startswith("_ZN3cro") and "sparse_kernelILj%dE" % leg in b.split("\n")[0]]
        sp = re.findall(r"GMMA\.SP\.[^;]*?, (0x[01])\b", blk[0])
        assert set(sp) == {"0x0", "0x1"}, (leg, sp)


@pytest.mark.skipif(_tool("nvcc") is None, reason="nvcc is not installed")
def test_no_sparse_kernel_spills(tmp_path):
    out = subprocess.run([_tool("nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(CSRC, "sparse_kernels.cu"), "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True, check=True).stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", out)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len([e for e in entries if "sparse_kernel" in e]) == 6 and len(spills) >= 6, out
    assert all(s == ("0", "0") for s in spills), out
    assert "C7519" not in out, out          # no warpgroup.arrive between the .sp instructions
