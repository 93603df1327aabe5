"""The L2 probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the annotation emitter and the
classification against oracle/l2.py, the L2 health reader through a stand-in NVML, and the march kernel as ptxas and
cuobjdump see it (no spills, no local memory, every buffer access an L1-bypassing 128-bit .STRONG.GPU one)."""
import ctypes
import json
import os
import random
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
U = "GPU-5ca90000-0000-0000-0000-000000000003"

FIELDS = {
    "cro_l2_opts": ("L2Opts", ["bytes", "iterations", "a1_counters", "a2_counters", "deadline_ms", "test_inject_leg",
                               "test_inject_sm", "test_inject_element", "test_inject_iteration", "test_inject_word",
                               "test_inject_mask"]),
    "cro_l2_health": ("L2Health", ["nvml", "threshold_exceeded", "sram_corrected", "sram_uncorrected", "l2_corrected",
                                   "l2_uncorrected", "unc_bucket_l2"]),
    "cro_l2_result": ("L2Result", [
        "status", "verdict", "seed", "seed_atomic", "call", "bytes", "sm_count", "nsmid", "ctas", "blocks", "delta",
        "iterations", "cuda_error", "health", "sms_covered", "unpublished", "mismatches", "recorded", "overflow",
        "sms_listed", "bad_sms", "bad_lines", "bad_sm", "bad_line", "fold_xor", "fold_sum", "fold_wsum", "expect_xor",
        "expect_sum", "expect_wsum", "fold_ok", "a1_counters", "a2_counters", "a2_tickets", "a1_bad", "a2_holes", "a2_bad",
        "a1_bad_counter", "a2_bad_counter", "element_ns", "march_ns", "march_bytes", "a1_ns", "a1_check_ns", "a2_ns",
        "a2_check_ns", "l2_bytes", "wall_ns", "helper_ns", "before", "after"]),
    "cro_l2_sm": ("L2Sm", ["smid", "mark", "launches", "reserved", "mismatches", "last", "words_read", "ns"]),
    "cro_l2_fault": ("L2Fault", ["element", "iteration", "smid", "cta", "writer_cta", "writer_smid", "word", "expected",
                                 "actual", "line", "reserved"]),
}
CONSTANTS = ["CRO_L2_BLOCK_BYTES", "CRO_L2_MIN_BYTES", "CRO_L2_MAX_L2_MULTIPLE", "CRO_L2_ELEMENTS", "CRO_L2_RECORDS",
             "CRO_L2_MAX_SMS", "CRO_L2_MAX_ITERATIONS", "CRO_L2_MAX_A1_COUNTERS", "CRO_L2_MAX_A2_COUNTERS", "CRO_L2_MAX_LINES",
             "CRO_L2_MAX_COUNTERS", "CRO_L2_MARCH", "CRO_L2_A1", "CRO_L2_A2", "CRO_L2_NONE", "CRO_L2_SM", "CRO_L2_LINE",
             "CRO_L2_ATOMIC", "CRO_L2_ALL", "CRO_L2_PERSISTENT", "CRO_L2_INTERMITTENT",
             "CRO_L2_HEALTH_SRAM_CORRECTED_DURING", "CRO_L2_HEALTH_SRAM_UNCORRECTED_DURING",
             "CRO_L2_HEALTH_L2_CORRECTED_DURING", "CRO_L2_HEALTH_L2_UNCORRECTED_DURING", "CRO_L2_HEALTH_THRESHOLD_EXCEEDED",
             "CRO_L2_HEALTH_L2_BUCKET", "CRO_L2_NVML_SRAM_CORRECTED", "CRO_L2_NVML_SRAM_UNCORRECTED",
             "CRO_L2_NVML_L2_CORRECTED", "CRO_L2_NVML_L2_UNCORRECTED", "CRO_L2_NVML_STATUS"]


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
        assert [f for f, _ in cls._fields_] == fields, cname
        for f in fields:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k


# ---- the emitter against oracle/l2.py -------------------------------------------------------------------------------
def as_dict(r):
    d = {f: getattr(r, f) for f in ("status", "verdict", "cuda_error", "sm_count", "sms_covered", "unpublished", "fold_ok",
                                    "overflow", "bytes", "iterations", "march_bytes", "march_ns", "health", "bad_sms",
                                    "bad_lines", "a1_bad", "a2_bad", "a2_holes")}
    for f in ("mismatches", "bad_sm", "bad_line", "a1_bad_counter", "a2_bad_counter"):
        d[f] = list(getattr(r, f))
    return d


def make_result(cro, rng, **kw):
    r = cro.L2Result()
    r.status = kw.get("status", 0)
    r.verdict = kw.get("verdict", rng.randrange(6))
    r.cuda_error = kw.get("cuda_error", 0)
    r.sm_count = rng.choice([132, 114, 0])
    r.sms_covered = rng.choice([r.sm_count, 120, 0, rng.randrange(256)])
    r.bytes = rng.choice([32 << 20, 1 << 20, rng.randrange(1 << 34)])
    r.iterations = rng.choice([0, 1, 16, 256])
    r.march_bytes = rng.choice([0, rng.randrange(1 << 44)])
    r.march_ns = rng.choice([0, 1, rng.randrange(1 << 30)])
    r.bad_sms = kw.get("bad_sms", rng.choice([0, 0, 1, 2, 16, 17, 132]))
    r.bad_lines = kw.get("bad_lines", rng.choice([0, 0, 1, 8, 9, 4096]))
    r.a1_bad = kw.get("a1_bad", rng.choice([0, 0, 1, 8, 9, 65536]))
    r.a2_bad = kw.get("a2_bad", rng.choice([0, 0, 1, 7, 1024]))
    r.a2_holes = rng.choice([0, 0, 1, 1 << 20])
    r.overflow = rng.choice([0, 0, 1])
    for j in range(16):
        r.bad_sm[j] = rng.randrange(256)
    for j in range(8):
        r.bad_line[j] = rng.randrange(1 << 34) * 8
        r.a1_bad_counter[j] = rng.randrange(1 << 20)
        r.a2_bad_counter[j] = rng.randrange(8192)
    r.health = kw.get("health", rng.randrange(64))
    return r


def crafted(cro):
    rng = random.Random(20261015)
    yield cro.L2Result()
    for st, ce in [(0, 0), (cro.ERR_CHECKSUM, 0), (cro.ERR_CUDA, 214), (cro.ERR_CUDA, 0), (cro.ERR_OOM, 0),
                   (cro.ERR_INVALID_ARG, 0), (cro.ERR_DEADLINE, 0), (cro.ERR_UNSUPPORTED, 0)]:
        for v in range(6):
            yield make_result(cro, rng, status=st, cuda_error=ce, verdict=v)
    for h in range(64):
        yield make_result(cro, rng, health=h)
    for cap in (0, 1, 8, 9, 16, 17):
        yield make_result(cro, rng, bad_sms=cap, bad_lines=cap, a1_bad=cap, a2_bad=cap, status=cro.ERR_CHECKSUM)
    for _ in range(300):
        yield make_result(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM, cro.ERR_CHECKSUM, cro.ERR_CUDA]),
                          cuda_error=rng.choice([0, 214, 999]))


def test_emitter_equals_the_restatement(cro):
    import l2
    seen, n = set(), 0
    for r in crafted(cro):
        got = cro.emit_l2_annotations_json(r).encode()
        want = l2.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(l2.annotations(as_dict(r))["cohdi.io/probe-l2-verdict"].split(":")[0])
        n += 1
    assert n > 400 and seen == {"ok", "sm", "line", "atomic", "all", "cuda-error", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.L2Result()
    r.status, r.verdict, r.sm_count, r.sms_covered, r.bytes, r.iterations = cro.ERR_CHECKSUM, cro.L2_LINE, 132, 132, 32 << 20, 16
    r.march_bytes, r.march_ns = 10 * (32 << 20) * 16, 1000000
    r.bad_lines, r.bad_line[0], r.bad_line[1] = 2, 8, 4096
    r.a2_bad, r.a2_holes, r.a2_bad_counter[0] = 1, 1, 17
    r.health = cro.L2_HEALTH_SRAM_CORRECTED_DURING | cro.L2_HEALTH_L2_BUCKET
    p = "cohdi.io/probe-l2-"
    assert json.loads(cro.emit_l2_annotations_json(r)) == {
        p + "verdict": "line", p + "sms": "132/132", p + "bytes": str(32 << 20), p + "iterations": "16",
        p + "march-gbs": str(10 * (32 << 20) * 16 // 1000000), p + "bad-lines": "8,4096", p + "a2-bad-counters": "17",
        p + "a2-holes": "1", p + "health": "sram-corrected,l2-bucket"}


def test_null_arguments_are_refused(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_l2_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_l2_health(None, ctypes.byref(cro.L2Health())) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_l2_health(b"GPU-x", None) == cro.ERR_INVALID_ARG
    r, k, ks = cro.L2Result(), ctypes.c_int(-1), ctypes.c_int(-1)
    sms, faults = (cro.L2Sm * 4)(), (cro.L2Fault * 4)()
    assert cro.lib.cro_probe_l2(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    assert cro.lib.cro_selftest_l2_classify(None, sms, 0, faults, 0) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_selftest_l2_classify(ctypes.byref(r), None, 1, faults, 0) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_selftest_l2_classify(ctypes.byref(r), sms, 0, None, 2) == cro.ERR_INVALID_ARG


# ---- the classification against oracle/l2.py ------------------------------------------------------------------------
def record_set(cro, rng, kind):
    """A result, SM entries and records of one of the shapes the probe can report."""
    G = rng.choice([132, 114, 8])
    covered = sorted(rng.sample(range(256), G))
    r = cro.L2Result()
    r.sms_covered = len(covered)
    r.fold_ok = 0 if kind == "fold" else 1
    r.unpublished = 1 if kind == "silent" else 0
    faults = []

    def add(smid, word, element, iteration):
        f = cro.L2Fault()
        f.smid, f.word, f.element, f.iteration = smid, word, element, iteration
        faults.append(f)

    words = rng.sample(range(1 << 22), 64)
    if kind in ("reader", "mixed", "overflow"):
        for s in rng.sample(covered, rng.choice([1, 2, 5])):
            for w in rng.sample(words, rng.randrange(1, 6)):
                add(s, w, rng.randrange(1, 6), rng.randrange(4))
    if kind in ("line", "mixed"):
        for w in rng.sample(words, rng.randrange(1, 12)):
            for s in rng.sample(covered, rng.randrange(2, 6)):
                add(s, w, rng.randrange(1, 6), rng.randrange(4))
    if kind == "every-sm":
        for s in covered:
            add(s, rng.choice(words), 3, 0)
    if kind == "atomic":
        r.a1_bad = rng.choice([0, 1, 3])
        r.a2_bad = 0 if r.a1_bad else rng.choice([1, 2])
    rng.shuffle(faults)
    per = {}
    for f in faults:
        per.setdefault(f.smid, [0] * 6)[f.element] += 1
    if kind == "overflow":                                    # exact counts past the records, on SMs with none recorded too
        r.overflow = 1
        for s in rng.sample(covered, 3):
            per.setdefault(s, [0] * 6)[rng.randrange(1, 6)] += rng.randrange(1, 1 << 20)
    sms = []
    for s in covered:
        e = cro.L2Sm()
        e.smid = s
        m = per.get(s, [0] * 6)
        for k in range(6):
            e.mismatches[k] = m[k]
            # fewer blocks than CTAs leaves some SMs without a block in an element; a reader of an element read it
            e.words_read[k] = 0 if k == 0 else 2048 * (m[k] > 0 or rng.random() < 0.8) * rng.choice([1, 2])
        e.last = rng.choice([0, m[rng.randrange(6)]])
        sms.append(e)
    for k in range(6):
        r.mismatches[k] = sum(s.mismatches[k] for s in sms)
    return r, sms, faults


def sm_dict(s):
    return {"smid": s.smid, "mismatches": list(s.mismatches), "last": s.last, "words_read": list(s.words_read)}


def test_classification_equals_the_restatement(cro):
    import l2
    rng = random.Random(11)
    kinds = ["none", "reader", "line", "mixed", "atomic", "overflow", "every-sm", "fold", "silent"]
    seen = set()
    for i in range(540):
        r, sms, faults = record_set(cro, rng, kinds[i % len(kinds)])
        got, got_sms, got_faults = cro.selftest_l2_classify(r, sms, faults)
        want = l2.classify(as_dict(r), [sm_dict(s) for s in sms],
                           [{"element": f.element, "iteration": f.iteration, "smid": f.smid, "word": f.word} for f in faults])
        assert (got.verdict, got.status, got.bad_sms, list(got.bad_sm), got.bad_lines, list(got.bad_line)) == \
            (want["verdict"], want["status"], want["bad_sms"], want["bad_sm"], want["bad_lines"], want["bad_line"]), kinds[i % 9]
        assert {s.smid: s.mark for s in got_sms} == want["marks"]
        assert [f.line for f in got_faults] == want["line"]
        seen.add(got.verdict)
    assert seen == {cro.L2_NONE, cro.L2_SM, cro.L2_LINE, cro.L2_ATOMIC, cro.L2_ALL}


def test_a_word_two_readers_saw_wrong_is_a_line_and_one_reader_is_the_sm(cro):
    r = cro.L2Result()
    r.sms_covered, r.fold_ok = 132, 1
    faults = []
    for smid, word in ((3, 100), (9, 100), (5, 7), (5, 8)):
        f = cro.L2Fault()
        f.smid, f.word, f.element = smid, word, 2
        faults.append(f)
    sms = []
    for s, last in ((3, 1), (5, 0), (9, 0), (11, 0)):
        e = cro.L2Sm()
        e.smid, e.last = s, last
        e.mismatches[2] = {3: 1, 5: 2, 9: 1, 11: 0}[s]
        e.words_read[2] = 4096
        sms.append(e)
    got, got_sms, got_faults = cro.selftest_l2_classify(r, sms, faults)
    assert got.verdict == cro.L2_LINE and got.status == cro.ERR_CHECKSUM
    assert got.bad_lines == 1 and got.bad_line[0] == 800 and got.bad_sms == 1 and got.bad_sm[0] == 5
    assert [f.line for f in got_faults] == [1, 1, 0, 0]
    assert [s.mark for s in got_sms] == [cro.L2_PERSISTENT, cro.L2_INTERMITTENT, cro.L2_INTERMITTENT, 0]


def test_a_fault_every_reader_of_an_element_saw_is_all_even_when_some_sms_read_nothing_there(cro):
    """W below G blocks: in one element half the SMs own no block.  Every SM that did read in it failing is a common
    cause, not the half that happened to read; one reader that read it right makes it the failing SMs' own."""
    import l2
    r = cro.L2Result()
    r.fold_ok, r.sms_covered = 1, 132
    sms, faults = [], []
    for s in range(132):
        e = cro.L2Sm()
        e.smid = s
        for k in range(1, 6):
            e.words_read[k] = 2048 if (s + k) % 2 else 0
        if e.words_read[3]:
            e.mismatches[3] = e.last = 2048
            f = cro.L2Fault()
            f.smid, f.word, f.element = s, 2048 * s, 3
            faults.append(f)
        sms.append(e)
    got, _, _ = cro.selftest_l2_classify(r, sms, faults)
    assert got.verdict == cro.L2_ALL and got.bad_sms == 66
    assert l2.classify(as_dict(r), [sm_dict(s) for s in sms], [{"element": 3, "iteration": 0, "smid": f.smid, "word": f.word}
                                                             for f in faults])["verdict"] == l2.ALL
    reader = next(s for s in sms if s.words_read[3])       # one reader of M3 read it right
    reader.mismatches[3] = reader.last = 0
    faults = [f for f in faults if f.smid != reader.smid]
    got, _, _ = cro.selftest_l2_classify(r, sms, faults)
    assert got.verdict == cro.L2_SM and got.bad_sms == 65


# ---- the L2 health reader through a stand-in NVML -------------------------------------------------------------------
READER = r"""
import ctypes, importlib, json, os, sys
sys.path.insert(0, sys.argv[1])
cro = importlib.import_module("composable-resource-operator_b200")
out = []
for env, uuid in json.loads(sys.argv[2]):
    os.environ["FAKE_L2_HEALTH"] = env
    h = cro.read_l2_health(uuid)
    out.append({f: getattr(h, f) for f, _ in cro.L2Health._fields_})
print(json.dumps(out))
"""


def read_through(tmp_path, cases, no_status=False):
    d = tmp_path / ("nvml_nostatus" if no_status else "nvml")
    d.mkdir()
    lib = d / "libnvidia-ml.so.1"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-Werror", "-o", str(lib), os.path.join(HERE, "fake_nvml_l2.c")]
                          + (["-DNO_SRAM_STATUS"] if no_status else []))
    env = dict(os.environ, LD_LIBRARY_PATH=str(d) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([sys.executable, "-c", READER, ROOT, json.dumps(cases)], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout)


def test_health_reader_passes_nvml_values_through(cro, tmp_path):
    line = "%s 17 2 5 1 1 3 %d"
    other = "GPU-00000000-0000-0000-0000-000000000009 99 99 99 99 0 0 0"
    cases = [(line % (U, 0), U), (other + ";" + line % (U, 0), U)] + [(line % (U, m), U) for m in range(1, 32)]
    cases.append((line % (U, 0), "GPU-not-listed"))
    got = read_through(tmp_path, cases)
    for (env, uuid), h in zip(cases, got):
        if uuid != U:
            assert h == {f: 0 for f in h}
            continue
        refuse = int(env.split()[-1])
        assert h == {"nvml": 31 & ~refuse, "sram_corrected": 0 if refuse & 1 else 17, "sram_uncorrected": 0 if refuse & 2 else 2,
                     "l2_corrected": 0 if refuse & 4 else 5, "l2_uncorrected": 0 if refuse & 8 else 1,
                     "threshold_exceeded": 0 if refuse & 16 else 1, "unc_bucket_l2": 0 if refuse & 16 else 3}, (refuse, h)


def test_a_library_without_the_sram_status_leaves_its_fields_clear(cro, tmp_path):
    (h,) = read_through(tmp_path, [("%s 1 0 4 0 1 9 0" % U, U)], no_status=True)
    assert h == {"nvml": 15, "threshold_exceeded": 0, "sram_corrected": 1, "sram_uncorrected": 0, "l2_corrected": 4,
                 "l2_uncorrected": 0, "unc_bucket_l2": 0}


def test_health_bits_never_change_the_verdict_or_status(cro):
    """The classification reads no health field: a clean result stays ok and a failed one keeps its verdict whatever
    NVML said before and after the call."""
    sm = cro.L2Sm()
    sm.smid, sm.words_read[1] = 4, 2048
    for health in range(64):
        for before, after in ((0, 31), (31, 31), (31, 0)):
            r = cro.L2Result()
            r.fold_ok, r.health = 1, health
            r.before.nvml, r.after.nvml = before, after
            r.before.sram_corrected, r.after.sram_corrected, r.after.threshold_exceeded, r.after.unc_bucket_l2 = 1, 9, 1, 5
            got, _, _ = cro.selftest_l2_classify(r, [sm], [])
            assert (got.verdict, got.status, got.health) == (cro.L2_NONE, cro.OK, health)
            r.a2_bad = 1
            got, _, _ = cro.selftest_l2_classify(r, [sm], [])
            assert (got.verdict, got.status) == (cro.L2_ATOMIC, cro.ERR_CHECKSUM)


# ---- the rotation map ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [5, 8, 114, 132, 144])
def test_every_word_is_read_by_five_ctas_none_of_them_its_writer(G):
    import l2
    d = l2.delta(G)
    assert 0 < 4 * d < G
    for b in range(3 * G):
        readers = [l2.owner(b, e, G) for e in range(1, 6)]
        assert len(set(readers)) == 5
        assert all(l2.owner(b, e - 1, G) != l2.owner(b, e, G) for e in range(1, 6))
    assert l2.delta(4) == 0


def test_a1_closed_forms_equal_the_word_by_word_sums():
    import l2
    seed, n, G = 0x1234567890ABCDEF, 37, 9
    s, x = l2.a1_counters(seed, n, G)
    for i in range(n):
        vs = [l2.pattern(seed, j * n + i) for j in range(G)]
        assert int(s[i]) == sum(vs) & l2.U64
        acc = 0
        for v in vs:
            acc ^= v
        assert int(x[i]) == acc


# ---- the march kernel as the compiler built it ----------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_l2_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "l2_kernels.cu"), "-o",
                                             os.path.join(d, "l.o")], capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\S+)'", text)
    assert len(kernels) == 6 and all("l2_" in k for k in kernels), kernels
    assert text.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == 6, text


def march_sass(obj):
    lines, on = [], False
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", obj], text=True).splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            on = "l2_march_kernel" in m.group(1)
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if on and m:
            lines.append(m.group(1))
    return lines


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_every_march_access_bypasses_l1(cro):
    ops = march_sass(os.path.join(CSRC, "build", "l2_kernels.cu.o"))
    assert ops, "no l2_march_kernel in the object"
    assert not [o for o in ops if o.split(".")[0] in ("LDL", "STL", "LD", "ST", "LDG.E.CONSTANT")]     # no local memory
    loads = [o for o in ops if o.startswith("LDG")]
    vec = [o for o in ops if o.startswith(("LDG", "STG")) and ".128" in o]
    # the buffer: four loads and four stores per batch, each 128-bit .STRONG.GPU (ld / st.relaxed.gpu: L1 bypassed)
    assert sum(o.startswith("LDG") for o in vec) == 4 and sum(o.startswith("STG") for o in vec) >= 4, vec
    assert all(o.endswith(".128.STRONG.GPU") for o in vec), vec
    # the only other load is the record claim's volatile read of the claim count, which bypasses L1 too
    assert all(".STRONG." in o for o in loads), loads


# ---- the helper form (cro_probe_l2_uuid) through a stand-in helper named by CRO_HELPER_PATH ---------------------------
# l2-raw's stdout: cro_l2_result (616 bytes), uint64_t n_sms and n, CRO_L2_MAX_SMS cro_l2_sm entries, then n faults.
L2_HELPER = """
import json, os, struct, sys
d = os.path.dirname(os.path.abspath(sys.argv[0]))
open(os.path.join(d, "argv.json"), "w").write(json.dumps({"argv": sys.argv[1:], "cvd": os.environ.get("CUDA_VISIBLE_DEVICES")}))
assert sys.argv[1] == "l2-raw" and len(sys.argv) == 15, sys.argv
seed_base, nbytes, iters, a1, a2, leg, sm, element, iteration, word, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(616)
struct.pack_into("<iIQQQQ", r, 0, -6, 1, seed_base + 7, seed_base + 8, 0, nbytes)
struct.pack_into("<II", r, 144, 1, 0)
struct.pack_into("<H", r, 152, sm & 0xFFFF)
struct.pack_into("<Q", r, 128, n)
sms = bytearray(256 * 128)
struct.pack_into("<I", sms, 0, 4)
struct.pack_into("<I", sms, 128, sm & 0xFFFFFFFF)
faults = b"".join(struct.pack("<IIIIIIQQQII", element & 0xFFFFFFFF, iteration, sm & 0xFFFFFFFF, 9, 8, 5, (word + j) & (2 ** 64 - 1), 5, 5 ^ mask, 0, 0) for j in range(n))
sys.stdout.buffer.write(bytes(r) + struct.pack("<QQ", 2, n) + bytes(sms) + faults + b"%s")
sys.exit(1)
"""


def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, 0o755)
    return p


def seen(tmp_path):
    with open(os.path.join(str(tmp_path), "argv.json")) as f:
        return json.load(f)


def test_helper_argv_carries_every_option_and_a_fresh_seed_base(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, L2_HELPER % ""))
    bases = []
    for _ in range(3):
        cro.probe_l2_uuid(None, U, bytes=4 << 20, iterations=3, a1_counters=100, a2_counters=7,
                          inject=(cro.L2_MARCH, 9, -1, 2, 4095, 1 << 37), cap=5)
        s = seen(tmp_path)
        assert s["cvd"] == U and s["argv"][:2] == ["l2-raw", U] and len(s["argv"]) == 14
        assert s["argv"][3:] == [str(v) for v in (4 << 20, 3, 100, 7, 0, 9, -1, 2, 4095, 1 << 37, 5)]
        bases.append(int(s["argv"][2]))
    assert len(set(bases)) == 3 and all(b and b & 0xFF == 0 for b in bases), [hex(b) for b in bases]
    cro.probe_l2_uuid(None, U)                                          # defaults go to the helper as zeroes
    assert seen(tmp_path)["argv"][3:] == ["0"] * 10 + ["256"]


def test_helper_result_sms_and_faults_come_back(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, L2_HELPER % ""))
    r, sms, faults = cro.probe_l2_uuid(None, U, iterations=3, inject=(cro.L2_MARCH, 9, 4, 2, 100, 1 << 37))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and list(r.bad_sm[:r.bad_sms]) == [9]
    assert r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2 and [s.smid for s in sms] == [4, 9]
    assert [(f.element, f.iteration, f.smid, f.cta, f.writer_cta, f.writer_smid, f.word, f.actual) for f in faults] == \
        [(4, 2, 9, 9, 8, 5, 100 + j, 5 ^ (1 << 37)) for j in range(3)]
    r, sms, faults = cro.probe_l2_uuid(None, U, cap=2)                  # the helper is asked for at most cap faults
    assert len(faults) == 2 and r.recorded == 2


def test_helper_failures_are_loud(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, L2_HELPER % "x"))       # one byte too many
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_l2_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "L2 helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_l2_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_helper_is_killed_at_its_deadline_and_reaped(cro, tmp_path, monkeypatch):
    import time
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_l2_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "L2 helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


@pytest.mark.parametrize("kw", [dict(bytes=(1 << 20) - 16384), dict(bytes=(1 << 20) + 8), dict(iterations=257),
                                dict(a1_counters=(1 << 20) + 1), dict(a2_counters=8193), dict(deadline_ms=-1),
                                dict(inject=(3, 0, 1, 0, 0, 1)), dict(inject=(0, 256, 1, 0, 0, 1)),
                                dict(inject=(0, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 6, 0, 0, 1)),
                                dict(inject=(0, 0, 1, 2, 0, 1), iterations=2), dict(inject=(0, 0, 1, 0, -2, 1)),
                                dict(inject=(0, 0, 1, 0, (4 << 20) // 8, 1), bytes=4 << 20),
                                dict(inject=(1, 0, 0, 0, 65536, 1)), dict(inject=(2, 0, 0, 0, 1024, 1)),
                                dict(inject=(2, 0, 0, 0, 3, 1 << 40))])
def test_helper_options_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_l2_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "L2 probe:" in str(e.value), kw
    assert not marker.exists()


def test_helper_null_arguments_are_refused(cro):
    r, k, ks = cro.L2Result(), ctypes.c_int(-1), ctypes.c_int(-1)
    sms, faults = (cro.L2Sm * 4)(), (cro.L2Fault * 4)()
    assert cro.lib.cro_probe_l2_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                     ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_l2_uuid(None, U.encode(), None, ctypes.byref(r), sms, 4, ctypes.byref(ks), None, 4,
                                     ctypes.byref(k)) == cro.ERR_INVALID_ARG


@pytest.mark.parametrize("argv", [["l2-raw", U, "0"], ["l2-raw", U] + ["0"] * 11, ["l2-raw", U] + ["0"] * 13])
def test_cli_refuses_a_wrong_l2_raw_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64
