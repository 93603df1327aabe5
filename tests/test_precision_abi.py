"""The SM precision probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the library's answers
against oracle/precision.py, the exactness bounds on real data, the operands' encodings, the annotation emitter against
the restatement, the helper form through a stand-in helper, and the instructions and register use of its kernels."""
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
SEEDS = [0, 1, 0x00C0FFEE00000000 + (1 << 58), (1 << 64) - 1, 0xD1B54A32D192ED03, 0x0123456789ABCDEF,
         0x8000000000000000, 0x00C0FFEE00000003 + (1 << 58) + 5 * 0xD1B54A32D192ED03]
U = "GPU-5ca90000-0000-0000-0000-000000000003"
RESULT, SM, FAULT, MAX_SMS = 808, 288, 32, 256

FIELDS = {
    "cro_precision_opts": ("PrecisionOpts", ["iterations", "alu_iterations", "legs", "max_rounds", "test_inject_leg",
                                             "test_inject_sm", "test_inject_iteration", "test_inject_row", "test_inject_col",
                                             "reserved", "test_inject_mask"]),
    "cro_precision_result": ("PrecisionResult", ["status", "verdict", "seed", "call", "sm_count", "legs", "host_ref_ns",
                                                 "nsmid", "bad_sms", "bad_sm", "leg"]),
    "cro_precision_sm": ("PrecisionSm", ["smid", "reserved", "leg"]),
    "cro_precision_fault": ("PrecisionFault", ["leg", "smid", "row", "col", "expected", "actual_bits"]),
}
CONSTANTS = ["CRO_PRECISION_LEG_F64", "CRO_PRECISION_LEG_DFMA", "CRO_PRECISION_LEG_TF32", "CRO_PRECISION_LEG_F16",
             "CRO_PRECISION_LEG_F16ACC", "CRO_PRECISION_LEG_E5M2", "CRO_PRECISION_LEG_HFMA2", "CRO_PRECISION_LEGS",
             "CRO_PRECISION_ALL_LEGS", "CRO_PRECISION_ANSWER_WIDE", "CRO_PRECISION_ANSWER_SMALL128",
             "CRO_PRECISION_ANSWER_SMALL", "CRO_PRECISION_ANSWER_NARROW", "CRO_PRECISION_ANSWERS", "CRO_PRECISION_M",
             "CRO_PRECISION_N", "CRO_PRECISION_K", "CRO_PRECISION_F64_N", "CRO_PRECISION_F64_K", "CRO_PRECISION_TF32_K",
             "CRO_PRECISION_RECORDS", "CRO_PRECISION_MAX_SMS", "CRO_PRECISION_MAX_ITERATIONS",
             "CRO_PRECISION_MAX_ALU_ITERATIONS", "CRO_PRECISION_MAX_ROUNDS"]


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


@pytest.mark.parametrize("seed", SEEDS)
def test_answers_agree_between_library_and_numpy(cro, seed):
    import precision
    for a in range(cro.PRECISION_ANSWERS):
        m, n, _ = precision.SHAPE[a]
        assert (np.array(cro.precision_expected(a, seed)).reshape(m, n) == precision.answer(a, seed)).all(), a


def test_precision_expected_refuses_an_unknown_answer(cro):
    out = (ctypes.c_int64 * (128 * 256))()
    assert cro.lib.cro_precision_expected(4, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_precision_expected(-1, 0, out) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_precision_expected(0, 0, None) == cro.ERR_INVALID_ARG


@pytest.mark.parametrize("seed", SEEDS)
def test_every_partial_sum_stays_within_the_answers_bound(seed):
    import precision
    for a, bound in precision.BOUND.items():
        assert precision.abs_sum(a, seed).max() <= bound, a
    assert precision.BOUND[precision.WIDE] < 1 << 53 and precision.BOUND[precision.NARROW] <= 2048
    assert precision.BOUND[precision.SMALL] <= 1 << 13


def test_the_operands_span_their_ranges(cro):
    import precision
    ranges = {precision.WIDE: (-(1 << 19), (1 << 19) - 1), precision.SMALL: (-4, 3), precision.SMALL128: (-4, 3),
              precision.NARROW: (-2, 1)}
    for a, (lo, hi) in ranges.items():
        x, y = precision.operands(a, SEEDS[5])
        v = np.concatenate([x.ravel(), y.ravel()])
        assert v.min() >= lo and v.max() <= hi and (a == precision.WIDE or set(v.tolist()) == set(range(lo, hi + 1)))


def test_every_small_and_narrow_value_round_trips_through_each_encoding():
    for v in range(-4, 4):
        f32 = np.float32(v).view(np.uint32)
        assert f32 & 0x1FFF == 0 and float(np.uint32(f32 & 0xFFFFE000).view(np.float32)) == v       # tf32: top 19 bits
        f16 = np.float16(v).view(np.uint16)
        assert float(np.float16(v)) == v
        assert f16 & 0xFF == 0 and float(np.uint16(f16 & 0xFF00).view(np.float16)) == v           # e5m2: fp16's top byte
    for bound in (1024, 4096):
        assert all(float(np.float32(v)) == v for v in range(-bound, bound + 1))
    assert all(float(np.float16(v)) == v for v in range(-2048, 2049))                               # every narrow partial sum


def test_the_fold_of_an_answer_is_its_encoding_weighted_by_position():
    import precision
    tile = np.array([[0, -1], [2, -3]], dtype=np.int64)
    for leg, enc in ((0, lambda v: np.float64(v).view(np.uint64)), (2, lambda v: np.float32(v).view(np.uint32)),
                     (4, lambda v: np.float16(v).view(np.uint16))):
        want = sum(int(enc(v)) * (2 * e + 1) for e, v in enumerate(tile.ravel())) % (1 << 64)
        assert precision.cta_fold(leg, tile) == want
    neg0 = precision.encode(2, np.array([0], dtype=np.int64))
    assert int(neg0[0]) == 0


# ---- the emitter against oracle/precision.py ----------------------------------------------------------------------
def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "sm_count": r.sm_count, "legs": r.legs, "bad_sms": r.bad_sms,
            "bad_sm": list(r.bad_sm),
            "leg": [{"ops": L.ops, "ns": L.ns, "sms_covered": L.sms_covered, "mismatches": L.mismatches,
                     "fold_mismatches": L.fold_mismatches, "unpublished": L.unpublished, "slowest_sm": L.slowest_sm,
                     "slow_permille": L.slow_permille} for L in r.leg]}


def make_result(cro, rng, **kw):
    r = cro.PrecisionResult()
    r.status = kw.get("status", 0)
    r.verdict = kw.get("verdict", 0)
    r.sm_count = kw.get("sm_count", rng.choice([132, 114, 1, 256]))
    r.legs = kw.get("legs", rng.choice([0x7F, 0x7F, 0x03, 0x7C, 0x40, rng.randrange(0, 128)]))
    n_bad = kw.get("bad_sms", rng.choice([0, 0, 1, 3, 16, 17, 132]))
    r.bad_sms = n_bad
    for i, x in enumerate(sorted(rng.sample(range(256), min(n_bad, 16)))):
        r.bad_sm[i] = x
    for i in range(7):
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
    rng = random.Random(20261016)
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
    import precision
    seen = set()
    for r in crafted(cro):
        got = cro.emit_precision_annotations_json(r).encode()
        want = precision.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(precision.annotations(as_dict(r))["cohdi.io/probe-precision-verdict"])
    assert seen == {"ok", "sm", "all", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.PrecisionResult()
    r.status, r.verdict, r.sm_count, r.legs, r.bad_sms = cro.ERR_CHECKSUM, cro.COMPUTE_SM, 132, 0x7F, 2
    r.bad_sm[0], r.bad_sm[1] = 7, 131
    for i in range(7):
        r.leg[i].sms_covered = 132
        r.leg[i].ops, r.leg[i].ns = 3 * 10 ** 12, 10 ** 7
    r.leg[2].sms_covered = 130
    r.leg[6].fold_mismatches = 1
    r.leg[1].mismatches = 1
    r.leg[4].slowest_sm, r.leg[4].slow_permille = 9, 1234
    ann = json.loads(cro.emit_precision_annotations_json(r))
    p = "cohdi.io/probe-precision-"
    assert ann == {p + "verdict": "sm", p + "sms": "130/132", p + "bad-sms": "7,131", p + "failed-legs": "dfma,hfma2",
                   p + "f64-gflops": "300000", p + "tf32-gflops": "300000", p + "f16-gflops": "300000",
                   p + "f16acc-gflops": "300000", p + "e5m2-gflops": "300000", p + "slowest-sm": "9 1234"}


def test_emitter_rejects_a_null_result(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_precision_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_probe_precision_without_a_context_is_refused(cro):
    r = cro.PrecisionResult()
    n, n_sms = ctypes.c_int(-1), ctypes.c_int(-1)
    sms = (cro.PrecisionSm * 4)()
    faults = (cro.PrecisionFault * 4)()
    assert cro.lib.cro_probe_precision(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(n_sms), faults, 4,
                                       ctypes.byref(n)) == cro.ERR_INVALID_ARG


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
assert sys.argv[1] == "precision-raw" and len(sys.argv) == 15, sys.argv
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
    cro.probe_precision_uuid(None, U, iterations=9, alu_iterations=5, legs=0b1010110, max_rounds=11,
                             inject=(0, 131, 8, -1, 63, 1 << 63), cap=6)
    s = seen(tmp_path)
    assert s["cvd"] == U
    argv = s["argv"]
    assert argv[:2] == ["precision-raw", U] and len(argv) == 14
    assert int(argv[2]) and int(argv[2]) & 0xFF == 0
    assert argv[3:] == [str(v) for v in (9, 5, 0b1010110, 11, 0, 131, 8, -1, 63, 1 << 63, 6)]
    cro.probe_precision_uuid(None, U)
    assert seen(tmp_path)["argv"][3:] == ["0", "0", str(cro.PRECISION_ALL_LEGS), "0", "0", "0", "0", "0", "0", "0", "256"]


def test_each_call_passes_a_new_seed_base(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    bases = []
    for _ in range(3):
        cro.probe_precision_uuid(None, U)
        bases.append(int(seen(tmp_path)["argv"][2]))
    assert len(set(bases)) == len(bases) and all(b and b & 0xFF == 0 for b in bases), [hex(b) for b in bases]


def test_result_sms_and_faults_come_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, seed=12)
    r, sms, faults, ns = cro.probe_precision_uuid(None, U)
    with open(os.path.join(str(tmp_path), "out.bin"), "rb") as f:
        out = f.read()
    head = RESULT + 16 + MAX_SMS * SM
    assert r.status == cro.ERR_CHECKSUM and ns > 0 and bytes(r) == out[:RESULT]
    assert len(sms) == 2 and b"".join(bytes(s) for s in sms) == out[RESULT + 16:RESULT + 16 + 2 * SM]
    assert len(faults) == 3 and b"".join(bytes(f) for f in faults) == out[head:]
    fake(tmp_path, monkeypatch, status=cro.OK)
    assert cro.probe_precision_uuid(None, U)[0].status == cro.OK


@pytest.mark.parametrize("how", [dict(extra="x"), dict(n_sms=MAX_SMS + 1)], ids=["one-more", "n_sms"])
def test_malformed_output_is_loud(cro, tmp_path, monkeypatch, how):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, **how)
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_precision_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "precision helper for %s failed" % U in str(e.value)


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    import time
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_precision_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "precision helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


REFUSED = [dict(legs=0x80), dict(iterations=65537), dict(alu_iterations=4097), dict(max_rounds=65),
           dict(inject=(7, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 1)),
           dict(inject=(0, -2, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 64, 1)),
           dict(inject=(1, 0, 0, 0, 64, 1)), dict(inject=(2, 0, 0, 0, 256, 1)), dict(inject=(0, 0, 0, -2, 0, 1)),
           dict(inject=(2, 0, 3, 0, 0, 1), iterations=3), dict(inject=(6, 0, 2, 0, 0, 1), alu_iterations=2),
           dict(inject=(2, 0, 0, 0, 0, 1 << 32)), dict(inject=(5, 0, 0, 0, 0, 1 << 32)), dict(inject=(4, 0, 0, 0, 0, 1 << 16)),
           dict(inject=(6, 0, 0, 0, 0, 1 << 16))]


@pytest.mark.parametrize("kw", REFUSED, ids=[json.dumps(k) for k in REFUSED])
def test_arguments_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_precision_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "): precision probe: legs must be" in str(e.value)
    assert not marker.exists()


def test_the_largest_legal_options_do_reach_the_helper(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_precision_uuid(None, U, iterations=65536, alu_iterations=4096, max_rounds=64, inject=(0, 255, 65535, 127, 63, (1 << 64) - 1))
    assert seen(tmp_path)["argv"][3:7] == ["65536", "4096", str(cro.PRECISION_ALL_LEGS), "64"]
    cro.probe_precision_uuid(None, U, inject=(4, 255, 0, 127, 255, 0xFFFF))
    assert seen(tmp_path)["argv"][-2] == str(0xFFFF)


@pytest.mark.parametrize("argv", [["precision-raw", U, "0"], ["precision-raw", U] + ["0"] * 13, ["precision-raw"]],
                         ids=["short", "long", "bare"])
def test_cli_refuses_a_wrong_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64


# ---- the kernels ----------------------------------------------------------------------------------------------------
def _tool(name):
    return shutil.which(name) or ("/usr/local/cuda/bin/" + name if os.path.exists("/usr/local/cuda/bin/" + name) else None)


@pytest.mark.skipif(_tool("cuobjdump") is None, reason="cuobjdump is not installed")
def test_the_library_issues_every_precision_instruction(cro):
    sass = subprocess.check_output([_tool("cuobjdump"), "-sass", cro.LIB_PATH], text=True)
    for op in ("DMMA.16x8x16", "DFMA", "HGMMA.64x256x8.F32.TF32", "HGMMA.64x256x16.F16", "QGMMA.64x256x32.F32.E5M2.E5M2",
               "HFMA2"):
        assert op in sass, op
    # f16 inputs with f32 accumulation: the F16 leg's kernel (the compute probe's bf16 form also spells HGMMA...F32)
    f16 = [blk for blk in sass.split("Function : ") if blk.startswith("_ZN3cro") and "precision_kernelILj3E" in blk.split("\n")[0]]
    assert len(f16) == 1 and "HGMMA.64x256x16.F32 " in f16[0] and ".BF16" not in f16[0]


@pytest.mark.skipif(_tool("nvcc") is None, reason="nvcc is not installed")
def test_no_precision_kernel_spills(tmp_path):
    out = subprocess.run([_tool("nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-c", os.path.join(CSRC, "precision_kernels.cu"), "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True, check=True).stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", out)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len([e for e in entries if "precision_kernel" in e]) == 7 and len(spills) >= 7, out
    assert all(s == ("0", "0") for s in spills), out


def _sass_pin():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_kernel_sass
    return make_kernel_sass, json.load(open(os.path.join(ROOT, "tests", "golden", "precision_sass.json")))


@pytest.mark.skipif(_tool("cuobjdump") is None or _tool("nvcc") is None, reason="the CUDA tools are not installed")
def test_precision_kernels_sass_and_ptxas_are_pinned(cro):
    # every precision kernel's machine code and resources as recorded (tests/golden/make_kernel_sass.py)
    mk, want = _sass_pin()
    got = mk.sass_digests(mk.obj_of("precision_kernels.cu"))
    assert sorted(got) == sorted(want["sass_sha256"])
    assert got == want["sass_sha256"], [k for k in got if got[k] != want["sass_sha256"][k]]
    assert mk.ptxas_lines("precision_kernels.cu") == want["ptxas"]
