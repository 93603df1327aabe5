"""The whole-HBM scan without a GPU: the ctypes mirrors against the header as gcc lays it out, the annotation emitter
against oracle/scan.py, the DRAM health readers through a stand-in NVML, the scan helper's wire format and deadline,
and the probe kernels the scan reuses, unchanged (per-kernel SASS and ptxas resources against the golden record)."""
import ctypes
import json
import os
import random
import shutil
import stat
import struct
import subprocess
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
U = "GPU-5ca90000-0000-0000-0000-000000000001"

FIELDS = {
    "cro_scan_opts": ("ScanOpts", ["max_bytes", "reserve_bytes", "seed", "deadline_ms", "reserved0", "test_chunk_bytes",
                                   "test_force_first", "test_force_count", "test_force_and", "test_force_or"]),
    "cro_hbm_health": ("HbmHealth", ["nvml", "remap_corrected", "remap_uncorrected", "remap_pending", "remap_failure",
                                     "histogram", "ecc_corrected", "ecc_uncorrected"]),
    "cro_scan_pass": ("ScanPass", ["invert", "words_scanned", "mismatches", "recorded", "granules", "bit_flips"]),
    "cro_scan_chunk": ("ScanChunk", ["word0", "bytes", "fold_xor", "fold_sum", "fold_wsum", "expect_xor", "expect_sum",
                                     "expect_wsum"]),
    "cro_scan_report": ("ScanReport", ["status", "cuda_error", "health", "complete", "seed", "total_bytes", "free_bytes",
                                       "held_bytes", "covered_bytes", "n_chunks", "elements_done", "located", "recorded",
                                       "flip_or", "element_ns", "alloc_ns", "nvml_ns", "wall_ns", "helper_ns", "before",
                                       "after", ("pass", "pass_"), "chunk"]),
}
CONSTANTS = ["CRO_SCAN_CHUNK_BYTES", "CRO_SCAN_RESERVE_BYTES", "CRO_SCAN_MAX_CHUNKS", "CRO_SCAN_PASSES", "CRO_SCAN_ELEMENTS",
             "CRO_SCAN_HEALTH_ECC_CORRECTED_DURING", "CRO_SCAN_HEALTH_ECC_UNCORRECTED_DURING", "CRO_SCAN_HEALTH_REMAP_PENDING",
             "CRO_SCAN_HEALTH_REMAP_FAILURE", "CRO_HBM_NVML_ECC_CORRECTED", "CRO_HBM_NVML_ECC_UNCORRECTED",
             "CRO_HBM_NVML_REMAP", "CRO_HBM_NVML_HISTOGRAM"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            c = f[0] if isinstance(f, tuple) else f
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
        for f in fields:
            c, p = f if isinstance(f, tuple) else (f, f)
            assert getattr(cls, p).offset == got[(cname, c)], (cname, c)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k


# ---- the emitter against oracle/scan.py -----------------------------------------------------------------------------
def health_dict(h):
    return {"nvml": h.nvml, "ecc_corrected": h.ecc_corrected, "ecc_uncorrected": h.ecc_uncorrected,
            "remap_corrected": h.remap_corrected, "remap_uncorrected": h.remap_uncorrected,
            "remap_pending": h.remap_pending, "remap_failure": h.remap_failure, "histogram": list(h.histogram)}


def as_dict(r):
    return {"status": r.status, "cuda_error": r.cuda_error, "health": r.health, "seed": r.seed,
            "covered_bytes": r.covered_bytes, "free_bytes": r.free_bytes, "element_ns": list(r.element_ns),
            "pass": [{"mismatches": P.mismatches, "granules": P.granules, "bit_flips": list(P.bit_flips)} for P in r.pass_],
            "before": health_dict(r.before), "after": health_dict(r.after)}


def fill_health(h, rng, nvml):
    h.nvml = nvml
    h.ecc_corrected = rng.choice([0, 1, rng.randrange(1 << 40)]) if nvml & 1 else 0
    h.ecc_uncorrected = rng.choice([0, 0, 3]) if nvml & 2 else 0
    if nvml & 4:
        h.remap_corrected, h.remap_uncorrected = rng.choice([0, 2]), rng.choice([0, 0, 1])
        h.remap_pending, h.remap_failure = rng.choice([0, 0, 1]), rng.choice([0, 0, 1])
    if nvml & 8:
        for b in range(5):
            h.histogram[b] = rng.choice([0, rng.randrange(10000)])


def make_report(cro, rng, **kw):
    r = cro.ScanReport()
    r.status = kw.get("status", 0)
    r.cuda_error = kw.get("cuda_error", 0)
    r.seed = rng.randrange(1 << 64)
    r.covered_bytes = kw.get("covered", rng.choice([0, 16, (256 << 20) + (3 << 20) + 112, rng.randrange(1 << 37)]))
    r.free_bytes = r.covered_bytes + rng.choice([0, 1 << 30, rng.randrange(1 << 34)])
    for e in range(4):
        r.element_ns[e] = kw.get("ns", rng.choice([0, 1, rng.randrange(1, 1 << 32)]))
    for p in range(2):
        P = r.pass_[p]
        P.mismatches = rng.choice([0, 0, 1, rng.randrange(1 << 30)])
        P.granules = rng.choice([0, 1, rng.randrange(40960)])
        for b in rng.sample(range(64), rng.choice([0, 0, 1, 5, 64])):
            P.bit_flips[b] = rng.randrange(1, 1 << 20)
    fill_health(r.before, rng, kw.get("nvml_before", rng.choice([0, 3, 7, 15, rng.randrange(16)])) & 7)
    fill_health(r.after, rng, kw.get("nvml_after", rng.choice([0, 7, 15, rng.randrange(16)])))
    r.health = rng.randrange(16)
    return r


def crafted(cro):
    rng = random.Random(20261015)
    yield cro.ScanReport()                                                              # empty report
    yield make_report(cro, rng, ns=0, covered=0, nvml_before=0, nvml_after=0)
    for st, ce in [(0, 0), (cro.ERR_CHECKSUM, 0), (cro.ERR_CUDA, 214), (cro.ERR_CUDA, 0), (cro.ERR_OOM, 0),
                   (cro.ERR_INVALID_ARG, 0), (cro.ERR_DEADLINE, 0), (cro.ERR_EXEC, 0)]:
        yield make_report(cro, rng, status=st, cuda_error=ce)
    for nb in range(8):                                                                  # every combination of answered reads
        for na in range(16):
            yield make_report(cro, rng, nvml_before=nb, nvml_after=na)
    for _ in range(300):
        yield make_report(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM, cro.ERR_CUDA]), cuda_error=rng.choice([0, 214, 999]))


def test_emitter_equals_the_restatement(cro):
    import scan
    seen = set()
    n = 0
    for r in crafted(cro):
        got = cro.emit_scan_annotations_json(r).encode()
        want = scan.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(scan.annotations(as_dict(r))["cohdi.io/hbm-scan-verdict"].split(":")[0])
        n += 1
    assert n > 400 and seen == {"ok", "corrupt", "cuda-error", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.ScanReport()
    r.status, r.covered_bytes, r.free_bytes, r.seed = cro.ERR_CHECKSUM, 80 << 30, 81 << 30, 0xABC
    r.element_ns[:] = [25_000_000, 25_000_000, 25_000_000, 25_000_000]
    r.pass_[0].mismatches, r.pass_[1].mismatches, r.pass_[0].granules, r.pass_[1].granules = 0, 7, 0, 1
    r.pass_[1].bit_flips[3] = 7
    r.health = cro.SCAN_HEALTH_ECC_CORRECTED_DURING | cro.SCAN_HEALTH_REMAP_PENDING
    r.before.nvml, r.after.nvml = 3, 15
    r.before.ecc_corrected, r.after.ecc_corrected = 5, 12
    r.after.remap_corrected, r.after.remap_uncorrected, r.after.remap_pending = 1, 0, 1
    r.after.histogram[:] = [640, 0, 0, 0, 0]
    p = "cohdi.io/hbm-scan-"
    assert json.loads(cro.emit_scan_annotations_json(r)) == {
        p + "verdict": "corrupt", p + "covered-bytes": str(80 << 30), p + "free-bytes": str(81 << 30),
        p + "seed": "0000000000000abc", p + "mismatches": "0,7", p + "granules": "0,1", p + "gbs": "3435",
        p + "bits": "3", p + "health": "ecc-corrected,remap-pending", p + "ecc-corrected": "7", p + "ecc-uncorrected": "0",
        p + "remapped": "1,0", p + "remap-histogram": "640,0,0,0,0"}


def test_null_arguments_are_refused(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_scan_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_hbm_health(None, ctypes.byref(cro.HbmHealth())) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_hbm_health(b"GPU-x", None) == cro.ERR_INVALID_ARG
    rep, k = cro.ScanReport(), ctypes.c_int(-1)
    words = (cro.FaultWord * 4)()
    assert cro.lib.cro_scan_hbm(None, 0, None, ctypes.byref(rep), words, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_scan_hbm_uuid(None, None, None, ctypes.byref(rep), words, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_scan_hbm_uuid(None, U.encode(), None, ctypes.byref(rep), None, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the DRAM health readers through a stand-in NVML ----------------------------------------------------------------
READER = r"""
import ctypes, importlib, json, os, sys
sys.path.insert(0, sys.argv[1])
cro = importlib.import_module("composable-resource-operator_b200")
out = []
for env, uuid in json.loads(sys.argv[2]):
    os.environ["FAKE_HBM_HEALTH"] = env
    h = cro.read_hbm_health(uuid)
    out.append({f: (list(getattr(h, f)) if f == "histogram" else getattr(h, f)) for f, _ in cro.HbmHealth._fields_})
print(json.dumps(out))
"""


def read_through(tmp_path, cases, no_histogram=False):
    d = tmp_path / ("nvml_nohist" if no_histogram else "nvml")
    d.mkdir()
    lib = d / "libnvidia-ml.so.1"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-Werror", "-o", str(lib), os.path.join(HERE, "fake_nvml_health.c")]
                          + (["-DNO_HISTOGRAM"] if no_histogram else []))
    env = dict(os.environ, LD_LIBRARY_PATH=str(d) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([sys.executable, "-c", READER, ROOT, json.dumps(cases)], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout)


def test_health_readers_pass_nvml_values_through(cro, tmp_path):
    line = "%s 17 2 3 1 1 0 600 30 7 2 1 %d"
    other = "GPU-00000000-0000-0000-0000-000000000002 99 99 99 99 1 1 9 9 9 9 9 0"
    cases = [(line % (U, 0), U), (other + ";" + line % (U, 0), U)] + [(line % (U, m), U) for m in range(1, 16)]
    cases.append((line % (U, 0), "GPU-not-listed"))
    got = read_through(tmp_path, cases)
    full = {"ecc_corrected": 17, "ecc_uncorrected": 2, "remap_corrected": 3, "remap_uncorrected": 1, "remap_pending": 1,
            "remap_failure": 0, "histogram": [600, 30, 7, 2, 1]}
    for (env, uuid), h in zip(cases, got):
        if uuid != U:                                                                   # a device NVML does not know
            assert h == {"nvml": 0, **{k: ([0] * 5 if k == "histogram" else 0) for k in full}}
            continue
        refuse = int(env.split()[-1])
        assert h["nvml"] == 15 & ~refuse, (refuse, h)
        want = dict(full)
        if refuse & 1:
            want["ecc_corrected"] = 0
        if refuse & 2:
            want["ecc_uncorrected"] = 0
        if refuse & 4:
            want.update(remap_corrected=0, remap_uncorrected=0, remap_pending=0, remap_failure=0)
        if refuse & 8:
            want["histogram"] = [0] * 5
        assert {k: h[k] for k in want} == want, (refuse, h)


def test_a_library_without_the_histogram_leaves_its_flag_clear(cro, tmp_path):
    (h,) = read_through(tmp_path, [("%s 1 0 0 0 0 0 5 5 5 5 5 0" % U, U)], no_histogram=True)
    assert h["nvml"] == 7 and h["histogram"] == [0] * 5 and h["ecc_corrected"] == 1


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_without_nvml_nothing_is_answered(cro):
    assert cro.read_hbm_health(U).nvml == 0


# ---- the scan helper's wire format: report, then `recorded` words ----------------------------------------------------
def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


SCAN_HELPER = """
import os, struct, sys
assert sys.argv[1] == "scan-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 12, sys.argv
max_b, reserve, seed, chunk, first, count, and_m, or_m, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(12632)
struct.pack_into("<iiII", r, 0, -6, 0, 0, 1)
struct.pack_into("<QQQQQII", r, 16, seed, 80 << 30, 79 << 30, 0, max_b, 1, 4)
struct.pack_into("<QQ", r, 64, 3, n)
words = b"".join(struct.pack("<QQQII", first + j, 5, 4, 1, 0) for j in range(n))
sys.stdout.buffer.write(bytes(r) + words + b"%s")
sys.exit(1)
"""


def test_scan_helper_report_and_words_come_back(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, SCAN_HELPER % ""))
    rep, words = cro.scan_hbm_uuid(None, U, max_bytes=1 << 30, seed=77, force=(10, 3, 0, 1))
    assert rep.status == cro.ERR_CHECKSUM and rep.seed == 77 and rep.covered_bytes == 1 << 30 and rep.elements_done == 4
    assert rep.recorded == 3 and rep.complete == 1 and rep.helper_ns > 0
    assert [(w.word_index, w.expected, w.actual, w.passes) for w in words] == [(10, 5, 4, 1), (11, 5, 4, 1), (12, 5, 4, 1)]
    rep, words = cro.scan_hbm_uuid(None, U, cap=2)                    # the helper is asked for at most cap words
    assert len(words) == 2 and rep.recorded == 2


def test_scan_helper_failures_are_loud(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, SCAN_HELPER % "x"))       # one byte too many
    with pytest.raises(cro.ProbeError) as e:
        cro.scan_hbm_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "scan helper for %s failed" % U in str(e.value) and "12729 result bytes" in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.scan_hbm_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_scan_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.scan_hbm_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "scan helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    pid = int(marker.read_text())
    with pytest.raises(ProcessLookupError):                            # killed and reaped: no process is left behind
        os.kill(pid, 0)


def test_cli_refuses_a_short_scan_raw(cro):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli, "scan-raw", U, "0"], capture_output=True).returncode == 64


# ---- the kernels the scan reuses are the parent's, instruction for instruction ---------------------------------------
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def golden():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_kernel_sass
    return make_kernel_sass, json.load(open(os.path.join(HERE, "golden", "kernel_sass.json")))


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_kernel_sass_is_unchanged(cro):
    mk, want = golden()
    got = mk.sass_digests(mk.OBJ)
    assert sorted(got) == sorted(want["sass_sha256"])
    assert got == want["sass_sha256"], [k for k in got if got[k] != want["sass_sha256"][k]]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_kernel_ptxas_resources_are_unchanged(cro):
    mk, want = golden()
    assert mk.ptxas_lines() == want["ptxas"]
