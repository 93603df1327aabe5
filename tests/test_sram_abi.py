"""The SRAM probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the annotation emitter
against oracle/sram.py, the SRAM health readers through a stand-in NVML, the SRAM helper's wire format and deadline,
and the new kernels as ptxas and cuobjdump see them (no spills; every march element one shared load and / or store)."""
import collections
import ctypes
import json
import os
import random
import re
import shutil
import stat
import struct
import subprocess
import sys
import tempfile
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
U = "GPU-5ca90000-0000-0000-0000-000000000002"

FIELDS = {
    "cro_sram_opts": ("SramOpts", ["legs", "iterations", "cluster", "max_rounds", "deadline_ms", "test_inject_leg",
                                   "test_inject_sm", "test_inject_element", "test_inject_iteration", "test_inject_word",
                                   "test_inject_mask"]),
    "cro_sram_health": ("SramHealth", ["nvml", "threshold_exceeded", "ecc_corrected", "ecc_uncorrected"]),
    "cro_sram_pair": ("SramPair", [("from", "from_"), "owner", "direction"]),
    "cro_sram_leg": ("SramLeg", ["iterations", "rounds", "bytes", "ns", "timer_ns", "sms_covered", "complete", "mismatches",
                                 "fold_mismatches", "recorded", "failed_sms", "unpublished", "ctas", "cluster", "fold_xor",
                                 "fold_sum", "fold_wsum", "expect_xor", "expect_sum", "expect_wsum"]),
    "cro_sram_result": ("SramResult", ["status", "verdict", "seed", "call", "sm_count", "legs", "nsmid", "cuda_error",
                                       "bytes_per_sm", "health", "bad_sms", "bad_sm", "bad_pairs", "sms_listed", "bad_pair",
                                       "recorded", "wall_ns", "helper_ns", "before", "after", "leg"]),
    "cro_sram_sm_leg": ("SramSmLeg", ["mismatches", "fold_mismatches", "ns", "cycles", "ctas", "mark"]),
    "cro_sram_sm": ("SramSm", ["smid", "reserved", "leg"]),
    "cro_sram_fault": ("SramFault", ["leg", "element", "iteration", "smid", "peer_smid", "direction", "word", "reserved",
                                     "expected", "actual"]),
}
CONSTANTS = ["CRO_SRAM_SMEM", "CRO_SRAM_DSMEM", "CRO_SRAM_LEGS", "CRO_SRAM_LEG_SMEM", "CRO_SRAM_LEG_DSMEM",
             "CRO_SRAM_ALL_LEGS", "CRO_SRAM_ELEMENTS", "CRO_SRAM_RECORDS", "CRO_SRAM_MAX_SMS", "CRO_SRAM_MAX_ITERATIONS",
             "CRO_SRAM_MAX_ROUNDS", "CRO_SRAM_MAX_PAIRS", "CRO_SRAM_NONE", "CRO_SRAM_SM", "CRO_SRAM_LINK", "CRO_SRAM_ALL",
             "CRO_SRAM_PERSISTENT", "CRO_SRAM_INTERMITTENT", "CRO_SRAM_DIR_LOCAL", "CRO_SRAM_DIR_READ", "CRO_SRAM_DIR_WRITE",
             "CRO_SRAM_HEALTH_CORRECTED_DURING", "CRO_SRAM_HEALTH_UNCORRECTED_DURING", "CRO_SRAM_HEALTH_THRESHOLD_EXCEEDED",
             "CRO_SRAM_NVML_ECC_CORRECTED", "CRO_SRAM_NVML_ECC_UNCORRECTED", "CRO_SRAM_NVML_STATUS"]


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


# ---- the emitter against oracle/sram.py -----------------------------------------------------------------------------
def health_dict(h):
    return {"nvml": h.nvml, "threshold_exceeded": h.threshold_exceeded, "ecc_corrected": h.ecc_corrected,
            "ecc_uncorrected": h.ecc_uncorrected}


def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sm_count": r.sm_count, "legs": r.legs,
            "bytes_per_sm": r.bytes_per_sm, "health": r.health, "sms_covered": [L.sms_covered for L in r.leg],
            "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm), "bad_pairs": r.bad_pairs,
            "bad_pair": [(p.from_, p.owner, p.direction) for p in r.bad_pair],
            "before": health_dict(r.before), "after": health_dict(r.after)}


def fill_health(h, rng, nvml):
    h.nvml = nvml
    h.ecc_corrected = rng.choice([0, 1, rng.randrange(1 << 40)]) if nvml & 1 else 0
    h.ecc_uncorrected = rng.choice([0, 0, 3]) if nvml & 2 else 0
    h.threshold_exceeded = rng.choice([0, 0, 1]) if nvml & 4 else 0


def make_result(cro, rng, **kw):
    r = cro.SramResult()
    r.status = kw.get("status", 0)
    r.verdict = kw.get("verdict", rng.randrange(4))
    r.cuda_error = kw.get("cuda_error", 0)
    r.sm_count = rng.choice([132, 114, 0])
    r.legs = kw.get("legs", rng.choice([1, 2, 3, 3]))
    r.bytes_per_sm = rng.choice([232192, 0, rng.randrange(1 << 20)])
    for L in r.leg:
        L.sms_covered = rng.choice([r.sm_count, 120, 0, rng.randrange(256)])
    r.bad_sms = kw.get("bad_sms", rng.choice([0, 0, 1, 2, 16, 17, 132]))
    for j in range(16):
        r.bad_sm[j] = rng.randrange(256)
    r.bad_pairs = kw.get("bad_pairs", rng.choice([0, 0, 1, 3, 8, 9, 40]))
    for j in range(8):
        r.bad_pair[j].from_, r.bad_pair[j].owner, r.bad_pair[j].direction = rng.randrange(256), rng.randrange(256), rng.choice([1, 2])
    fill_health(r.before, rng, kw.get("nvml_before", rng.randrange(4)))
    fill_health(r.after, rng, kw.get("nvml_after", rng.randrange(8)))
    r.health = kw.get("health", rng.randrange(8))
    return r


def crafted(cro):
    rng = random.Random(20261015)
    yield cro.SramResult()                                                              # empty result
    for st, ce in [(0, 0), (cro.ERR_CHECKSUM, 0), (cro.ERR_CUDA, 214), (cro.ERR_CUDA, 0), (cro.ERR_OOM, 0),
                   (cro.ERR_INVALID_ARG, 0), (cro.ERR_DEADLINE, 0), (cro.ERR_UNSUPPORTED, 0), (cro.ERR_EXEC, 0)]:
        for v in range(4):
            yield make_result(cro, rng, status=st, cuda_error=ce, verdict=v)
    for nb in range(4):                                                                  # every combination of answered reads
        for na in range(8):
            for h in (0, 7):
                yield make_result(cro, rng, nvml_before=nb, nvml_after=na, health=h)
    for legs in (1, 2, 3):
        for cap in (0, 1, 8, 9, 16, 17):
            yield make_result(cro, rng, legs=legs, bad_sms=cap, bad_pairs=cap, status=cro.ERR_CHECKSUM)
    for _ in range(300):
        yield make_result(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM, cro.ERR_CHECKSUM, cro.ERR_CUDA]),
                          cuda_error=rng.choice([0, 214, 999]))


def test_emitter_equals_the_restatement(cro):
    import sram
    seen = set()
    n = 0
    for r in crafted(cro):
        got = cro.emit_sram_annotations_json(r).encode()
        want = sram.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(sram.annotations(as_dict(r))["cohdi.io/probe-sram-verdict"].split(":")[0])
        n += 1
    assert n > 400 and seen == {"ok", "sm", "link", "all", "cuda-error", "error"}


def test_emitter_spells_the_keys(cro):
    r = cro.SramResult()
    r.status, r.verdict, r.sm_count, r.legs, r.bytes_per_sm = cro.ERR_CHECKSUM, cro.SRAM_LINK, 132, 3, 232192
    r.leg[0].sms_covered, r.leg[1].sms_covered = 132, 120
    r.bad_pairs = 2
    r.bad_pair[0].from_, r.bad_pair[0].owner, r.bad_pair[0].direction = 4, 5, cro.SRAM_DIR_READ
    r.bad_pair[1].from_, r.bad_pair[1].owner, r.bad_pair[1].direction = 9, 8, cro.SRAM_DIR_WRITE
    r.health = cro.SRAM_HEALTH_CORRECTED_DURING | cro.SRAM_HEALTH_THRESHOLD_EXCEEDED
    r.before.nvml, r.after.nvml = 3, 7
    r.before.ecc_corrected, r.after.ecc_corrected, r.after.threshold_exceeded = 5, 12, 1
    p = "cohdi.io/probe-sram-"
    assert json.loads(cro.emit_sram_annotations_json(r)) == {
        p + "verdict": "link", p + "sms": "120/132", p + "bad-pairs": "4-5:r,9-8:w", p + "bytes-per-sm": "232192",
        p + "health": "corrected,threshold-exceeded", p + "ecc-corrected": "7", p + "ecc-uncorrected": "0"}


def test_health_bits_equal_the_restatement(cro):
    import sram
    rng = random.Random(7)
    for _ in range(200):
        r = make_result(cro, rng)
        b, a = health_dict(r.before), health_dict(r.after)
        want = sram.health_bits(b, a)
        assert want == (((b["nvml"] & a["nvml"] & 1) and a["ecc_corrected"] > b["ecc_corrected"]) * 1 |
                        ((b["nvml"] & a["nvml"] & 2) and a["ecc_uncorrected"] > b["ecc_uncorrected"]) * 2 |
                        ((a["nvml"] & 4) and a["threshold_exceeded"]) * 4)


def test_null_arguments_are_refused(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_sram_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_sram_health(None, ctypes.byref(cro.SramHealth())) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_read_sram_health(b"GPU-x", None) == cro.ERR_INVALID_ARG
    r, k, ks = cro.SramResult(), ctypes.c_int(-1), ctypes.c_int(-1)
    sms, faults = (cro.SramSm * 4)(), (cro.SramFault * 4)()
    assert cro.lib.cro_probe_sram(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4, ctypes.byref(k)) == \
        cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_sram_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                       ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_sram_uuid(None, U.encode(), None, ctypes.byref(r), sms, 4, ctypes.byref(ks), None, 4,
                                       ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_sram_uuid(None, U.encode(), None, ctypes.byref(r), None, 4, ctypes.byref(ks), faults, 4,
                                       ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the SRAM health readers through a stand-in NVML ----------------------------------------------------------------
READER = r"""
import ctypes, importlib, json, os, sys
sys.path.insert(0, sys.argv[1])
cro = importlib.import_module("composable-resource-operator_b200")
out = []
for env, uuid in json.loads(sys.argv[2]):
    os.environ["FAKE_SRAM_HEALTH"] = env
    h = cro.read_sram_health(uuid)
    out.append({f: getattr(h, f) for f, _ in cro.SramHealth._fields_})
print(json.dumps(out))
"""


def read_through(tmp_path, cases, no_status=False):
    d = tmp_path / ("nvml_nostatus" if no_status else "nvml")
    d.mkdir()
    lib = d / "libnvidia-ml.so.1"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-Werror", "-o", str(lib), os.path.join(HERE, "fake_nvml_sram.c")]
                          + (["-DNO_SRAM_STATUS"] if no_status else []))
    env = dict(os.environ, LD_LIBRARY_PATH=str(d) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([sys.executable, "-c", READER, ROOT, json.dumps(cases)], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout)


def test_health_readers_pass_nvml_values_through(cro, tmp_path):
    line = "%s 17 2 1 %d"
    other = "GPU-00000000-0000-0000-0000-000000000009 99 99 0 0"
    cases = [(line % (U, 0), U), (other + ";" + line % (U, 0), U)] + [(line % (U, m), U) for m in range(1, 8)]
    cases.append((line % (U, 0), "GPU-not-listed"))
    got = read_through(tmp_path, cases)
    for (env, uuid), h in zip(cases, got):
        if uuid != U:                                                                   # a device NVML does not know
            assert h == {"nvml": 0, "threshold_exceeded": 0, "ecc_corrected": 0, "ecc_uncorrected": 0}
            continue
        refuse = int(env.split()[-1])
        assert h["nvml"] == 7 & ~refuse, (refuse, h)
        assert h == {"nvml": 7 & ~refuse, "ecc_corrected": 0 if refuse & 1 else 17, "ecc_uncorrected": 0 if refuse & 2 else 2,
                     "threshold_exceeded": 0 if refuse & 4 else 1}, (refuse, h)


def test_a_library_without_the_sram_status_leaves_its_flag_clear(cro, tmp_path):
    (h,) = read_through(tmp_path, [("%s 1 0 1 0" % U, U)], no_status=True)
    assert h == {"nvml": 3, "threshold_exceeded": 0, "ecc_corrected": 1, "ecc_uncorrected": 0}


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_without_nvml_nothing_is_answered(cro):
    assert cro.read_sram_health(U).nvml == 0


# ---- the SRAM helper's wire format: result, CRO_SRAM_MAX_SMS per-SM entries, then `recorded` faults ------------------
def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


SRAM_HELPER = """
import os, struct, sys
assert sys.argv[1] == "sram-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 14, sys.argv
legs, iters, cluster, rounds, leg, sm, element, iteration, word, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(568)
struct.pack_into("<iIQQII", r, 0, -6, 1, 1234, 0, 132, legs)
struct.pack_into("<Q", r, 40, 232192)
struct.pack_into("<II", r, 52, 1, 0)
struct.pack_into("<H", r, 56, sm)
struct.pack_into("<II", r, 88, 0, 2)
struct.pack_into("<Q", r, 160, n)
sms = bytearray(256 * 168)
struct.pack_into("<I", sms, 0, 3)
struct.pack_into("<I", sms, 168, sm)
faults = b"".join(struct.pack("<IIIIIIIIQQ", 0, element, iteration, sm, sm, 0, word + j, 0, 5, 5 ^ mask) for j in range(n))
sys.stdout.buffer.write(bytes(r) + bytes(sms) + faults + b"%s")
sys.exit(1)
"""


def test_sram_helper_result_sms_and_faults_come_back(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, SRAM_HELPER % ""))
    r, sms, faults = cro.probe_sram_uuid(None, U, iterations=3, inject=(0, 9, 4, 2, 100, 1 << 37))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.SRAM_SM and r.seed == 1234 and r.bytes_per_sm == 232192
    assert list(r.bad_sm[:r.bad_sms]) == [9] and r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2
    assert [s.smid for s in sms] == [3, 9]
    assert [(f.element, f.iteration, f.smid, f.word, f.expected, f.actual) for f in faults] == \
        [(4, 2, 9, 100 + j, 5, 5 ^ (1 << 37)) for j in range(3)]
    r, sms, faults = cro.probe_sram_uuid(None, U, cap=2)                # the helper is asked for at most cap faults
    assert len(faults) == 2 and r.recorded == 2


def test_sram_helper_failures_are_loud(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, SRAM_HELPER % "x"))       # one byte too many
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sram_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC and "SRAM helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sram_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_sram_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_sram_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "SRAM helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    pid = int(marker.read_text())
    with pytest.raises(ProcessLookupError):                            # killed and reaped: no process is left behind
        os.kill(pid, 0)


def test_cli_refuses_a_short_sram_raw(cro):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli, "sram-raw", U, "0"], capture_output=True).returncode == 64


# ---- the new kernels as the compiler built them ---------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_sram_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "sram_kernels.cu"), "-o",
                                             os.path.join(d, "s.o")], capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\S+)'", text)
    assert len(kernels) == 2 and all("sram_" in k for k in kernels), kernels
    assert text.count("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") == 2, text


def sass_counts(obj):
    """{kernel: Counter of SASS memory opcodes} of the object's two SRAM kernels."""
    out, name = {}, None
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", obj], text=True).splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            name = "dsmem" if "sram_dsmem_kernel" in m.group(1) else "smem" if "sram_smem_kernel" in m.group(1) else None
            if name:
                out[name] = collections.Counter()
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if name and m and m.group(1).split(".")[0] in ("LDS", "STS", "LD", "ST", "ATOMS"):
            out[name][m.group(1).split(".")[0] + "." + ".".join(p for p in m.group(1).split(".")[1:] if p in ("64", "128"))] += 1
    return out


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_every_march_element_is_one_64_bit_shared_access(cro):
    c = sass_counts(os.path.join(CSRC, "build", "sram_kernels.cu.o"))
    # Besides the march, each kernel clears its bookkeeping with one STS.64 and reads it back with LDS.128, and every
    # 64-bit shared atomic is a compare-and-swap loop that reads its word once with an LDS.64.
    s, d = c["smem"], c["dsmem"]
    assert s["STS.64"] == 5 + 1, s                                   # M0 .. M4 write
    assert s["LDS.64"] == 5 + s["ATOMS.64"], s                       # M1 .. M5 read
    assert s["LD.64"] == s["ST.64"] == 0, s                          # nothing over the network
    assert d["STS.64"] == 1 + 1, d                                   # D0 writes locally
    assert d["LDS.64"] == 1 + d["ATOMS.64"], d                       # D3 reads locally
    assert d["LD.64"] == 1 and d["ST.64"] == 1, d                    # D1 reads, D2 writes over the network
