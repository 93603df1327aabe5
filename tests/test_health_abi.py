"""The health check without a GPU: the ctypes mirrors against the header as gcc lays it out, the stop and status rules
and the annotation emitter against oracle/health.py, and the helper form through a stand-in helper (CRO_HELPER_PATH):
what goes on its argv, how its frame is read back, and what is refused before any helper starts."""
import ctypes
import json
import os
import random
import struct
import subprocess
import sys
import time

import pytest

import test_compute_abi
import test_hbm_scan_abi
import test_host_link_abi
import test_l2_abi
import test_precision_abi
import test_sram_abi
from test_helper_probes_abi import fake_helper, last_thread_error, seen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = "GPU-5ca90000-0000-0000-0000-000000000003"
OK, ERR_CUDA, ERR_OOM, ERR_CHECKSUM, ERR_INVALID_ARG = 0, -4, -5, -6, -1

FIELDS = {
    "cro_health_opts": ("HealthOpts", ["checks", "reserved0", "compute", "precision", "sram", "l2", "link", "scan"]),
    "cro_health_result": ("HealthResult", ["status", "checks", "ran", "failed", "errored", "not_run", "incomplete", "reserved0",
                                           "check_status", "check_ns", "seed_base", "helper_ns", "compute", "precision", "sram",
                                           "l2", "link", "scan"]),
    "cro_health_records": ("HealthRecords", [f for n in ("compute_sms", "compute_faults", "precision_sms", "precision_faults",
                                                         "sram_sms", "sram_faults", "l2_sms", "l2_faults", "link_faults",
                                                         "scan_words") for f in (n, n + "_cap", n + "_n")]),
}
CONSTANTS = ["CRO_HEALTH_COMPUTE", "CRO_HEALTH_PRECISION", "CRO_HEALTH_SRAM", "CRO_HEALTH_L2", "CRO_HEALTH_LINK",
             "CRO_HEALTH_SCAN", "CRO_HEALTH_ALL", "CRO_HEALTH_CHECKS"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    for k in CONSTANTS:
        src.append('printf("const %s %%lld\\n", (long long)(%s));' % (k, k))
    src.append("return 0; }")
    (tmp_path / "layout.c").write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I" + os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(exe)])
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


def test_the_sub_structs_are_each_checks_own(cro):
    opts, res = dict(cro.HealthOpts._fields_), dict(cro.HealthResult._fields_)
    assert [opts[n] for n in cro.HEALTH_NAMES] == [cro.ComputeOpts, cro.PrecisionOpts, cro.SramOpts, cro.L2Opts, cro.LinkOpts,
                                                   cro.ScanOpts]
    assert [res[n] for n in cro.HEALTH_NAMES] == [cro.ComputeResult, cro.PrecisionResult, cro.SramResult, cro.L2Result,
                                                  cro.LinkResult, cro.ScanReport]


# ---- the stop and status rules against oracle/health.py ---------------------------------------------------------------
def summary(r):
    return {"status": r.status, "checks": r.checks, "ran": r.ran, "failed": r.failed, "errored": r.errored,
            "not_run": r.not_run, "check_status": list(r.check_status)}


def agree(cro, checks, statuses):
    import health
    r, nxt = cro.selftest_health_classify(checks, statuses)
    want, want_next = health.classify(checks, statuses)
    assert (summary(r), nxt) == (want, want_next), (checks, statuses)
    return r, nxt


def test_a_cuda_error_stops_every_later_check(cro):
    for k in range(6):
        r, nxt = agree(cro, 0, [OK] * k + [ERR_CUDA])
        assert nxt == 0 and r.status == ERR_CUDA and r.ran == (1 << (k + 1)) - 1
        assert r.not_run == cro.HEALTH_ALL & ~((1 << (k + 1)) - 1) and r.errored == 1 << k
        with pytest.raises(cro.ProbeError):                 # nothing may run after it
            cro.selftest_health_classify(0, [OK] * k + [ERR_CUDA, OK])


def test_checksum_outranks_an_earlier_error_and_only_cuda_stops(cro):
    r, nxt = agree(cro, 0, [OK, ERR_CHECKSUM, ERR_CUDA])
    assert r.status == ERR_CHECKSUM and r.failed == cro.HEALTH_PRECISION and nxt == 0
    assert r.not_run == cro.HEALTH_L2 | cro.HEALTH_LINK | cro.HEALTH_SCAN
    r, nxt = agree(cro, 0, [ERR_OOM, ERR_CHECKSUM])
    assert r.status == ERR_CHECKSUM and r.errored == cro.HEALTH_COMPUTE and nxt == cro.HEALTH_SRAM
    r, nxt = agree(cro, 0, [OK, ERR_OOM, OK, -9, OK, OK])
    assert r.status == ERR_OOM and nxt == 0 and r.ran == cro.HEALTH_ALL and r.not_run == 0


def test_an_empty_sequence_and_the_default_selection(cro):
    r, nxt = agree(cro, 0, [])
    assert r.status == OK and r.checks == cro.HEALTH_ALL and r.ran == 0 and nxt == cro.HEALTH_COMPUTE
    r, nxt = agree(cro, cro.HEALTH_SCAN | cro.HEALTH_SRAM, [])
    assert nxt == cro.HEALTH_SRAM
    r, nxt = agree(cro, cro.HEALTH_SCAN | cro.HEALTH_SRAM, [OK])
    assert nxt == cro.HEALTH_SCAN and r.ran == cro.HEALTH_SRAM
    for bad in (0x40, 0x80000000):
        with pytest.raises(cro.ProbeError):
            cro.selftest_health_classify(bad, [])


def test_a_seeded_sweep_of_subsets_and_status_sequences(cro):
    import health
    rng = random.Random(20261017)
    pool = [OK, OK, OK, ERR_CHECKSUM, ERR_CUDA, ERR_OOM, ERR_INVALID_ARG, -9, -10, -12]
    n = 0
    while n < 2500:
        checks = rng.randrange(64)
        statuses, cut = [], rng.randrange(7)
        for _ in range(cut):
            statuses.append(rng.choice(pool))
        try:
            want = health.classify(checks, statuses)
        except ValueError:
            with pytest.raises(cro.ProbeError):
                cro.selftest_health_classify(checks, statuses)
            continue
        r, nxt = cro.selftest_health_classify(checks, statuses)
        assert (summary(r), nxt) == want, (checks, statuses)
        n += 1


# ---- the emitter against oracle/health.py ------------------------------------------------------------------------------
SUBS = [(test_compute_abi, "make_result"), (test_precision_abi, "make_result"), (test_sram_abi, "make_result"),
        (test_l2_abi, "make_result"), (test_host_link_abi, "make_result"), (test_hbm_scan_abi, "make_report")]


def as_dict(r, cro):
    d = {"status": r.status, "ran": r.ran, "failed": r.failed, "errored": r.errored, "not_run": r.not_run,
         "incomplete": r.incomplete, "check_status": list(r.check_status), "check_ns": list(r.check_ns), "helper_ns": r.helper_ns}
    for c, (mod, _) in enumerate(SUBS):
        d[cro.HEALTH_NAMES[c]] = mod.as_dict(getattr(r, cro.HEALTH_NAMES[c]))
    return d


def crafted(cro):
    rng = random.Random(20261018)
    pool = [OK, OK, ERR_CHECKSUM, ERR_CUDA, ERR_OOM, -10]
    for k in range(400):
        checks = rng.randrange(1, 64)
        statuses = []
        for _ in range(bin(checks).count("1")):
            statuses.append(rng.choice(pool))
            if statuses[-1] == ERR_CUDA:
                break
        r, _ = cro.selftest_health_classify(checks, statuses)
        for c, (mod, make) in enumerate(SUBS):
            if r.ran >> c & 1:
                st = r.check_status[c]
                kw = {"status": st}
                if mod is not test_compute_abi and mod is not test_precision_abi and mod is not test_host_link_abi:
                    kw["cuda_error"] = rng.choice([0, 214, 700])
                setattr(r, cro.HEALTH_NAMES[c], getattr(mod, make)(cro, rng, **kw))
        r.incomplete = rng.randrange(16) & r.ran
        for c in range(6):
            r.check_ns[c] = rng.randrange(1 << 40) if r.ran >> c & 1 else 0
        r.helper_ns = rng.choice([0, rng.randrange(1 << 40)])
        yield r


def test_emitter_equals_the_restatement(cro):
    import health
    verdicts, keys = set(), set()
    for r in crafted(cro):
        got = cro.emit_health_annotations_json(r).encode()
        want = health.annotations_json(as_dict(r, cro))
        assert got == want, (got, want)
        m = json.loads(got)
        assert list(m) == sorted(m)
        verdicts.add(m["cohdi.io/probe-health-verdict"].split(":")[0])
        keys |= {k for k in m if k.startswith("cohdi.io/probe-health-")}
        for field, key in (("failed", "failed"), ("errored", "errors"), ("not_run", "not-run"), ("incomplete", "incomplete")):
            assert (("cohdi.io/probe-health-" + key) in m) == bool(getattr(r, field))
    assert verdicts == {"ok", "fail", "cuda-error", "error"}
    assert keys == {"cohdi.io/probe-health-" + k for k in ("verdict", "failed", "errors", "not-run", "incomplete", "ms")}


def test_emitter_spells_the_keys(cro):
    r, _ = cro.selftest_health_classify(cro.HEALTH_COMPUTE | cro.HEALTH_SCAN, [ERR_CHECKSUM, ERR_CUDA])
    r.scan.status, r.scan.cuda_error, r.compute.status, r.compute.verdict = ERR_CUDA, 214, ERR_CHECKSUM, cro.COMPUTE_SM
    r.check_ns[0], r.check_ns[5], r.incomplete = 7 * 10 ** 6, 5 * 10 ** 6 + 1, cro.HEALTH_COMPUTE
    m = json.loads(cro.emit_health_annotations_json(r))
    p = "cohdi.io/probe-health-"
    assert {k: v for k, v in m.items() if k.startswith(p)} == {p + "verdict": "fail", p + "failed": "compute",
                                                               p + "errors": "scan", p + "incomplete": "compute", p + "ms": "12"}
    assert m["cohdi.io/probe-compute-verdict"] == "sm" and m["cohdi.io/hbm-scan-verdict"] == "cuda-error:214"
    r.status, r.failed = ERR_CUDA, 0
    assert json.loads(cro.emit_health_annotations_json(r))[p + "verdict"] == "cuda-error:214"
    assert cro.lib.cro_emit_health_annotations_json(None, None, 0, None) == ERR_INVALID_ARG


# ---- the helper form through a stand-in ---------------------------------------------------------------------------------
# (result, sms entry, record) sizes of each check's part, its per-SM block (0: none) and its count words, in run order
PARTS = [(600, 208, 24, 256, 2), (808, 288, 32, 256, 2), (568, 168, 48, 256, 0), (616, 128, 56, 256, 2), (984, 0, 40, 0, 1),
         (12632, 0, 32, 0, 0)]
HELD = [120, 720, 1528, 2096, 2712, 3696]
CAP_AT = [15, 26, 37, 48, 55, 64]                    # sys.argv index of each check's cap

# A stand-in health-raw: it leaves its argv in argv.json and writes a frame from cfg: the summary fields given, each ran
# check's result of random bytes (status, and the counts its part is read by, set), two per-SM entries and min(cap, n)
# records.  `extra` bytes are appended, `cut` dropped, `over` adds one record past a cap, `ran_extra` adds ran bits.
FAKE = r"""
import json, os, random, struct, sys
d = os.path.dirname(os.path.abspath(sys.argv[0]))
open(os.path.join(d, "argv.json"), "w").write(json.dumps({"argv": sys.argv[1:], "cvd": os.environ.get("CUDA_VISIBLE_DEVICES")}))
cfg = json.loads(%r)
PARTS, HELD, CAP_AT = %r, %r, %r
rng = random.Random(cfg["seed"])
blob = lambda k: bytes(rng.randrange(256) for _ in range(k))
assert sys.argv[1] == "health-raw" and len(sys.argv) == 65, len(sys.argv)
h = bytearray(blob(16328))
ran = cfg["ran"] | cfg.get("ran_extra", 0)
struct.pack_into("<i6I", h, 0, cfg["status"], int(sys.argv[4]), ran, cfg["failed"], cfg["errored"], cfg["not_run"], 0)
struct.pack_into("<6i", h, 32, *cfg["check_status"])
struct.pack_into("<Q", h, 104, int(sys.argv[3]))
parts = b""
for c in range(6):
    if not ran >> c & 1:
        continue
    res, sm, rec, max_sms, counts = PARTS[c]
    n = min(int(sys.argv[CAP_AT[c]]), cfg["n"]) + (1 if cfg.get("over") == c else 0)
    r = bytearray(h[HELD[c]:HELD[c] + res])
    struct.pack_into("<i", r, 0, cfg["check_status"][c])
    if c == 2:
        struct.pack_into("<I", r, 92, 2); struct.pack_into("<Q", r, 160, n)
    if c == 3:
        struct.pack_into("<Q", r, 128, n); struct.pack_into("<I", r, 140, 2)
    if c == 5:
        struct.pack_into("<I", r, 12, 1); struct.pack_into("<Q", r, 72, n)
    h[HELD[c]:HELD[c] + res] = r
    part = bytes(r) + (struct.pack("<QQ", 2, n) if counts == 2 else struct.pack("<Q", n) if counts == 1 else b"")
    part += blob(2 * sm) + bytes((max_sms - 2) * sm) if max_sms else b""
    parts += part + blob(rec * n)
out = bytes(h) + parts + cfg.get("extra", "").encode()
out = out[:len(out) - cfg.get("cut", 0)]
open(os.path.join(d, "out.bin"), "wb").write(out)
sys.stdout.buffer.write(out)
sys.exit(0 if cfg["status"] == 0 else 1)
"""


def fake(cro, tmp_path, monkeypatch, checks=0, statuses=None, seed=1, n=3, **extra):
    import health
    s, _ = health.classify(checks, statuses if statuses is not None else [OK] * bin(checks or 63).count("1"))
    cfg = dict(s, seed=seed, n=n, **extra)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, FAKE % (json.dumps(cfg), PARTS, HELD, CAP_AT)))
    return s


def written(tmp_path):
    with open(os.path.join(str(tmp_path), "out.bin"), "rb") as f:
        return f.read()


def test_defaults_reach_argv_as_zeroes(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch)
    r, _, ns = cro.check_health_uuid(None, U)
    s = seen(tmp_path)
    assert s["cvd"] == U and r.status == OK and ns > 0 and r.helper_ns == ns
    argv = s["argv"]
    assert argv[:2] == ["health-raw", U] and int(argv[2]) & 0xFF == 0 and argv[3] == "63"
    want = ["0"] * 10 + ["256"] + ["0"] * 10 + ["256"] + ["0"] * 10 + ["256"] + ["0"] * 10 + ["256"] + ["0"] * 6 + ["256"] + \
        ["0"] * 8 + ["256"]
    assert argv[4:] == want


def test_every_option_of_every_check_reaches_argv(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch)
    MiB = 1 << 20
    cro.check_health_uuid(None, U,
                          compute=dict(iterations=9, alu_iterations=5, legs=0b10110, max_rounds=11, inject=(2, 131, 8, -1, 255, 1 << 30)),
                          precision=dict(iterations=7, alu_iterations=3, legs=0x41, max_rounds=12, inject=(6, 5, 2, 127, -1, 1 << 9)),
                          sram=dict(legs=2, iterations=13, cluster=4, max_rounds=14, inject=(1, 77, 2, 12, -1, 1 << 50)),
                          l2=dict(bytes=2 * MiB, iterations=15, a1_counters=99, a2_counters=98, inject=(0, -1, 3, 14, 4097, 1 << 60)),
                          link=dict(bytes=3 * MiB + 112, hops=4097, ctas=300, inject=(3, 12345, 1 << 40)),
                          scan=dict(max_bytes=5 * MiB, reserve_bytes=6 * MiB, seed=0xABC, chunk_bytes=1 << 20, force=(1, 2, 3, 4)),
                          caps={"compute_faults": 1, "precision_faults": 2, "sram_faults": 3, "l2_faults": 4, "link_faults": 5,
                                "scan_words": 6})
    argv = seen(tmp_path)["argv"]
    assert argv[4:] == [str(v) for v in (9, 5, 0b10110, 11, 2, 131, 8, -1, 255, 1 << 30, 1,
                                          7, 3, 0x41, 12, 6, 5, 2, 127, -1, 1 << 9, 2,
                                          2, 13, 4, 14, 1, 77, 2, 12, -1, 1 << 50, 3,
                                          2 * MiB, 15, 99, 98, 0, -1, 3, 14, 4097, 1 << 60, 4,
                                          3 * MiB + 112, 4097, 300, 3, 12345, 1 << 40, 5,
                                          5 * MiB, 6 * MiB, 0xABC, 1 << 20, 1, 2, 3, 4, 6)]


def test_each_call_passes_a_new_seed_base(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch)
    bases = []
    for _ in range(4):
        r, _, _ = cro.check_health_uuid(None, U)
        bases.append(int(seen(tmp_path)["argv"][2]))
        assert r.seed_base == bases[-1]
    assert len(set(bases)) == 4 and all(b and b & 0xFF == 0 for b in bases)


def test_the_frame_comes_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch, statuses=[OK, ERR_CHECKSUM, OK, ERR_OOM, OK, ERR_CUDA], seed=7)
    caps = {"compute_faults": 2, "precision_faults": 3, "sram_faults": 1, "l2_faults": 3, "link_faults": 0, "scan_words": 2}
    r, rec, _ = cro.check_health_uuid(None, U, caps=caps)
    out = written(tmp_path)
    assert r.status == ERR_CHECKSUM and r.ran == cro.HEALTH_ALL and r.failed == cro.HEALTH_PRECISION
    assert r.errored == cro.HEALTH_L2 | cro.HEALTH_SCAN and r.check_status[5] == ERR_CUDA
    at = 16328
    for c, name in enumerate(cro.HEALTH_NAMES):
        res, sm, size, max_sms, counts = PARTS[c]
        sub = bytes(getattr(r, name))
        assert sub == out[HELD[c]:HELD[c] + res] == out[at:at + res], name
        n = min(caps[[k for k in caps if k.startswith(name)][0]], 3)
        head = at + res + 8 * counts
        if max_sms:
            assert b"".join(bytes(x) for x in rec[name + "_sms"]) == out[head:head + 2 * sm], name
            head += max_sms * sm
        lst = rec[name + ("_words" if name == "scan" else "_faults")]
        assert len(lst) == n and b"".join(bytes(x) for x in lst) == out[head:head + n * size], name
        at = head + n * size
    assert at == len(out)


def test_a_subset_reads_only_its_checks(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch, checks=cro.HEALTH_SRAM | cro.HEALTH_LINK)
    r, rec, _ = cro.check_health_uuid(None, U, checks=cro.HEALTH_SRAM | cro.HEALTH_LINK)
    assert seen(tmp_path)["argv"][3] == str(cro.HEALTH_SRAM | cro.HEALTH_LINK)
    assert r.ran == cro.HEALTH_SRAM | cro.HEALTH_LINK and len(rec["sram_faults"]) == 3 and len(rec["link_faults"]) == 3
    assert rec["compute_faults"] == [] and bytes(r.compute) == bytes(cro.ComputeResult())


def test_a_cuda_error_result_is_returned(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch, statuses=[OK, OK, ERR_CUDA])
    r, rec, _ = cro.check_health_uuid(None, U)
    assert r.status == ERR_CUDA and r.not_run == cro.HEALTH_L2 | cro.HEALTH_LINK | cro.HEALTH_SCAN
    assert r.sram.status == ERR_CUDA and len(rec["sram_faults"]) == 3 and rec["scan_words"] == []


@pytest.mark.parametrize("how", [dict(cut=1), dict(extra="x"), dict(over=0), dict(over=4), dict(over=5),
                                 dict(ran_extra=0x40)], ids=["short", "long", "compute-over-cap", "link-over-cap",
                                                             "scan-over-cap", "ran-outside-checks"])
def test_malformed_frames_are_loud(cro, tmp_path, monkeypatch, how):
    fake(cro, tmp_path, monkeypatch, **how)
    caps = {name: 2 for name, _ in cro.HEALTH_LISTS if not name.endswith("_sms")} if "over" in how else {}
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(None, U, caps=caps)
    assert e.value.code == cro.ERR_EXEC and "health helper for %s failed" % U in str(e.value)


def test_ran_outside_the_selection_is_loud(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch, checks=cro.HEALTH_COMPUTE, ran_extra=cro.HEALTH_SCAN)
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(None, U, checks=cro.HEALTH_COMPUTE)
    assert e.value.code == cro.ERR_EXEC


def test_exit_3_is_no_device_and_a_wedged_helper_is_killed(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "health helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    with pytest.raises(ProcessLookupError):
        os.kill(int(marker.read_text()), 0)


REFUSED = [dict(checks=0x40), dict(sram=dict(deadline_ms=5)), dict(l2=dict(deadline_ms=5)), dict(scan=dict(deadline_ms=5)),
           dict(compute=dict(legs=0x20)), dict(precision=dict(iterations=65537)), dict(sram=dict(cluster=3)),
           dict(l2=dict(bytes=12345)), dict(link=dict(bytes=24)), dict(scan=dict(chunk_bytes=8))]


@pytest.mark.parametrize("kw", REFUSED, ids=[json.dumps(k) for k in REFUSED])
def test_bad_options_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    with pytest.raises(cro.ProbeError) as e:
        cro.check_health_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG
    assert not marker.exists()


def test_an_unselected_checks_options_are_not_checked(cro, tmp_path, monkeypatch):
    fake(cro, tmp_path, monkeypatch, checks=cro.HEALTH_COMPUTE)
    r, _, _ = cro.check_health_uuid(None, U, checks=cro.HEALTH_COMPUTE, sram=dict(cluster=3))
    assert r.status == OK


def test_null_and_negative_arguments_are_refused(cro, tmp_path, monkeypatch):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    r, rec = cro.HealthResult(), cro.HealthRecords()
    f = cro.lib.cro_check_health_uuid
    assert f(None, None, None, 0, ctypes.byref(r), None, None) == ERR_INVALID_ARG
    assert f(None, U.encode(), None, 0, None, None, None) == ERR_INVALID_ARG
    rec.link_faults_cap = 1                                            # a cap without its array
    assert f(None, U.encode(), None, 0, ctypes.byref(r), ctypes.byref(rec), None) == ERR_INVALID_ARG
    rec.link_faults_cap = -1
    assert f(None, U.encode(), None, 0, ctypes.byref(r), ctypes.byref(rec), None) == ERR_INVALID_ARG
    assert cro.lib.cro_check_health(None, 0, None, ctypes.byref(r), None) == ERR_INVALID_ARG
    assert cro.lib.cro_selftest_health_classify(0, None, 1, ctypes.byref(r), ctypes.byref(ctypes.c_uint32())) == ERR_INVALID_ARG
    assert not marker.exists()
    o = cro.HealthOpts()
    o.l2.deadline_ms = 1
    assert f(None, U.encode(), ctypes.byref(o), 0, ctypes.byref(r), None, None) == ERR_INVALID_ARG
    assert r.status == ERR_INVALID_ARG and "one deadline" in last_thread_error(cro)


@pytest.mark.parametrize("argv", [["health-raw", U, "0"], ["health-raw", U] + ["0"] * 63, ["health-raw"]],
                         ids=["short", "long", "bare"])
def test_cli_refuses_a_wrong_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64
