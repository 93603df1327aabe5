"""The helper forms of the host link and compute probes without a GPU: what the library puts on the helper's argv, how
it reads the helper's output back (link-raw: result, n, n faults; compute-raw: result, n_sms, n, CRO_COMPUTE_MAX_SMS
per-SM entries, n faults), its deadline, its fresh seed bases, and the arguments it refuses before any helper starts.
The helper here is a stand-in script named by CRO_HELPER_PATH."""
import ctypes
import json
import os
import stat
import subprocess
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = "GPU-5ca90000-0000-0000-0000-000000000003"
MiB = 1 << 20
LINK_RESULT, LINK_FAULT = 984, 40
COMPUTE_RESULT, COMPUTE_SM, COMPUTE_FAULT, MAX_SMS = 600, 208, 24, 256


def test_layouts_the_framing_relies_on(cro):
    assert (ctypes.sizeof(cro.LinkResult), ctypes.sizeof(cro.LinkFault)) == (LINK_RESULT, LINK_FAULT)
    assert (ctypes.sizeof(cro.ComputeResult), ctypes.sizeof(cro.ComputeSm), ctypes.sizeof(cro.ComputeFault)) == \
        (COMPUTE_RESULT, COMPUTE_SM, COMPUTE_FAULT)
    assert cro.COMPUTE_MAX_SMS == MAX_SMS


# A stand-in helper: it leaves its argv and CUDA_VISIBLE_DEVICES in <dir>/argv.json, then writes a result whose bytes
# come from random.Random(<seed>) with the given status, min(cap, 3) records and, for compute-raw, two per-SM entries.
# `extra` is appended to stdout, `cut` bytes are dropped from its end, and `n_sms` overrides the per-SM count.
FAKE = r"""
import json, os, random, struct, sys
d = os.path.dirname(os.path.abspath(sys.argv[0]))
open(os.path.join(d, "argv.json"), "w").write(json.dumps({"argv": sys.argv[1:], "cvd": os.environ.get("CUDA_VISIBLE_DEVICES")}))
cfg = json.loads(%r)
rng = random.Random(cfg["seed"])
blob = lambda k: bytes(rng.randrange(256) for _ in range(k))
cmd, cap = sys.argv[1], int(sys.argv[-1])
n = min(cap, 3)
if cmd == "link-raw":
    assert len(sys.argv) == 11, sys.argv
    r = bytearray(blob(%d))
    struct.pack_into("<i", r, 0, cfg["status"])
    out = bytes(r) + struct.pack("<Q", n) + blob(%d * n)
else:
    assert cmd == "compute-raw" and len(sys.argv) == 15, sys.argv
    r = bytearray(blob(%d))
    struct.pack_into("<i", r, 0, cfg["status"])
    sms = blob(2 * %d) + bytes((%d - 2) * %d)
    out = bytes(r) + struct.pack("<QQ", cfg.get("n_sms", 2), n) + sms + blob(%d * n)
out += cfg.get("extra", "").encode()
out = out[:len(out) - cfg.get("cut", 0)]
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
    body = FAKE % (json.dumps(cfg), LINK_RESULT, LINK_FAULT, COMPUTE_RESULT, COMPUTE_SM, MAX_SMS, COMPUTE_SM, COMPUTE_FAULT)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, body))


def seen(tmp_path):
    with open(os.path.join(str(tmp_path), "argv.json")) as f:
        return json.load(f)


def written(tmp_path):
    with open(os.path.join(str(tmp_path), "out.bin"), "rb") as f:
        return f.read()


# ---- argv ------------------------------------------------------------------------------------------------------------
def test_link_argv_carries_every_option(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_host_link_uuid(None, U, bytes=3 * MiB + 112, hops=4097, ctas=300, inject=(3, 12345, 1 << 40), cap=7)
    s = seen(tmp_path)
    assert s["cvd"] == U
    argv = s["argv"]
    assert argv[:2] == ["link-raw", U] and len(argv) == 10
    base = int(argv[2])
    assert base and base & 0xFF == 0
    assert argv[3:] == [str(v) for v in (3 * MiB + 112, 4097, 300, 3, 12345, 1 << 40, 7)]


def test_compute_argv_carries_every_option(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_compute_uuid(None, U, iterations=9, alu_iterations=5, legs=0b10110, max_rounds=11,
                           inject=(2, 131, 8, -1, 255, 1 << 30), cap=6)
    s = seen(tmp_path)
    assert s["cvd"] == U
    argv = s["argv"]
    assert argv[:2] == ["compute-raw", U] and len(argv) == 14
    base = int(argv[2])
    assert base and base & 0xFF == 0
    assert argv[3:] == [str(v) for v in (9, 5, 0b10110, 11, 2, 131, 8, -1, 255, 1 << 30, 6)]


def test_defaults_go_to_the_helper_as_zeroes(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_host_link_uuid(None, U)
    assert seen(tmp_path)["argv"][3:] == ["0", "0", "0", "0", "0", "0", "256"]
    cro.probe_compute_uuid(None, U)
    assert seen(tmp_path)["argv"][3:] == ["0", "0", str(cro.COMPUTE_ALL_LEGS), "0", "0", "0", "0", "0", "0", "0", "256"]


def test_each_call_passes_a_new_seed_base_with_the_low_byte_clear(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    bases = []
    for call in (cro.probe_host_link_uuid, cro.probe_compute_uuid, cro.probe_host_link_uuid, cro.probe_compute_uuid):
        call(None, U)
        bases.append(int(seen(tmp_path)["argv"][2]))
    assert len(set(bases)) == len(bases) and all(b and b & 0xFF == 0 for b in bases), [hex(b) for b in bases]


# ---- what comes back -------------------------------------------------------------------------------------------------
def test_link_result_and_faults_come_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, seed=11)
    r, faults, ns = cro.probe_host_link_uuid(None, U)
    out = written(tmp_path)
    assert r.status == cro.ERR_CHECKSUM and ns > 0
    assert bytes(r) == out[:LINK_RESULT]
    assert int.from_bytes(out[LINK_RESULT:LINK_RESULT + 8], "little") == len(faults) == 3
    assert b"".join(bytes(f) for f in faults) == out[LINK_RESULT + 8:]
    r, faults, _ = cro.probe_host_link_uuid(None, U, cap=2)          # the helper is asked for at most cap faults
    assert len(faults) == 2 and b"".join(bytes(f) for f in faults) == written(tmp_path)[LINK_RESULT + 8:]
    r, faults, _ = cro.probe_host_link_uuid(None, U, cap=0)
    assert faults == [] and bytes(r) == written(tmp_path)[:LINK_RESULT]


def test_compute_result_sms_and_faults_come_back_byte_for_byte(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, seed=12)
    r, sms, faults, ns = cro.probe_compute_uuid(None, U)
    out = written(tmp_path)
    head = COMPUTE_RESULT + 16 + MAX_SMS * COMPUTE_SM
    assert r.status == cro.ERR_CHECKSUM and ns > 0
    assert bytes(r) == out[:COMPUTE_RESULT]
    assert len(sms) == 2 and b"".join(bytes(s) for s in sms) == out[COMPUTE_RESULT + 16:COMPUTE_RESULT + 16 + 2 * COMPUTE_SM]
    assert len(faults) == 3 and b"".join(bytes(f) for f in faults) == out[head:]
    r, sms, faults, _ = cro.probe_compute_uuid(None, U, cap=1)
    assert len(faults) == 1 and bytes(faults[0]) == written(tmp_path)[head:]


def test_a_clean_result_returns_ok(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.OK)
    assert cro.probe_host_link_uuid(None, U)[0].status == cro.OK
    assert cro.probe_compute_uuid(None, U)[0].status == cro.OK


def test_the_probes_own_error_is_the_calls(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch, status=cro.ERR_CUDA)                 # a failed launch is a result
    assert cro.probe_host_link_uuid(None, U)[0].status == cro.ERR_CUDA
    assert cro.probe_compute_uuid(None, U)[0].status == cro.ERR_CUDA
    fake(tmp_path, monkeypatch, status=cro.ERR_OOM)
    for call, name in ((cro.probe_host_link_uuid, "link"), (cro.probe_compute_uuid, "compute")):
        with pytest.raises(cro.ProbeError) as e:
            call(None, U)
        assert e.value.code == cro.ERR_OOM and "%s helper for %s" % (name, U) in str(e.value)


@pytest.mark.parametrize("how", [dict(extra="x"), dict(cut=1), dict(n_sms=MAX_SMS + 1)], ids=["one-more", "one-less", "n_sms"])
def test_malformed_output_is_loud(cro, tmp_path, monkeypatch, how):
    fake(tmp_path, monkeypatch, status=cro.ERR_CHECKSUM, **how)
    calls = [(cro.probe_compute_uuid, "compute")]
    if "n_sms" not in how:
        calls.append((cro.probe_host_link_uuid, "link"))
    for call, name in calls:
        with pytest.raises(cro.ProbeError) as e:
            call(None, U)
        assert e.value.code == cro.ERR_EXEC and "%s helper for %s failed" % (name, U) in str(e.value)


def test_a_crash_is_loud(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, signal\nos.kill(os.getpid(), signal.SIGSEGV)\n"))
    for call, name in ((cro.probe_host_link_uuid, "link"), (cro.probe_compute_uuid, "compute")):
        with pytest.raises(cro.ProbeError) as e:
            call(None, U)
        assert e.value.code == cro.ERR_EXEC and "%s helper for %s failed" % (name, U) in str(e.value)


def test_exit_3_is_no_device(cro, tmp_path, monkeypatch):
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    for call in (cro.probe_host_link_uuid, cro.probe_compute_uuid):
        with pytest.raises(cro.ProbeError) as e:
            call(None, U)
        assert e.value.code == cro.ERR_NO_DEVICE


@pytest.mark.parametrize("which", ["link", "compute"])
def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch, which):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    call = cro.probe_host_link_uuid if which == "link" else cro.probe_compute_uuid
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        call(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "%s helper" % which in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    pid = int(marker.read_text())
    with pytest.raises(ProcessLookupError):                            # killed and reaped: no process is left behind
        os.kill(pid, 0)


# ---- refused before any helper starts --------------------------------------------------------------------------------
LINK_REFUSED = [dict(bytes=8), dict(bytes=24), dict(bytes=MiB + 8), dict(hops=(1 << 24) + 1), dict(ctas=4097),
                dict(inject=(5, 0, 1)), dict(inject=(-1, 0, 1)), dict(bytes=MiB, inject=(0, MiB // 8, 1)),
                dict(inject=(4, (256 * MiB) // 8, 1))]
COMPUTE_REFUSED = [dict(legs=0x20), dict(iterations=65537), dict(alu_iterations=1025), dict(max_rounds=65),
                   dict(inject=(5, 0, 0, 0, 0, 1)), dict(inject=(-1, 0, 0, 0, 0, 1)), dict(inject=(0, 256, 0, 0, 0, 1)),
                   dict(inject=(0, -2, 0, 0, 0, 1)), dict(inject=(0, 0, 0, 128, 0, 1)), dict(inject=(0, 0, 0, 0, 256, 1)),
                   dict(inject=(0, 0, 0, -2, 0, 1)), dict(inject=(0, 0, 3, 0, 0, 1), iterations=3),
                   dict(inject=(3, 0, 4, 0, 0, 1)), dict(inject=(4, 0, 2, 0, 0, 1), alu_iterations=2)]


def marker_helper(tmp_path, monkeypatch):
    marker = tmp_path / "ran"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('ran')\n" % str(marker)))
    return marker


def last_thread_error(cro):
    buf = ctypes.create_string_buffer(1024)
    cro.lib.cro_last_error(None, buf, 1024)
    return buf.value.decode()


@pytest.mark.parametrize("kw", LINK_REFUSED, ids=[json.dumps(k) for k in LINK_REFUSED])
def test_link_arguments_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = marker_helper(tmp_path, monkeypatch)
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_host_link_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "): host link probe: L = " in str(e.value)
    assert not marker.exists()


@pytest.mark.parametrize("kw", COMPUTE_REFUSED, ids=[json.dumps(k) for k in COMPUTE_REFUSED])
def test_compute_arguments_are_refused_before_spawning(cro, tmp_path, monkeypatch, kw):
    marker = marker_helper(tmp_path, monkeypatch)
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_compute_uuid(None, U, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG and "): compute probe: legs must be" in str(e.value)
    assert not marker.exists()


def test_the_largest_legal_options_do_reach_the_helper(cro, tmp_path, monkeypatch):
    fake(tmp_path, monkeypatch)
    cro.probe_host_link_uuid(None, U, bytes=16, hops=1 << 24, ctas=4096, inject=(4, 1, 1))
    assert seen(tmp_path)["argv"][3:6] == ["16", str(1 << 24), "4096"]
    cro.probe_compute_uuid(None, U, iterations=65536, alu_iterations=1024, max_rounds=64, inject=(4, 255, 1023, 127, -1, 1))
    assert seen(tmp_path)["argv"][3:7] == ["65536", "1024", str(cro.COMPUTE_ALL_LEGS), "64"]


def test_null_and_negative_arguments_are_refused(cro, tmp_path, monkeypatch):
    marker = marker_helper(tmp_path, monkeypatch)
    L, lf, n, ns = cro.LinkResult(), (cro.LinkFault * 4)(), ctypes.c_int(-1), ctypes.c_uint64()
    link = cro.lib.cro_probe_host_link_uuid
    assert link(None, None, None, 0, ctypes.byref(L), lf, 4, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert link(None, U.encode(), None, 0, None, lf, 4, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert link(None, U.encode(), None, 0, ctypes.byref(L), lf, -1, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert link(None, U.encode(), None, 0, ctypes.byref(L), None, 4, ctypes.byref(n), ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    assert link(None, U.encode(), None, 0, ctypes.byref(L), lf, 4, None, ctypes.byref(ns)) == cro.ERR_INVALID_ARG
    C, sms, cf, k = cro.ComputeResult(), (cro.ComputeSm * 4)(), (cro.ComputeFault * 4)(), ctypes.c_int(-1)
    comp = cro.lib.cro_probe_compute_uuid
    ok = dict(ctx=None, uuid=U.encode(), opts=None, dl=0, out=ctypes.byref(C), sms=sms, sms_cap=4, n_sms=ctypes.byref(k),
              faults=cf, cap=4, n=ctypes.byref(n), ns=ctypes.byref(ns))
    for bad in (dict(uuid=None), dict(out=None), dict(sms=None), dict(sms_cap=-1), dict(n_sms=None), dict(faults=None),
                dict(cap=-1), dict(n=None)):
        a = dict(ok, **bad)
        assert comp(*a.values()) == cro.ERR_INVALID_ARG, bad
    assert not marker.exists()


def test_a_bad_option_sets_the_thread_error(cro, tmp_path, monkeypatch):
    marker_helper(tmp_path, monkeypatch)
    o, r, n = cro.LinkOpts(), cro.LinkResult(), ctypes.c_int()
    o.bytes = 24
    assert cro.lib.cro_probe_host_link_uuid(None, U.encode(), ctypes.byref(o), 0, ctypes.byref(r), None, 0, ctypes.byref(n),
                                            None) == cro.ERR_INVALID_ARG
    assert r.status == cro.ERR_INVALID_ARG and r.first_fail == cro.LINK_NO_FAIL
    assert last_thread_error(cro).startswith("host link probe: L = 24 must be a multiple of 16 in [16, 24]")


# ---- the helper's own argv checks ------------------------------------------------------------------------------------
@pytest.mark.parametrize("argv", [["link-raw", U, "0"], ["link-raw", U] + ["0"] * 9, ["compute-raw", U, "0"],
                                  ["compute-raw", U] + ["0"] * 13, ["link-raw"], ["compute-raw"]],
                         ids=["link-short", "link-long", "compute-short", "compute-long", "link-bare", "compute-bare"])
def test_cli_refuses_a_wrong_argument_count(cro, argv):
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    assert subprocess.run([cli] + argv, capture_output=True, timeout=60).returncode == 64
