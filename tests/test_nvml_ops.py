"""csrc/nvml_ops.cpp: the detach side's nvidia-smi invocations answered through NVML in the agent's own process
(reference: internal/utils/gpus.go:125,134 compute apps; :970 drain -q; :267,269,311 the three mutating commands).

This container has no NVML, so the CPU tests load tests/fake_nvml.c as the library; the texts they expect for the two
QUERIES are the ones captured from the real nvidia-smi on a GPU box (tests/golden/nvidia_smi_texts.json, made by
tools/smi_texts.sh).  The GPU test compares the native answers with the box's real nvidia-smi byte for byte."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "nvidia_smi_texts.json")))["cases"]
SMI = "/usr/bin/nvidia-smi"
A, B = "GPU-aaaaaaaa-0000-0000-0000-000000000001", "GPU-bbbbbbbb-0000-0000-0000-000000000002"
FMT = "--format=csv,noheader,nounits"
APPS = [SMI, "--query-compute-apps=gpu_uuid,process_name", FMT]


@pytest.fixture(scope="module")
def fake_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("fake_nvml") / "libfake-nvml.so"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-o", str(out), os.path.join(HERE, "fake_nvml.c")])
    return str(out)


@pytest.fixture
def node(tmp_path, monkeypatch):
    """Two GPUs at 0000:40:00.0 and 0000:41:00.0, nothing running, nothing draining."""
    (tmp_path / "gpus").write_text("%s 00000000:40:00.0 1\n%s 00000000:41:00.0 1\n" % (A, B))
    (tmp_path / "procs").write_text("")
    (tmp_path / "drain").write_text("00000000:40:00.0 0\n00000000:41:00.0 0\n")
    monkeypatch.setenv("FAKE_NVML_DIR", str(tmp_path))
    return tmp_path


def calls(node):
    p = node / "calls"
    return p.read_text().splitlines() if p.exists() else []


def test_compute_apps(cro, fake_lib, node):
    out = cro.local_exec(APPS, nvml_lib=fake_lib)
    assert out == {"how": "native", "failed": False, "exec_err": "", "stdout": GOLD["apps_idle"]["stdout"], "stderr": ""}
    (node / "procs").write_text("%s 192 python\n%s 200 /usr/bin/gpu_load_progress\n%s 77 -\n" % (A, B, B))
    out = cro.local_exec(["/bin/chroot", "/host-root"] + APPS, nvml_lib=fake_lib)
    assert out["how"] == "native" and not out["failed"]
    # the captured line is "<uuid>, python\n": same separator, same name column
    assert out["stdout"].splitlines()[0] == GOLD["apps_busy2"]["stdout"].strip().replace("GPU-00000000-0000-0000-0000-000000000000", A)
    assert out["stdout"] == "%s, python\n%s, /usr/bin/gpu_load_progress\n%s, [Not Found]\n" % (A, B, B)
    # more processes than the first buffer holds: NVML says INSUFFICIENT_SIZE with the count, the call is repeated
    (node / "procs").write_text("".join("%s %d p%d\n" % (A, 1000 + i, i) for i in range(150)))
    out = cro.local_exec(APPS, nvml_lib=fake_lib)
    assert out["stdout"].count("\n") == 150 and out["stdout"].endswith("%s, p149\n" % A)


def test_no_devices_is_the_references_empty_node(cro, fake_lib, node):
    """CheckNoGPULoads returns nil on 'No devices were found' BEFORE looking at the exec error (gpus.go:143-147)."""
    (node / "gpus").write_text("")
    out = cro.local_exec(APPS, nvml_lib=fake_lib)
    assert out["stdout"] == "No devices were found\n" and out["failed"] and out["exec_err"] == "command terminated with exit code 6"
    res = cro.local_node_op(None, {"op": "check_no_gpu_loads", "node": "worker-0", "device_id": A, "driver_container": True, "nvml_lib": fake_lib})
    assert res["error"] == "" and res["exec_log"][0]["how"] == "native"


def test_load_check_through_the_flow(cro, fake_lib, node):
    (node / "procs").write_text("%s 192 gpu_load_progress\n" % A)
    res = cro.local_node_op(None, {"op": "check_no_gpu_loads", "node": "worker-0", "device_id": A, "driver_container": True, "nvml_lib": fake_lib})
    assert res["error"] == "found gpu loads on node 'worker-0': '[GPUUUID: '%s', ProcessName: 'gpu_load_progress']'" % A
    assert [x["how"] for x in res["exec_log"]] == ["native"]


@pytest.mark.parametrize("case,bus", [("drain_q_short", "0000:40:00.0"), ("drain_q_lower", "0000:40:00.0"), ("drain_q_long", "00000000:40:00.0"),
                                      ("drain_q_bad", "0000:FE:00.0"), ("drain_q_junk", "junk")])
def test_drain_query_matches_the_captured_nvidia_smi(cro, fake_lib, node, case, bus):
    want = GOLD[case]
    out = cro.local_exec(["/bin/chroot", "/host-root", SMI, "drain", "-p", bus, "-q"], nvml_lib=fake_lib)
    assert out["how"] == "native" and out["stdout"] == want["stdout"] and out["stderr"] == want["stderr"]
    assert out["failed"] == (want["rc"] != 0)
    assert out["exec_err"] == ("command terminated with exit code %d" % want["rc"] if want["rc"] else "")


def test_draining_state_and_spellings(cro, fake_lib, node):
    (node / "drain").write_text("00000000:40:00.0 1\n00000000:41:00.0 0\n")
    for spelling in ("0000:40:00.0", "0000:40:00", "40:00.0", "0000:40:0.0"):
        out = cro.local_exec([SMI, "drain", "-p", spelling, "-q"], nvml_lib=fake_lib)
        assert out["stdout"] == "The current drain state of GPU 00000000:40:00.0 is: draining.\n", spelling
    out = cro.local_exec([SMI, "drain", "-p", "0000:41:00.0", "-q"], nvml_lib=fake_lib)
    assert out["stdout"] == "The current drain state of GPU 00000000:41:00.0 is: not draining.\n"


def test_mutating_commands_stay_behind_the_dry_run_gate(cro, fake_lib, node):
    for argv in ([SMI, "-i", A, "-pm", "0"], [SMI, "drain", "-p", "0000:40:00.0", "-m", "1"], [SMI, "drain", "-p", "0000:40:00.0", "-r"]):
        out = cro.local_exec(argv, nvml_lib=fake_lib)
        assert out["how"] == "skipped (dry run)" and not out["failed"], argv
    assert calls(node) == []


def test_detach_sequence_with_mutation_allowed(cro, fake_lib, node):
    """The reference's order (gpus.go:523-529): persistence mode off, maintenance mode on, remove."""
    out = cro.local_exec([SMI, "drain", "-p", "0000:40:00.0", "-r"], allow_mutation=True, nvml_lib=fake_lib)
    assert out["how"] == "native" and out["failed"] and out["exec_err"] == "command terminated with exit code 255"     # not draining yet
    assert out["stdout"] == "Failed to remove the GPU: In use by another client\n"
    out = cro.local_exec([SMI, "-i", A, "-pm", "0"], allow_mutation=True, nvml_lib=fake_lib)
    assert out == {"how": "native", "failed": False, "exec_err": "", "stdout": "Disabled persistence mode for GPU 00000000:40:00.0.\nAll done.\n", "stderr": ""}
    out = cro.local_exec([SMI, "drain", "-p", "0000:40:00.0", "-m", "1"], allow_mutation=True, nvml_lib=fake_lib)
    assert not out["failed"] and out["stdout"] == "Successfully set GPU 00000000:40:00.0 drain state to: draining.\n"
    out = cro.local_exec([SMI, "drain", "-p", "0000:40:00.0", "-q"], nvml_lib=fake_lib)
    assert out["stdout"].endswith("is: draining.\n")
    out = cro.local_exec([SMI, "drain", "-p", "0000:40:00.0", "-r"], allow_mutation=True, nvml_lib=fake_lib)
    assert not out["failed"] and out["stdout"] == "Successfully removed GPU 00000000:40:00.0\n"
    assert calls(node) == ["set_persistence %s 0" % A, "modify_drain 00000000:40:00.0 1 domain=0 bus=40 device=0",
                           "remove_gpu 00000000:40:00.0 gpu_state=1 link_state=0"]
    # an unknown device for -i: nvidia-smi's empty-selection answer
    out = cro.local_exec([SMI, "-i", "GPU-nope", "-pm", "0"], allow_mutation=True, nvml_lib=fake_lib)
    assert out["stdout"] == "No devices were found\n" and out["exec_err"] == "command terminated with exit code 6"


def test_nvml_failure_is_an_exec_failure(cro, fake_lib, node):
    (node / "fail").write_text("nvmlDeviceModifyDrainState 4\n")
    out = cro.local_exec([SMI, "drain", "-p", "0000:40:00.0", "-m", "1"], allow_mutation=True, nvml_lib=fake_lib)
    assert out["failed"] and out["stdout"] == "Failed to set the GPU drain state: Insufficient Permissions\n"
    assert calls(node) == []


def test_without_nvml_the_command_is_spawned(cro, tmp_path):
    """No library (this container) or native_nvml off: the reference's way, a child process."""
    out = cro.local_exec(APPS, nvml_lib=str(tmp_path / "no-such-lib.so"))
    assert out["how"] == "spawned"
    out = cro.local_exec(APPS, native_nvml=False)
    assert out["how"] == "spawned"


@pytest.mark.gpu
def test_native_answers_equal_the_real_nvidia_smi(cro):
    """On the box: same bytes as the command the reference execs — compute apps (this process holds a CUDA context, so
    there is a row) and the drain query in the spelling the reference passes (4-digit domain, gpus.go:406)."""
    if not os.path.exists(SMI):
        pytest.skip("no nvidia-smi on this box")
    with cro.ProbeContext(sweep_bytes=64 << 20, devices=[0], read_sweeps=1, copy_sweeps=1) as ctx:
        ctx.probe_device(0)
        bus = ctx.own_devices()[0].pci_bus_id.decode()
        native = cro.local_exec(APPS)
        real = cro.local_exec(APPS, native_nvml=False)
        assert native["how"] == "native" and real["how"] == "spawned"
        assert native["stdout"] and sorted(native["stdout"].splitlines()) == sorted(real["stdout"].splitlines())
        assert (native["failed"], native["stderr"]) == (real["failed"], real["stderr"])
        for spelling in (bus[4:], bus[4:].lower(), bus, "0000:FE:00.0", "junk"):
            argv = [SMI, "drain", "-p", spelling, "-q"]
            native, real = cro.local_exec(argv), cro.local_exec(argv, native_nvml=False)
            assert native["how"] == "native" and real["how"] == "spawned"
            assert {k: native[k] for k in ("stdout", "stderr", "failed", "exec_err")} == {k: real[k] for k in ("stdout", "stderr", "failed", "exec_err")}, spelling
        print("native == nvidia-smi:", native["stdout"].strip())


def test_query_gpu_without_a_probe_context(cro, fake_lib, node):
    out = cro.local_exec([SMI, "--query-gpu=device_minor,gpu_uuid,pci.bus_id", FMT], nvml_lib=fake_lib)
    assert out["how"] == "native" and out["stdout"] == "0, %s, 00000000:40:00.0\n1, %s, 00000000:41:00.0\n" % (A, B)
    # a host whose NVML will not give PCI info (NVML_ERROR_NOT_SUPPORTED): nvidia-smi prints "[N/A]" for the bus id
    (node / "fail").write_text("nvmlDeviceGetPciInfo_v3 3\n")
    out = cro.local_exec([SMI, "--query-gpu=gpu_uuid,pci.bus_id", FMT], nvml_lib=fake_lib)
    assert out["how"] == "native" and out["stdout"] == "%s, [N/A]\n%s, [N/A]\n" % (A, B)
    # a field this library does not know is nvidia-smi's to answer
    out = cro.local_exec([SMI, "--query-gpu=temperature.gpu", FMT], nvml_lib=fake_lib)
    assert out["how"] == "spawned"
    (node / "gpus").write_text("")
    out = cro.local_exec([SMI, "--query-gpu=gpu_uuid", FMT], nvml_lib=fake_lib)
    assert out["stdout"] == "No devices were found\n"


def test_whole_drain_is_library_calls(cro, fake_lib, node, tmp_path):
    """DrainGPU, OCP + DEVICE_PLUGIN flavour (gpus.go:556-664), on the node with mutation allowed: enumerate, persistence
    mode off, open-file scan of /dev/nvidia<minor>, maintenance mode, remove — no child process anywhere."""
    proc = tmp_path / "proc"
    (proc / "100" / "fd").mkdir(parents=True)
    (proc / "100" / "cmdline").write_bytes(b"/usr/bin/sleep\09\0")
    (proc / "100" / "comm").write_text("sleep\n")
    req = {"op": "drain", "node": "worker-0", "device_id": B, "device_resource_type": "DEVICE_PLUGIN", "driver_container": True,
           "allow_mutation": True, "nvml_lib": fake_lib, "proc_root": str(proc)}
    res = cro.local_node_op(None, req)
    assert res["error"] == "", res
    assert [(x["kind"], x["how"]) for x in res["exec_log"]] == [("command", "native"), ("command", "native"), ("fd_scan", "native"),
                                                                ("command", "native"), ("command", "native")]
    assert [x["argv"][1:] for x in res["exec_log"] if x["kind"] == "command"] == [
        ["--query-gpu=device_minor,gpu_uuid,pci.bus_id", FMT], ["-i", B, "-pm", "0"],
        ["drain", "-p", ":41:00.0".join(["0000", ""]), "-m", "1"], ["drain", "-p", "0000:41:00.0", "-r"]]
    assert calls(node) == ["set_persistence %s 0" % B, "modify_drain 00000000:41:00.0 1 domain=0 bus=41 device=0",
                           "remove_gpu 00000000:41:00.0 gpu_state=1 link_state=0"]
    # the same request as a dry run changes nothing
    (node / "calls").unlink()
    res = cro.local_node_op(None, dict(req, allow_mutation=False))
    assert res["error"] == "" and calls(node) == []
    assert [x["how"] for x in res["exec_log"]] == ["native", "skipped (dry run)", "native", "skipped (dry run)", "skipped (dry run)"]
    # a GPU that is no longer enumerated was already drained (gpus.go:366)
    res = cro.local_node_op(None, dict(req, device_id="GPU-gone"))
    assert res["error"] == "" and len(res["exec_log"]) == 1


def test_a_refused_maintenance_mode_stops_the_drain_where_the_reference_stops(cro, fake_lib, node, tmp_path):
    (node / "fail").write_text("nvmlDeviceModifyDrainState 4\n")
    proc = tmp_path / "proc"
    proc.mkdir()
    res = cro.local_node_op(None, {"op": "drain", "node": "worker-0", "device_id": A, "device_resource_type": "DEVICE_PLUGIN",
                                   "driver_container": True, "allow_mutation": True, "nvml_lib": fake_lib, "proc_root": str(proc)})
    assert res["error"] == ("detach command 'set maintenance mode' failed: 'command terminated with exit code 255', stderr: '', "
                            "stdout: 'Failed to set the GPU drain state: Insufficient Permissions\n'")
    assert calls(node) == ["set_persistence %s 0" % A]          # no remove after the refusal


@pytest.mark.gpu
def test_probe_context_identity_follows_nvml_bus_id(cro, fake_lib, tmp_path):
    """A context takes the bus id from NVML when NVML knows the device, and spells it "[N/A]" — nvidia-smi's answer — when
    NVML refuses the PCI info.  A fresh process loads tests/fake_nvml.c as libnvidia-ml.so.1, listing this GPU's UUID."""
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC | cro.F_NO_NVML) as c:
        uuid = c.own_devices()[0].gpu_uuid.decode()
    libdir = tmp_path / "lib"
    libdir.mkdir()
    os.symlink(fake_lib, str(libdir / "libnvidia-ml.so.1"))
    state = tmp_path / "state"
    state.mkdir()
    (state / "gpus").write_text("%s 00000000:4A:00.0 1\n" % uuid)
    root = os.path.dirname(HERE)
    child = ("import importlib, sys; sys.path.insert(0, %r); cro = importlib.import_module('composable-resource-operator_b200')\n"
             "with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as c:\n"
             "    print(cro.emit_csv(c.own_devices(), 'gpu_uuid,pci.bus_id'), end='')\n" % root)
    env = dict(os.environ, LD_LIBRARY_PATH=str(libdir) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""), FAKE_NVML_DIR=str(state))
    for fail, want in (("", "00000000:4A:00.0"), ("nvmlDeviceGetPciInfo_v3 3\n", "[N/A]")):
        (state / "fail").write_text(fail)
        out = subprocess.run([sys.executable, "-c", child], env=env, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr[-1500:]
        assert out.stdout == "%s, %s\n" % (uuid, want), out.stdout

