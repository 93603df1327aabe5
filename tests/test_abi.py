"""The C-ABI library loads, exports every symbol include/croprobe.h declares,
keeps the 512-byte result layout, and fails loudly without a GPU."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "croprobe.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cro_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(cro):
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(cro.lib, s), "declared in croprobe.h but not exported: " + s
    assert sorted(cro.EXPORTS) == syms, set(cro.EXPORTS) ^ set(syms)


def test_result_struct_layout(cro):
    R = cro.ProbeResult
    assert ctypes.sizeof(R) == 512
    offs = {"gpu_uuid": 16, "pci_bus_id": 64, "hbm_bytes_total": 88, "checksum_xor": 112, "fill_ns": 128,
            "sm_count": 168, "p2p_read_ns": 184, "p2p_checksum_xor": 248, "p2p_latency_ns_x16": 312,
            "p2p_access": 344, "p2p_bytes": 352, "expect_wsum": 376, "checksum_wsum": 384, "copy_checksum_wsum": 408,
            "total_ns": 416, "p2p_write_ns": 424, "nonce": 488, "rank": 492, "copy_verified": 498, "fail_code": 499,
            "p2p_ok": 501, "t_start_ns": 504}
    assert ctypes.sizeof(cro.SweepResult) == 56 and ctypes.sizeof(cro.SweepTime) == 32 and ctypes.sizeof(cro.P2PDetail) == 120
    assert ctypes.sizeof(cro.FullBoxTime) == 64
    for k, v in offs.items():
        assert getattr(R, k).offset == v, k


def test_library_has_sm90a_code_and_hopper_instructions():
    so = os.path.join(ROOT, "composable-resource-operator_b200", "libcroprobe.so")
    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout and "sm_100" not in out.stdout
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass, "1-D TMA bulk copies must be present (cp.async.bulk)"
    assert "SYNCS" in sass, "mbarrier instructions must be present"
    assert "LDG.E.NA.128.CONSTANT" in sass, "128-bit read-only, no-L1-allocate global loads must be present"


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_no_gpu_fails_loudly(cro):
    """There is no CPU fallback: without a device the probe context refuses to exist."""
    with pytest.raises(cro.ProbeError) as e:
        cro.ProbeContext(sweep_bytes=1 << 20)
    assert e.value.code in (cro.ERR_NO_DEVICE, cro.ERR_CUDA)


def test_strerror_and_version(cro):
    assert cro.strerror(0) == "ok"
    assert cro.strerror(cro.ERR_CHECKSUM) == "hbm checksum mismatch"
    assert "sm_90a" in cro.version()


def build_c_harness(out_dir):
    """gcc (plain C, not nvcc / g++) against include/croprobe.h, linked to the shared library like cgo does.  The
    executable goes to out_dir: the checkout under test may be read-only."""
    exe = os.path.join(str(out_dir), "c_abi_harness")
    src = os.path.join(ROOT, "tests", "c_abi_harness.c")
    pkg = os.path.join(ROOT, "composable-resource-operator_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L" + pkg, "-lcroprobe", "-Wl,-rpath," + pkg])
    return exe


def test_c_harness_links_and_runs_like_cgo(cro, tmp_path):
    exe = build_c_harness(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "c abi harness ok" in out.stdout


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_cli_without_gpu(cro):
    """The helper process: an empty box enumerates as nvidia-smi says it ("No devices were found"),
    and a probe refuses loudly (no CPU fallback)."""
    cli = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
    out = subprocess.run([cli, "csv", "gpu_uuid"], capture_output=True, text=True)
    assert (out.returncode, out.stdout) == (0, "No devices were found\n")
    rc, js = cro.getGPUInfoFromNvidiaSmiOutput(out.stdout, "", None, "gpu_uuid")
    assert (rc, js) == (0, "[]")                      # and the reference's parse rule turns that into an empty list
    out = subprocess.run([cli, "probe", "0"], capture_output=True, text=True)
    assert out.returncode == 2 and "no CUDA device" in out.stderr


def test_product_never_touches_the_oracle():
    """The shipped path must not include, link or import anything under oracle/."""
    pkg = os.path.join(ROOT, "composable-resource-operator_b200")
    for dirpath, _dirs, files in os.walk(pkg):
        if "build" in dirpath:
            continue
        for f in files:
            if f.endswith((".cu", ".cpp", ".hpp", ".cuh", ".py", ".go", ".h")):
                t = open(os.path.join(dirpath, f), errors="replace").read()
                assert "cro_oracle" not in t and "liboracle" not in t and "import oracle" not in t, os.path.join(dirpath, f)
    so = os.path.join(pkg, "libcroprobe.so")
    out = subprocess.run(["nm", "-D", so], capture_output=True, text=True).stdout
    assert "oracle_" not in out


def test_no_exception_crosses_the_abi(cro):
    """Every entry point is a function-try-block (c_api_util.hpp: CRO_API_CATCH): an exception thrown behind the ABI comes
    back as a code, with its text kept for the calling thread."""
    import ctypes
    buf = ctypes.create_string_buffer(256)
    assert cro.lib.cro_selftest_exception_barrier(0) == cro.ERR_INTERNAL
    cro.lib.cro_last_error(None, buf, len(buf))
    assert buf.value == b"internal error: exception barrier self-test"
    assert cro.lib.cro_selftest_exception_barrier(1) == cro.ERR_OOM
    cro.lib.cro_last_error(None, buf, len(buf))
    assert buf.value == b"out of host memory"
    assert cro.lib.cro_selftest_exception_barrier(2) == cro.ERR_INTERNAL
    assert cro.lib.cro_selftest_exception_barrier(7) == cro.OK


def test_only_the_c_abi_is_exported():
    """csrc/croprobe.map: the C++ internals and the static CUDA runtime stay local to the library."""
    import subprocess
    out = subprocess.check_output(["nm", "-D", "--defined-only", os.path.join(ROOT, "composable-resource-operator_b200", "libcroprobe.so")], text=True)
    names = [ln.split()[-1] for ln in out.splitlines() if ln.strip()]
    assert names and all(n.startswith("cro_") for n in names), [n for n in names if not n.startswith("cro_")][:5]


def test_every_int_entry_point_has_the_barrier():
    """Source check: each `int cro_*(...)` definition in the extern "C" units opens with `try {` and ends in CRO_API_CATCH."""
    import re
    for unit in ("c_api.cu", "harness.cu"):
        text = open(os.path.join(ROOT, "composable-resource-operator_b200", "csrc", unit)).read()
        defs = re.findall(r"^int\s+(cro_\w+)\([^;{]*\)\s*(try\s*)?\{", text, re.M)
        assert defs, unit
        missing = [name for name, t in defs if not t]
        assert not missing, (unit, missing)
        assert text.count("CRO_API_CATCH") == len(defs), (unit, text.count("CRO_API_CATCH"), len(defs))
