"""CRO_* knobs are validated the way the reference validates its environment
(internal/controller/composableresource_adapter.go:42-45, :64, :67): strict parse, legal range, one wording."""
import os
import re
import shutil
import subprocess

import pytest

REF_LINE = "the env variable DEVICE_RESOURCE_TYPE has an invalid value: '%s'"     # composableresource_adapter.go:44


def test_wording_is_the_references(cro):
    msg = cro.validate_env("CRO_USE_GRAPH", "yes")
    assert msg == REF_LINE.replace("DEVICE_RESOURCE_TYPE", "CRO_USE_GRAPH") % "yes"


@pytest.mark.parametrize("name,value,ok", [
    ("CRO_TMA_READ_TILE", "32768", True), ("CRO_TMA_READ_TILE", "32769", False), ("CRO_TMA_READ_TILE", "512", False),
    ("CRO_TMA_READ_TILE", "0x8000", False), ("CRO_TMA_READ_TILE", " 32768", False), ("CRO_TMA_READ_TILE", "-16", False),
    ("CRO_TMA_READ_STAGES", "4", True), ("CRO_TMA_READ_STAGES", "1", False), ("CRO_TMA_READ_STAGES", "17", False),
    ("CRO_FUSED_THREADS", "160", True), ("CRO_FUSED_THREADS", "150", False), ("CRO_EXPECT_CTAS", "2", True), ("CRO_EXPECT_CTAS", "0", False),
    ("CRO_P2P_READ_VARIANT", "2", True), ("CRO_P2P_READ_VARIANT", "0", False), ("CRO_USE_GRAPH", "", True),
    ("CRO_HELPER_TIMEOUT_MS", "99999999999999999999", False), ("CRO_USE_GRAPH", "1x", False),
])
def test_each_knob_has_a_range(cro, name, value, ok):
    msg = cro.validate_env(name, value)
    assert (msg == "") == ok, (name, value, msg)
    if not ok:
        assert msg == "the env variable %s has an invalid value: '%s'" % (name, value)


def test_process_environment_is_checked_as_a_whole(cro, monkeypatch):
    assert cro.validate_env() == ""
    monkeypatch.setenv("CRO_FUSED_TILE", "114688")
    monkeypatch.setenv("CRO_FUSED_STAGES", "4")                 # 448 KiB of ring: more shared memory than a CTA may own
    assert cro.validate_env() == "the env variable CRO_FUSED_TILE has an invalid value: '114688'"
    monkeypatch.setenv("CRO_FUSED_STAGES", "2")
    assert cro.validate_env() == ""


def test_no_raw_atoi_of_the_environment_is_left():
    import glob
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for path in glob.glob(os.path.join(root, "composable-resource-operator_b200", "csrc", "*.cu")):
        src = open(path).read()
        assert not re.search(r"atoi\s*\(\s*getenv", src) and "env_int(" not in src and "env_u32(" not in src, path


def test_chase_end_matches_the_golden_vectors(cro):
    """The product's restatement of the latency permutation (std::mt19937_64 + Sattolo) against the vectors the pure-Python
    generator wrote (tests/golden/make_pattern_kats.py)."""
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    g = json.load(open(os.path.join(root, "tests", "golden", "pattern_kats.json")))
    for c in g["chase_ends"]:
        assert cro.chase_end(c["minor_src"], c["minor_dst"], c["hops"]) == c["end"], c


# An sm_90 CTA may own this much shared memory, static and dynamic together (cudaDevAttrMaxSharedMemoryPerBlockOptin
# of an H100).
SMEM_PER_BLOCK_OPTIN = 232448
RINGS = {          # knob prefix -> ring kernel
    "CRO_TMA_READ": "hbm_read_tma_kernel",
    "CRO_TMA_COPY": "hbm_copy_tma_kernel",
    "CRO_FUSED": "hbm_copy_fused_kernel",
}


def largest_ring_tile(cro, monkeypatch, prefix, stages):
    """Sets <prefix>_STAGES and the largest <prefix>_TILE the process-environment check accepts at that depth, and
    returns that tile.  Bisection in 16-byte steps: the tile's own range is [1024, 114688]."""
    monkeypatch.setenv(prefix + "_STAGES", str(stages))
    lo, hi = 1024 // 16, 114688 // 16          # 1024-byte tiles fit at every depth
    while lo < hi:
        mid = (lo + hi + 1) // 2
        monkeypatch.setenv(prefix + "_TILE", str(16 * mid))
        if cro.validate_env() == "":
            lo = mid
        else:
            hi = mid - 1
    monkeypatch.setenv(prefix + "_TILE", str(16 * lo))
    return 16 * lo


def ring_kernels_static_smem(cro):
    """Static shared memory of each ring kernel in the built library, as cudaFuncGetAttributes().sharedSizeBytes
    reports it.  cuobjdump's SHARED figure also counts the 1 KiB the system reserves per CTA, so that is taken off."""
    import __graft_entry__ as g
    nvcc = g._nvcc()
    tool = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.dirname(nvcc) else shutil.which("cuobjdump")
    out = subprocess.run([tool, "-res-usage", cro.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"\bSHARED:(\d+)", line)
        if m and fn:
            for kernel in RINGS.values():
                if kernel in fn:
                    found[kernel] = int(m.group(1)) - 1024
            fn = None
    assert set(found) == set(RINGS.values()), out
    return found


def test_largest_legal_ring_fits_beside_the_kernels_static_shared_memory(cro, monkeypatch):
    """Every ring cro_validate_env accepts must be one the device can launch: ring + the kernel's static shared memory
    within what a CTA may own.  Otherwise a legal knob setting fails at plan time."""
    static = ring_kernels_static_smem(cro)
    for prefix, kernel in RINGS.items():
        assert 0 < static[kernel] <= 2048, (kernel, static[kernel])
        for stages in (2, 3, 4, 5, 8, 16):
            tile = largest_ring_tile(cro, monkeypatch, prefix, stages)
            assert tile * stages + static[kernel] <= SMEM_PER_BLOCK_OPTIN, (prefix, stages, tile, static[kernel])
            if tile < 114688:                  # one step more is refused, with the tile knob's sentence
                monkeypatch.setenv(prefix + "_TILE", str(tile + 16))
                assert cro.validate_env() == "the env variable %s_TILE has an invalid value: '%d'" % (prefix, tile + 16)
            monkeypatch.delenv(prefix + "_TILE")
            monkeypatch.delenv(prefix + "_STAGES")
