"""The host link probe's C structs, annotation emitter and sysfs path reader, without a GPU.

The ctypes mirrors of cro_link_opts / cro_link_fault / cro_link_leg / cro_link_check / cro_link_result / cro_pci_hop /
cro_pci_path are held to the header as gcc lays it out; cro_emit_link_annotations_json is held byte for byte to
oracle/link.py on crafted results; cro_pci_link_path runs on fake sysfs trees."""
import ctypes
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = {
    "cro_link_opts": ("LinkOpts", ["bytes", "hops", "ctas", "test_inject_check", "reserved0", "test_inject_word",
                                   "test_inject_mask"]),
    "cro_link_fault": ("LinkFault", ["check", "reserved", "word_index", "expected", "actual", "host_value"]),
    "cro_link_leg": ("LinkLeg", ["bytes", "ns", "timer_ns"]),
    "cro_link_check": ("LinkCheck", ["words", "mismatches", "recorded", "seed", "fold_xor", "fold_sum", "fold_wsum",
                                     "expect_xor", "expect_sum", "expect_wsum"]),
    "cro_link_result": ("LinkResult", ["status", "first_fail", "bytes", "seed", "call", "leg", "ce_duplex_span_ns", "check",
                                       "chase_hops", "chase_end", "chase_expect", "chase_minor", "chase_ns", "dev_numa",
                                       "host_numa", "no_nvml", "degraded", "replays_before", "replays_after", "path"]),
    "cro_pci_hop": ("PciHop", ["bdf", "cur_speed", "cur_width", "max_speed", "max_width"]),
    "cro_pci_path": ("PciPath", ["numa_node", "n_hops", "bottleneck", "truncated", "hop"]),
}


def test_ctypes_layout_matches_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
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


# ---- the emitter against oracle/link.py ---------------------------------------------------------------------------
def as_dict(r):
    return {
        "status": r.status, "first_fail": r.first_fail,
        "leg": [{"bytes": g.bytes, "ns": g.ns} for g in r.leg], "ce_duplex_span_ns": r.ce_duplex_span_ns,
        "chase_hops": r.chase_hops, "chase_ns": r.chase_ns, "no_nvml": r.no_nvml,
        "replays_before": r.replays_before, "replays_after": r.replays_after, "degraded": r.degraded,
        "path": {"bottleneck": r.path.bottleneck,
                 "hop": [{"bdf": h.bdf.decode(), "cur_speed": h.cur_speed, "cur_width": h.cur_width,
                          "max_speed": h.max_speed, "max_width": h.max_width} for h in r.path.hop]},
    }


SPEEDS = [0, 25, 50, 80, 160, 320, 640]


def make_result(cro, rng, **kw):
    r = cro.LinkResult()
    r.status = kw.get("status", 0)
    r.first_fail = kw.get("first_fail", cro.LINK_NO_FAIL)
    L = kw.get("bytes", rng.choice([16, 3 * (1 << 20) + 112, 64 << 20, 1 << 30]))
    r.bytes = L
    for g in range(cro.LINK_LEGS):
        r.leg[g].bytes = L
        r.leg[g].ns = kw.get("ns", rng.choice([0, 1, rng.randrange(1, 1 << 40)]))
    r.ce_duplex_span_ns = kw.get("span", rng.choice([0, rng.randrange(1, 1 << 40)]))
    r.chase_hops = kw.get("hops", rng.choice([0, 1, 1024, 65536]))
    r.chase_ns = rng.choice([0, rng.randrange(0, 1 << 36)])
    r.no_nvml = kw.get("no_nvml", rng.choice([0, 1]))
    r.replays_before = rng.choice([0, rng.randrange(0, 1 << 32)])
    r.replays_after = r.replays_before + rng.choice([0, 0, 1, rng.randrange(0, 1 << 20)])
    r.degraded = kw.get("degraded", rng.randrange(0, 16))
    n = rng.randrange(1, cro.PCI_MAX_HOPS + 1)
    r.path.n_hops = n
    for i in range(n):
        h = r.path.hop[i]
        h.bdf = ("0000:%02x:%02x.%x" % (rng.randrange(256), rng.randrange(32), rng.randrange(8))).encode()
        h.cur_speed, h.max_speed = rng.choice(SPEEDS), rng.choice(SPEEDS)
        h.cur_width, h.max_width = rng.choice([0, 1, 4, 8, 16]), rng.choice([0, 1, 4, 8, 16])
    r.path.bottleneck = kw.get("bottleneck", rng.randrange(0, n))
    return r


def crafted(cro):
    rng = random.Random(20261015)
    yield make_result(cro, rng, ns=0, span=0, hops=0, degraded=0)                          # zero ns everywhere
    for ck in range(cro.LINK_CHECKS):                                                          # each failing check
        yield make_result(cro, rng, status=cro.ERR_CHECKSUM, first_fail=ck)
    yield make_result(cro, rng, status=cro.ERR_CUDA)                                           # a call that failed
    for bit in (1, 2, 4, 8, 15):                                                               # every degraded flag
        yield make_result(cro, rng, degraded=bit)
    yield make_result(cro, rng, no_nvml=1)
    yield make_result(cro, rng, bottleneck=cro.PCI_MAX_HOPS, degraded=8)                      # index past the array
    for _ in range(400):
        yield make_result(cro, rng, status=rng.choice([0, 0, cro.ERR_CHECKSUM]),
                          first_fail=rng.choice([cro.LINK_NO_FAIL, cro.LINK_NO_FAIL, rng.randrange(0, 7)]))


def test_emitter_equals_the_restatement(cro):
    import link
    seen = set()
    for r in crafted(cro):
        got = cro.emit_link_annotations_json(r).encode()
        want = link.annotations_json(as_dict(r))
        assert got == want, (got, want)
        seen.add(link.annotations(as_dict(r))["cohdi.io/probe-link-verdict"])
    assert seen >= {"ok", "error"} | {"corrupt:" + n for n in link.CHECK_NAMES}


def test_emitter_spells_speeds_and_rates():
    import link
    assert link.speed_text(0) == "unknown" and link.speed_text(640) == "64.0GT/s" and link.speed_text(25) == "2.5GT/s"
    assert link.mbps(1 << 30, 0) == "0" and link.mbps(1 << 30, 1 << 30) == "1000"


def test_emitter_rejects_a_null_result(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    assert cro.lib.cro_emit_link_annotations_json(None, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


# ---- cro_pci_link_path on fake sysfs trees -------------------------------------------------------------------------
def fake_function(root, chain, links, numa=None):
    """devices/pci0000:00/<chain...> with link files per bdf (links[bdf] = (cur speed text, cur width, max speed text,
    max width), None entries are missing files), and bus/pci/devices/<bdf> symlinks into it."""
    d = root / "devices" / "pci0000:00"
    d.mkdir(parents=True, exist_ok=True)
    bus = root / "bus" / "pci" / "devices"
    bus.mkdir(parents=True, exist_ok=True)
    for bdf in chain:
        d = d / bdf
        d.mkdir(exist_ok=True)
        for name, v in zip(["current_link_speed", "current_link_width", "max_link_speed", "max_link_width"],
                           links.get(bdf, (None,) * 4)):
            if v is not None:
                (d / name).write_text("%s\n" % v)
        if numa is not None:
            (d / "numa_node").write_text("%d\n" % numa)
        link_path = bus / bdf
        if not link_path.exists():
            link_path.symlink_to(os.path.relpath(d, bus))
    return root


GEN5 = ("32.0 GT/s PCIe", 16, "32.0 GT/s PCIe", 16)


def hops_of(p):
    return [(p.hop[i].bdf.decode(), p.hop[i].cur_speed, p.hop[i].cur_width, p.hop[i].max_speed, p.hop[i].max_width)
            for i in range(p.n_hops)]


def test_direct_root_port_attach(cro, tmp_path):
    fake_function(tmp_path, ["0000:00:01.0", "0000:01:00.0"], {"0000:00:01.0": GEN5, "0000:01:00.0": GEN5}, numa=1)
    p = cro.pci_link_path("00000000:01:00.0", str(tmp_path))
    assert hops_of(p) == [("0000:01:00.0", 320, 16, 320, 16), ("0000:00:01.0", 320, 16, 320, 16)]
    assert (p.numa_node, p.bottleneck, p.truncated) == (1, 0, 0)


def test_switch_with_a_narrow_upstream_link_names_the_bottleneck(cro, tmp_path):
    import link
    chain = ["0000:00:01.0", "0000:01:00.0", "0000:02:08.0", "0000:03:00.0"]
    links = {"0000:00:01.0": ("32.0 GT/s PCIe", 4, "32.0 GT/s PCIe", 16),   # root port: the switch's upstream link
             "0000:01:00.0": ("32.0 GT/s PCIe", 4, "32.0 GT/s PCIe", 16),   # switch upstream port
             "0000:02:08.0": GEN5, "0000:03:00.0": GEN5}
    fake_function(tmp_path, chain, links, numa=0)
    p = cro.pci_link_path("0000:03:00.0", str(tmp_path))
    assert [h[0] for h in hops_of(p)] == list(reversed(chain))
    assert p.bottleneck == 2 and p.hop[2].bdf == b"0000:01:00.0" and p.hop[2].cur_width == 4
    hops = [dict(zip(["bdf", "cur_speed", "cur_width", "max_speed", "max_width"], h)) for h in hops_of(p)]
    assert link.bottleneck(hops) == p.bottleneck
    assert link.degraded(hops, p.bottleneck) == link.PATH | link.BOTTLENECK
    r = cro.LinkResult()
    r.path = p
    r.degraded = link.degraded(hops, p.bottleneck)
    r.no_nvml = 1
    ann = cro.emit_link_annotations_json(r)
    assert '"cohdi.io/probe-link-bottleneck":"0000:01:00.0 32.0GT/s x4"' in ann
    assert '"cohdi.io/probe-link-degraded":"path,bottleneck"' in ann
    assert '"cohdi.io/probe-link-link":"32.0GT/s x16 / 32.0GT/s x16"' in ann


def test_unknown_speeds_missing_files_and_no_numa_node(cro, tmp_path):
    chain = ["0000:00:03.0", "0000:40:00.0", "0000:41:00.0"]
    links = {"0000:00:03.0": ("8.0 GT/s PCIe", 16, "16.0 GT/s PCIe", None),   # root port without max_link_width
             # 0000:40:00.0 has no link files at all: not a hop
             "0000:41:00.0": ("Unknown", 16, "2.5 GT/s", 16)}
    fake_function(tmp_path, chain, links, numa=-1)
    p = cro.pci_link_path("0000:41:00.0", str(tmp_path))
    assert hops_of(p) == [("0000:41:00.0", 0, 16, 25, 16), ("0000:00:03.0", 80, 16, 160, 0)]
    assert p.numa_node == -1
    assert p.bottleneck == 1       # the device's speed is unknown: it is skipped
    import link
    hops = [dict(zip(["bdf", "cur_speed", "cur_width", "max_speed", "max_width"], h)) for h in hops_of(p)]
    assert link.degraded(hops, p.bottleneck) == link.PATH     # no device flag and no bottleneck without its speed


def test_missing_numa_file_reads_as_minus_one(cro, tmp_path):
    fake_function(tmp_path, ["0000:00:01.0", "0000:01:00.0"], {"0000:01:00.0": GEN5})
    p = cro.pci_link_path("0000:01:00.0", str(tmp_path))
    assert p.numa_node == -1 and p.n_hops == 1


def test_degraded_gpu_link(cro, tmp_path):
    import link
    fake_function(tmp_path, ["0000:00:01.0", "0000:01:00.0"],
                  {"0000:00:01.0": ("16.0 GT/s PCIe", 8, "32.0 GT/s PCIe", 16),
                   "0000:01:00.0": ("16.0 GT/s PCIe", 8, "64.0 GT/s PCIe", 16)})
    p = cro.pci_link_path("0000:01:00.0", str(tmp_path))
    hops = [dict(zip(["bdf", "cur_speed", "cur_width", "max_speed", "max_width"], h)) for h in hops_of(p)]
    assert p.hop[0].max_speed == 640
    assert link.degraded(hops, p.bottleneck) == link.SPEED | link.WIDTH | link.PATH


def test_both_bus_id_spellings_and_bad_ids(cro, tmp_path):
    fake_function(tmp_path, ["0000:00:01.0", "0000:1f:00.0"], {"0000:00:01.0": GEN5, "0000:1f:00.0": GEN5}, numa=0)
    a = cro.pci_link_path("00000000:1F:00.0", str(tmp_path))
    b = cro.pci_link_path("0000:1f:00.0", str(tmp_path))
    assert bytes(a) == bytes(b) and a.n_hops == 2
    with pytest.raises(cro.ProbeError) as e:
        cro.pci_link_path("not a bus id", str(tmp_path))
    assert e.value.code == cro.ERR_INVALID_ARG
    with pytest.raises(cro.ProbeError) as e:
        cro.pci_link_path("0000:2f:00.0", str(tmp_path))
    assert e.value.code == cro.ERR_NO_DEVICE
    assert cro.lib.cro_pci_link_path(None, None, None) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_probe_host_link_without_a_context_is_refused(cro):
    r = cro.LinkResult()
    n = ctypes.c_int(-1)
    faults = (cro.LinkFault * 4)()
    assert cro.lib.cro_probe_host_link(None, 0, None, ctypes.byref(r), faults, 4, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    o = cro.LinkOpts()
    o.bytes = 24
    assert cro.lib.cro_probe_host_link(None, 0, ctypes.byref(o), ctypes.byref(r), faults, 4, ctypes.byref(n)) == cro.ERR_INVALID_ARG
