"""The host link probe (cro_probe_host_link) on one H100, against the C oracle's pattern_word, checksums and chase.

Word indices are those of the buffer a check verified: word i of it must hold pattern_word(seed, i)."""
import ctypes
import json
import os

import pytest

MASK = (1 << 64) - 1
MiB = 1 << 20
RAGGED = 3 * MiB + 112
SEED_BASE = 0x00C0FFEE00000000
STRIDE = 0xD1B54A32D192ED03
S = 256 * MiB
CHECK_PATTERN = [0, 0, 1, 2, 0]              # P1, P1, P2, P3, P1
# which checks an injection into check k's buffer reaches: H0 is copied into B before check 1 runs
REACHES = {0: {0, 1}, 1: {1}, 2: {2}, 3: {3}, 4: {4}}
HOST_BUFFER_CHECKS = {0, 2, 4}               # the injection flips a word of host memory

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=S, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


def minor_of(ctx):
    return ctx.own_devices()[0].device_minor


def seeds(ctx, k):
    dev = SEED_BASE | minor_of(ctx)
    return [(dev + (1 << 62) + (3 * k + j) * STRIDE) & MASK for j in range(3)]


# The SM legs' grids beside the default: one CTA, a few, one per SM and the most ctas takes.  At 4096 CTAs and L = 16 B
# every warp but one has nothing to do and the ragged tail does all the work.
GRID_SIZES = [(16, "16B"), (4096 + 16, "4KiB+16B"), (RAGGED, "3MiB+112B"), (64 * MiB, "64MiB")]
GRID_CTAS = [1, 7, "sm_count", 4096]
GRIDS = [(L, c, "%s-ctas%s" % (name, c)) for L, name in GRID_SIZES for c in GRID_CTAS]


def grid(ctx, ctas):
    return ctx.own_devices()[0].sm_count if ctas == "sm_count" else ctas


@pytest.mark.parametrize("L,ctas", [pytest.param(64 * MiB, 0, id="64MiB"), pytest.param(256 * MiB, 0, id="256MiB"),
                                    pytest.param(RAGGED, 0, id="3MiB+112B")] +
                         [pytest.param(L, c, id=name) for L, c, name in GRIDS])
def test_clean_call(cro, coracle, ctx, L, ctas):
    n = L // 8
    r, faults = ctx.probe_host_link(0, bytes=L, ctas=grid(ctx, ctas))
    assert r.status == cro.OK and r.first_fail == cro.LINK_NO_FAIL and faults == []
    assert r.bytes == L and list(r.seed) == seeds(ctx, r.call)
    want = [coracle.checksum(r.seed[j], 0, n, threads=16) for j in range(3)]
    for k in range(cro.LINK_WORD_CHECKS):
        c = r.check[k]
        assert (c.words, c.mismatches, c.recorded, c.seed) == (n, 0, 0, r.seed[CHECK_PATTERN[k]]), k
        assert c.fold == want[CHECK_PATTERN[k]] and c.expect == want[CHECK_PATTERN[k]], k
    for g in range(cro.LINK_LEGS):
        assert r.leg[g].bytes == L and r.leg[g].ns > 0, g
    sm_legs = {cro.LINK_LEG_SM_H2D, cro.LINK_LEG_SM_D2H, cro.LINK_LEG_SM_DUPLEX_H2D, cro.LINK_LEG_SM_DUPLEX_D2H}
    for g in range(cro.LINK_LEGS):
        assert (r.leg[g].timer_ns > 0) == (g in sm_legs), g
    assert r.ce_duplex_span_ns >= max(r.leg[cro.LINK_LEG_CE_DUPLEX_H2D].ns, r.leg[cro.LINK_LEG_CE_DUPLEX_D2H].ns)
    assert r.chase_hops == 1024 and r.chase_end == r.chase_expect == coracle.chase_end(minor_of(ctx), minor_of(ctx), 1024)
    assert r.chase_ns > 0
    ann = json.loads(cro.emit_link_annotations_json(r))
    assert ann["cohdi.io/probe-link-verdict"] == "ok"
    if L >= 4096:          # the rates are whole MB/s: 16 B in the tens of microseconds a leg takes rounds to 0
        assert int(ann["cohdi.io/probe-link-h2d-mbps"]) > 0 and int(ann["cohdi.io/probe-link-duplex-mbps"]) > 0
    r2, _ = ctx.probe_host_link(0, bytes=L, ctas=grid(ctx, ctas))
    assert r2.status == cro.OK and r2.call == r.call + 1 and not set(r2.seed) & set(r.seed)


# at the default grid and 64 MiB, every check and place; per grid of GRIDS, the last word of checks 0 and 2 (the SMs
# read a host buffer there)
@pytest.mark.parametrize("where,check,L,ctas",
                         [pytest.param(w, k, 64 * MiB, 0, id="%s-%d" % (w, k)) for w in ["first", "middle", "last"]
                          for k in range(5)] +
                         [pytest.param("last", k, L, c, id="last-%d-%s" % (k, name)) for L, c, name in GRIDS for k in (0, 2)])
def test_injected_fault_is_found_where_it_reaches(cro, coracle, ctx, where, check, L, ctas):
    n = L // 8
    word = {"first": 0, "middle": n // 2 + 3, "last": n - 1}[where]
    mask = (1 << 63) | (1 << 17) | 1
    r, faults = ctx.probe_host_link(0, bytes=L, inject=(check, word, mask), ctas=grid(ctx, ctas))
    assert r.status == cro.ERR_CHECKSUM and r.first_fail == min(REACHES[check])
    assert {f.check for f in faults} == REACHES[check], [(f.check, f.word_index) for f in faults]
    for k in range(cro.LINK_WORD_CHECKS):
        assert r.check[k].mismatches == (1 if k in REACHES[check] else 0), k
        assert r.check[k].recorded == r.check[k].mismatches
    for f in faults:
        e = coracle.pattern_word(r.seed[CHECK_PATTERN[f.check]], word)
        assert (f.word_index, f.expected, f.actual) == (word, e, e ^ mask), f.check
        assert f.host_value == (f.actual if check in HOST_BUFFER_CHECKS else f.expected), f.check
        c = r.check[f.check]
        assert c.fold_xor ^ c.expect_xor == mask                       # the fold saw exactly that word
        assert (c.fold_sum - c.expect_sum) & MASK == (f.actual - f.expected) & MASK
    ann = json.loads(cro.emit_link_annotations_json(r))
    names = ["d2h-copy", "h2d-copy", "sm-write", "duplex-write", "duplex-d2h-copy"]
    assert ann["cohdi.io/probe-link-verdict"] == "corrupt:" + names[min(REACHES[check])]


@pytest.mark.parametrize("hops", [1, 1024, 65536])
def test_chase_through_host_memory_ends_where_the_oracle_says(cro, coracle, ctx, hops):
    r, _ = ctx.probe_host_link(0, bytes=MiB, hops=hops)
    m = minor_of(ctx)
    assert r.status == cro.OK and r.chase_minor == m & 0xFFFFFFFF
    assert (r.chase_hops, r.chase_end, r.chase_expect) == (hops, coracle.chase_end(m, m, hops), coracle.chase_end(m, m, hops))


def test_probe_in_flight_stays_collectable_and_halves_are_unknown_after(cro, ctx):
    ctx.probe_begin(0)
    r, _ = ctx.probe_host_link(0, bytes=64 * MiB)
    assert r.status == cro.OK
    p = ctx.probe_end(0)
    assert p.status == cro.OK and p.checksum == p.expect
    rep, words = ctx.locate_faults(0, retest=False)
    assert rep.status == cro.OK and rep.pass_[0].halves == 0 and rep.pass_[0].skipped == 3 and words == []
    assert ctx.probe_device(0).status == cro.OK


def sysfs_bdf(bus_id):
    dom, bus, rest = bus_id.split(":")
    dev, fn = rest.split(".")
    return "%04x:%02x:%02x.%x" % (int(dom, 16), int(bus, 16), int(dev, 16), int(fn, 16))


def read(path):
    try:
        with open(path) as f:
            return f.read().strip()
    except OSError:
        return None


def speed(text):
    if not text or not text[0].isdigit():
        return 0
    num = text.split()[0]
    whole, _, frac = num.partition(".")
    return int(whole) * 10 + (int(frac[0]) if frac else 0)


LINK_FILES = ["current_link_speed", "current_link_width", "max_link_speed", "max_link_width"]


def cuda_bus_id():
    """cuda:0's PCI location from the driver API (NVML may answer "[N/A]" on a virtualised host)."""
    cu = ctypes.CDLL("libcuda.so.1")
    dev = ctypes.c_int()
    buf = ctypes.create_string_buffer(32)
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(ctypes.byref(dev), 0) == 0
    assert cu.cuDeviceGetPCIBusId(buf, 32, dev) == 0
    return buf.value.decode()


def test_path_agrees_with_sysfs(cro, ctx):
    bus_id = cuda_bus_id()
    r, _ = ctx.probe_host_link(0, bytes=64 * MiB)
    dev = os.path.join("/sys/bus/pci/devices", sysfs_bdf(bus_id))
    if not os.path.isdir(dev):
        assert r.path.n_hops == 0 and r.dev_numa == -1
        return
    real = os.path.realpath(dev)
    hops = 1
    d = os.path.dirname(real)
    while ":" in os.path.basename(d) and not os.path.basename(d).startswith("pci"):
        if any(os.path.exists(os.path.join(d, f)) for f in LINK_FILES):
            hops += 1
        d = os.path.dirname(d)
    assert r.path.n_hops == min(hops, cro.PCI_MAX_HOPS)
    assert r.path.hop[0].bdf.decode() == sysfs_bdf(bus_id)
    assert r.path.hop[0].max_speed == speed(read(os.path.join(dev, "max_link_speed")))
    mw = read(os.path.join(dev, "max_link_width"))
    assert r.path.hop[0].max_width == (int(mw) if mw and mw.isdigit() else 0)
    numa = read(os.path.join(dev, "numa_node"))
    assert r.dev_numa == r.path.numa_node == (int(numa) if numa is not None else -1)
    p = cro.pci_link_path(bus_id)                     # the context-free reader, default /sys
    assert (p.n_hops, p.hop[0].max_speed, p.hop[0].max_width) == (r.path.n_hops, r.path.hop[0].max_speed, r.path.hop[0].max_width)


def nvml_replays_answer(uuid):
    try:
        nv = ctypes.CDLL("libnvidia-ml.so.1")
        get = nv.nvmlDeviceGetPcieReplayCounter
    except (OSError, AttributeError):
        return False
    if nv.nvmlInit_v2() != 0:
        return False
    h = ctypes.c_void_p()
    v = ctypes.c_uint()
    ok = nv.nvmlDeviceGetHandleByUUID(uuid, ctypes.byref(h)) == 0 and get(h, ctypes.byref(v)) == 0
    nv.nvmlShutdown()
    return ok


def test_replay_counter_is_present_when_nvml_is(cro, ctx):
    r, _ = ctx.probe_host_link(0, bytes=16 * MiB)
    uuid = ctx.own_devices()[0].gpu_uuid
    if nvml_replays_answer(uuid):
        assert r.no_nvml == 0 and r.replays_after >= r.replays_before
        assert "cohdi.io/probe-link-replays" in json.loads(cro.emit_link_annotations_json(r))
    else:
        assert r.no_nvml == 1
    with cro.ProbeContext(sweep_bytes=64 * MiB, devices=[0], flags=cro.F_NO_NVML) as c2:
        r2, _ = c2.probe_host_link(0, bytes=MiB)
        assert r2.status == cro.OK and r2.no_nvml == 1 and r2.replays_before == r2.replays_after == 0


@pytest.mark.parametrize("kw", [dict(bytes=8), dict(bytes=24), dict(bytes=S + 16), dict(bytes=2 * S),
                                dict(hops=(1 << 24) + 1), dict(inject=(5, 0, 1)), dict(inject=(-1, 0, 1)),
                                dict(bytes=MiB, inject=(0, MiB // 8, 1))],
                         ids=["8B", "24B", "S+16", "2S", "hops", "check5", "check-1", "word-past-L"])
def test_invalid_arguments_are_refused(cro, ctx, kw):
    with pytest.raises(cro.ProbeError) as e:
        ctx.probe_host_link(0, **kw)
    assert e.value.code == cro.ERR_INVALID_ARG


def test_bad_dev_index_is_refused(cro, ctx):
    with pytest.raises(cro.ProbeError) as e:
        ctx.probe_host_link(5, bytes=MiB)
    assert e.value.code == cro.ERR_INVALID_ARG
