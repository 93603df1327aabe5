"""Host restatement of the probe's device-side verdict: what probe_finalize and p2p_finalize must write into the
512-byte cro_probe_result, from the rules include/croprobe.h and DESIGN.md §4-§5 state.

Pure Python on integers of any size: every 64-bit field is reduced modulo 2^64 where the rule says so, and nothing
here imports the product.  Inputs are the same bytes the kernels see: the identity template (512 bytes) and slot
arrays of SLOT_COUNT 64-byte slots (x, s, w, t0, t1, stamp, n_words, pad, little-endian u64 each).
"""
from __future__ import annotations

import struct
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

MASK64 = (1 << 64) - 1
MAX_DEVICES = 16

# slot map (croprobe.h, CRO_SLOT_*)
SLOT_FILL, SLOT_SWEEP0, MAX_SWEEPS_EACH, SLOT_EXPECT, SLOT_PREFIX, SLOT_P2P0 = 0, 1, 30, 62, 63, 64
SLOT_COUNT = SLOT_P2P0 + 3 * MAX_DEVICES + 4

OK, ERR_CHECKSUM = 0, -6
FAIL_NONE, FAIL_EXPECT, FAIL_COPY_SRC, FAIL_READ, FAIL_P2P_READ, FAIL_P2P_PUSH, FAIL_P2P_CHASE, FAIL_STALE = range(8)
COPY_TMA_FUSED = 3

# cro_probe_result: (name, offset, struct format), in declaration order
FIELDS: List[Tuple[str, int, str]] = [
    ("abi_version", 0, "<I"), ("status", 4, "<i"), ("cuda_ordinal", 8, "<i"), ("device_minor", 12, "<i"),
    ("gpu_uuid", 16, "48s"), ("pci_bus_id", 64, "24s"), ("hbm_bytes_total", 88, "<Q"), ("sweep_bytes", 96, "<Q"),
    ("seed", 104, "<Q"), ("checksum_xor", 112, "<Q"), ("checksum_sum", 120, "<Q"), ("fill_ns", 128, "<Q"),
    ("read_best_ns", 136, "<Q"), ("read_median_ns", 144, "<Q"), ("copy_best_ns", 152, "<Q"),
    ("copy_median_ns", 160, "<Q"), ("sm_count", 168, "<I"), ("sm_clock_mhz", 172, "<I"), ("mem_clock_mhz", 176, "<I"),
    ("ecc_errors", 180, "<I"), ("p2p_read_ns", 184, "<8Q"), ("p2p_checksum_xor", 248, "<8Q"),
    ("p2p_latency_ns_x16", 312, "<8I"), ("p2p_access", 344, "<8B"), ("p2p_bytes", 352, "<Q"),
    ("expect_xor", 360, "<Q"), ("expect_sum", 368, "<Q"), ("expect_wsum", 376, "<Q"), ("checksum_wsum", 384, "<Q"),
    ("copy_checksum_xor", 392, "<Q"), ("copy_checksum_sum", 400, "<Q"), ("copy_checksum_wsum", 408, "<Q"),
    ("total_ns", 416, "<Q"), ("p2p_write_ns", 424, "<8Q"), ("nonce", 488, "<I"), ("rank", 492, "<B"),
    ("world", 493, "<B"), ("read_variant", 494, "<B"), ("copy_variant", 495, "<B"), ("read_sweeps", 496, "<B"),
    ("copy_sweeps", 497, "<B"), ("copy_verified", 498, "<B"), ("fail_code", 499, "<B"), ("fail_index", 500, "<B"),
    ("p2p_ok", 501, "<B"), ("reserved8", 502, "<2B"), ("t_start_ns", 504, "<Q"),
]
_FIELD = {name: (off, fmt) for name, off, fmt in FIELDS}
RESULT_BYTES = 512


class Slot(NamedTuple):
    x: int = 0
    s: int = 0
    w: int = 0
    t0: int = 0
    t1: int = 0
    stamp: int = 0
    n_words: int = 0
    pad: int = 0

    def fold(self) -> Tuple[int, int, int]:
        return (self.x, self.s, self.w)


ARMED = Slot(*([MASK64] * 8))      # what an unwritten slot holds: the probe sets every byte to 0xFF at init


def pack_slots(slots: Sequence[Slot]) -> bytes:
    assert len(slots) == SLOT_COUNT
    return b"".join(struct.pack("<8Q", *(v & MASK64 for v in s)) for s in slots)


def unpack_slots(raw: bytes) -> List[Slot]:
    return [Slot(*struct.unpack_from("<8Q", raw, 64 * i)) for i in range(len(raw) // 64)]


class Result:
    """A cro_probe_result as 512 mutable bytes with named access."""

    def __init__(self, raw: bytes) -> None:
        assert len(raw) == RESULT_BYTES
        self.raw = bytearray(raw)

    def get(self, name: str):
        off, fmt = _FIELD[name]
        v = struct.unpack_from(fmt, self.raw, off)
        return v[0] if len(v) == 1 else list(v)

    def set(self, name: str, value) -> None:
        off, fmt = _FIELD[name]
        if isinstance(value, (list, tuple)):
            struct.pack_into(fmt, self.raw, off, *value)
        elif fmt.endswith(("s", "i")):
            struct.pack_into(fmt, self.raw, off, value)
        else:                             # unsigned fields keep the low bits, as the C assignment does
            struct.pack_into(fmt, self.raw, off, value & ((1 << (8 * struct.calcsize(fmt))) - 1))

    def set_at(self, name: str, j: int, value: int) -> None:
        v = self.get(name)
        v[j] = value
        self.set(name, v)

    def bytes(self) -> bytes:
        return bytes(self.raw)


def diff_fields(a: bytes, b: bytes) -> Dict[str, Tuple[object, object]]:
    """{field: (a's value, b's value)} for every field the two structs disagree on."""
    ra, rb = Result(a), Result(b)
    return {name: (ra.get(name), rb.get(name)) for name, _, _ in FIELDS if ra.get(name) != rb.get(name)}


def best_and_median(times: Sequence[int]) -> Tuple[int, int]:
    """best = the minimum, median = sorted[n // 2] (the upper median for an even count); 0, 0 for no sweeps."""
    if not times:
        return 0, 0
    v = sorted(times)
    return v[0], v[len(v) // 2]


def probe_finalize(tmpl: bytes, slots: Sequence[Slot], seed: int, nonce: int, sweep_bytes: int, read_sweeps: int,
                   copy_sweeps: int, read_variant: int, copy_variant: int) -> bytes:
    """The struct probe_finalize writes.  copy_variant is the resolved variant of the copy sweeps; the struct reports
    it only when copies ran."""
    R, C = read_sweeps, copy_sweeps
    assert 0 <= R <= MAX_SWEEPS_EACH and 0 <= C <= MAX_SWEEPS_EACH
    r = Result(tmpl)                      # every field the verdict does not own passes through
    n_words = sweep_bytes >> 3
    fused = copy_variant == COPY_TMA_FUSED
    E, F = slots[SLOT_EXPECT], slots[SLOT_FILL]
    state = {"status": OK, "code": FAIL_NONE, "index": 0}

    def fail(code: int, index: int) -> None:  # the first failure wins
        if state["status"] == OK:
            state.update(status=ERR_CHECKSUM, code=code, index=index)

    def stale(s: Slot) -> bool:
        return s.stamp != nonce or s.n_words != n_words

    r.set("seed", seed)
    r.set("nonce", nonce)
    r.set("sweep_bytes", sweep_bytes)
    r.set("read_sweeps", R)
    r.set("copy_sweeps", C)
    r.set("read_variant", read_variant)
    r.set("copy_variant", copy_variant if C else 0)
    r.set("expect_xor", E.x)
    r.set("expect_sum", E.s)
    r.set("expect_wsum", E.w)
    if stale(E):
        fail(FAIL_EXPECT, 0)
    if stale(F):
        fail(FAIL_STALE, 0)
    verified = 0
    copy_times = []
    for i in range(C):                    # launch-order number of copy i is 1 + i
        s = slots[SLOT_SWEEP0 + i]
        copy_times.append((s.t1 - s.t0) & MASK64)
        if stale(s):
            fail(FAIL_STALE, 1 + i)
        elif fused:
            if s.fold() != E.fold():
                fail(FAIL_COPY_SRC, i)
            elif i > 0:
                verified += 1             # copy i folded copy i-1's destination and it matched
    shown = slots[SLOT_SWEEP0 + C]        # read sweep 0
    read_times = []
    for i in range(R):                    # launch-order number of read i is 1 + C + i
        s = slots[SLOT_SWEEP0 + C + i]
        read_times.append((s.t1 - s.t0) & MASK64)
        ok = True
        if stale(s) or s.fold() != E.fold():
            if state["status"] == OK:
                shown = s                 # the struct shows the read that failed first
            fail(FAIL_STALE if stale(s) else FAIL_READ, 1 + C + i if stale(s) else i)
            ok = False
        if i == 0 and ok and C > 0:
            verified += 1                 # read 0 folded the last copy's destination
    r.set("checksum_xor", shown.x)
    r.set("checksum_sum", shown.s)
    r.set("checksum_wsum", shown.w)
    if C > 0 and R > 0:
        d = slots[SLOT_SWEEP0 + C]
        r.set("copy_checksum_xor", d.x)
        r.set("copy_checksum_sum", d.s)
        r.set("copy_checksum_wsum", d.w)
    r.set("copy_verified", verified)
    r.set("fill_ns", (F.t1 - F.t0) & MASK64)
    best, med = best_and_median(read_times)
    r.set("read_best_ns", best)
    r.set("read_median_ns", med)
    best, med = best_and_median(copy_times)
    r.set("copy_best_ns", best)
    r.set("copy_median_ns", med)
    t_end = max([F.t1] + [slots[SLOT_SWEEP0 + i].t1 for i in range(C + R)])
    r.set("t_start_ns", F.t0)
    r.set("total_ns", (t_end - F.t0) & MASK64)
    r.set("fail_code", state["code"])
    r.set("fail_index", state["index"])
    r.set("status", state["status"])
    return r.bytes()


def latency_x16(ns: int, hops: int) -> int:
    """Mean hop latency x16, saturated to the 32-bit field."""
    return min(ns * 16 // hops, 0xFFFFFFFF)


def p2p_finalize(result: bytes, slots: Sequence[Slot], peer_slots: Sequence[Optional[Sequence[Slot]]],
                 peer_stamp: Sequence[int], chase_out: Sequence[int], chase_expect: Sequence[int], n: int, self_index: int,
                 hops: int, have_push: bool, push_folded: bool, p2p_bytes: int, stamp: int) -> bytes:
    """The struct p2p_finalize leaves: `result` as probe_finalize wrote it, updated with the NVLink checks of every
    peer j < min(n, 8) that is not this device, is reachable (p2p_access[j]) and has a slot array."""
    r = Result(result)
    state = {"status": r.get("status"), "code": r.get("fail_code"), "index": r.get("fail_index")}

    def fail(code: int, index: int) -> None:  # an earlier failure (HBM or another peer) wins
        if state["status"] == OK:
            state.update(status=ERR_CHECKSUM, code=code, index=index)

    access = r.get("p2p_access")
    ok_mask = 0
    r.set("p2p_bytes", p2p_bytes)
    for j in range(min(n, 8)):
        if j == self_index or not access[j] or peer_slots[j] is None:
            continue
        ok = True
        rd = slots[SLOT_P2P0 + 3 * j]                 # my read of j's prefix
        want = peer_slots[j][SLOT_PREFIX]             # j's own closed form of that prefix
        r.set_at("p2p_read_ns", j, (rd.t1 - rd.t0) & MASK64)
        r.set_at("p2p_checksum_xor", j, rd.x)
        if want.stamp != peer_stamp[j] or want.n_words != p2p_bytes >> 3:
            fail(FAIL_EXPECT, j)
            ok = False
        if rd.stamp != stamp or rd.fold() != want.fold():
            fail(FAIL_P2P_READ, j)
            ok = False
        ps = slots[SLOT_P2P0 + 3 * j + 1]             # my push into j
        if ps.stamp == stamp:
            r.set_at("p2p_write_ns", j, (ps.t1 - ps.t0) & MASK64)
        if have_push:
            rr = slots[SLOT_P2P0 + 3 * j + 2]         # my re-read of what j pushed into me
            if push_folded and (ps.stamp != stamp or ps.fold() != slots[SLOT_PREFIX].fold()):
                fail(FAIL_P2P_PUSH, j)
                ok = False
            if rr.stamp != stamp or rr.fold() != want.fold():
                fail(FAIL_P2P_PUSH, j)
                ok = False
        if hops:
            end, ns = chase_out[2 * j], chase_out[2 * j + 1]
            r.set_at("p2p_latency_ns_x16", j, latency_x16(ns, hops))
            if end != chase_expect[j]:
                fail(FAIL_P2P_CHASE, j)
                ok = False
        if ok:
            ok_mask |= 1 << j
    r.set("p2p_ok", ok_mask)
    r.set("fail_code", state["code"])
    r.set("fail_index", state["index"])
    r.set("status", state["status"])
    return r.bytes()
