"""Restatement of the host link probe's annotations (cro_emit_link_annotations_json) and of the PCIe path rules
(cro_pci_link_path: bottleneck and degraded flags).

Pure Python over a result given as plain values, so the emitter can be held to it without a GPU.  A result is a dict:
  {"status": int, "first_fail": int, "leg": [{"bytes": int, "ns": int}] * 8, "ce_duplex_span_ns": int,
   "chase_hops": int, "chase_ns": int, "no_nvml": int, "replays_before": int, "replays_after": int, "degraded": int,
   "path": {"bottleneck": int, "hop": [{"bdf": str, "cur_speed": int, "cur_width": int,
                                        "max_speed": int, "max_width": int}] * 8}}

Rules (include/croprobe.h): MB/s is bytes * 1000 // ns, 0 when ns is 0; the duplex rate counts both copy-engine duplex
legs over their span; latency is chase ns // hops; a speed in tenths of a GT/s prints as "<whole>.<tenth>GT/s", 0 as
"unknown".  The verdict names the first failing check, else "ok" for status 0, else "error".
"""
from __future__ import annotations

from typing import Dict, List

from oracle import go_marshal_string_map

CE_D2H, SM_H2D, CE_H2D, SM_D2H, SM_DUPLEX_H2D, SM_DUPLEX_D2H, CE_DUPLEX_H2D, CE_DUPLEX_D2H = range(8)
CHECK_NAMES = ["d2h-copy", "h2d-copy", "sm-write", "duplex-write", "duplex-d2h-copy", "chase"]
DEGRADED_NAMES = ["speed", "width", "path", "bottleneck"]
SPEED, WIDTH, PATH, BOTTLENECK = 1, 2, 4, 8
MAX_HOPS = 8
U64 = (1 << 64) - 1


def speed_text(tenths: int) -> str:
    return "unknown" if tenths == 0 else "%d.%dGT/s" % (tenths // 10, tenths % 10)


def mbps(nbytes: int, ns: int) -> str:
    return str(nbytes * 1000 // ns if ns else 0)


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-link-"
    leg = r["leg"]
    ff = r["first_fail"]
    m = {
        p + "verdict": ("corrupt:" + CHECK_NAMES[ff]) if ff < len(CHECK_NAMES) else ("ok" if r["status"] == 0 else "error"),
        p + "h2d-mbps": mbps(leg[CE_H2D]["bytes"], leg[CE_H2D]["ns"]),
        p + "d2h-mbps": mbps(leg[CE_D2H]["bytes"], leg[CE_D2H]["ns"]),
        p + "duplex-mbps": mbps(leg[CE_DUPLEX_H2D]["bytes"] + leg[CE_DUPLEX_D2H]["bytes"], r["ce_duplex_span_ns"]),
        p + "sm-h2d-mbps": mbps(leg[SM_H2D]["bytes"], leg[SM_H2D]["ns"]),
        p + "sm-d2h-mbps": mbps(leg[SM_D2H]["bytes"], leg[SM_D2H]["ns"]),
        p + "latency-ns": str(r["chase_ns"] // r["chase_hops"] if r["chase_hops"] else 0),
    }
    g = r["path"]["hop"][0]
    m[p + "link"] = "%s x%d / %s x%d" % (speed_text(g["cur_speed"]), g["cur_width"], speed_text(g["max_speed"]),
                                        g["max_width"])
    b = r["path"]["bottleneck"]
    if r["degraded"] & BOTTLENECK and b < MAX_HOPS:
        h = r["path"]["hop"][b]
        m[p + "bottleneck"] = "%s %s x%d" % (h["bdf"], speed_text(h["cur_speed"]), h["cur_width"])
    deg = [DEGRADED_NAMES[i] for i in range(4) if r["degraded"] >> i & 1]
    if deg:
        m[p + "degraded"] = ",".join(deg)
    if not r["no_nvml"]:
        m[p + "replays"] = str((r["replays_after"] - r["replays_before"]) & U64)
    return m


def annotations_json(r: Dict) -> bytes:
    """The bytes json.Marshal of the annotation map gives (keys sorted)."""
    return go_marshal_string_map(annotations(r)).encode()


def bottleneck(hops: List[Dict]) -> int:
    """Index of the least cur_speed * cur_width among hops with both known, the lowest index on a tie; 0 if none."""
    best = None
    for i, h in enumerate(hops):
        if not h["cur_speed"] or not h["cur_width"]:
            continue
        if best is None or h["cur_speed"] * h["cur_width"] < hops[best]["cur_speed"] * hops[best]["cur_width"]:
            best = i
    return 0 if best is None else best


def degraded(hops: List[Dict], bottleneck_index: int) -> int:
    """CRO_LINK_DEGRADED_* of a path whose hop 0 is the device."""
    if not hops:
        return 0
    f = 0

    def below(h, cur, mx):
        return h[cur] and h[mx] and h[cur] < h[mx]
    g = hops[0]
    if below(g, "cur_speed", "max_speed"):
        f |= SPEED
    if below(g, "cur_width", "max_width"):
        f |= WIDTH
    if any(below(h, "cur_speed", "max_speed") or below(h, "cur_width", "max_width") for h in hops[1:]):
        f |= PATH
    rate = lambda h: h["cur_speed"] * h["cur_width"]   # noqa: E731
    if rate(g) and bottleneck_index != 0 and rate(hops[bottleneck_index]) < rate(g):
        f |= BOTTLENECK
    return f
