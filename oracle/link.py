"""Restatement of the host link probe's annotations (cro_emit_link_annotations_json), of the PCIe path rules
(cro_pci_link_path: bottleneck and degraded flags) and of the word checks' and the chase's verdict (classify,
cro_selftest_link_classify).

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

from typing import Callable, Dict, List, Tuple

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


CHECK_PATTERN = [0, 0, 1, 2, 0]     # P1, P1, P2, P3, P1: the pattern word check k's buffer must hold
WORD_CHECKS, CHECK_CHASE, NO_FAIL, RECORDS = 5, 5, 0xFFFFFFFF, 4096
SLOT_EXPECT = WORD_CHECKS + 2       # slots: [k] check k's fold, the two write roles, then the closed forms of P1..P3
OK, ERR_CHECKSUM = 0, -6


def classify(call: Dict, chase_end: Callable[[int, int, int], int]) -> Tuple[Dict, List[Dict]]:
    """The word checks' and the chase's part of the result, and the faults, that cro_probe_host_link makes of what its
    kernels wrote (cro_selftest_link_classify).  call: {"bytes", "seeds": [3], "minor", "hops", "counters": [5 x
    {"mismatches", "claims"}], "records": [5 x [{"word", "expected", "actual"}]] (the first min(claims, RECORDS) of
    each check), "host": [5 x [L / 8 words]], "slots": [10 slots {"x", "s", "w", "n_words", ...}], "chase_out": [end,
    ns], "cap"}.  chase_end(minor_src, minor_dst, hops): the host walk of the latency permutation.

    From include/croprobe.h: check k must hold pattern_word(seed, i) for its pattern's seed over L / 8 words; it fails
    when it counted a mismatch, or its fold or closed form covered another number of words, or its fold is not the
    closed form.  The chase fails when it did not end on the host walk's slot (an armed output, all ones, never does
    and reports no time).  first_fail is the lowest failing check.  The faults run by check, then word index, and
    host_value is word word_index of the host buffer the check involved, 0 past L / 8."""
    n = call["bytes"] // 8
    first_fail = NO_FAIL
    checks, found = [], []
    for k in range(WORD_CHECKS):
        c, recs = call["counters"][k], call["records"][k]
        assert len(recs) == min(c["claims"], RECORDS)
        s, cf = call["slots"][k], call["slots"][SLOT_EXPECT + CHECK_PATTERN[k]]
        checks.append(dict(words=n, mismatches=c["mismatches"], recorded=len(recs), seed=call["seeds"][CHECK_PATTERN[k]],
                           fold_xor=s["x"], fold_sum=s["s"], fold_wsum=s["w"], expect_xor=cf["x"], expect_sum=cf["s"],
                           expect_wsum=cf["w"]))
        bad = c["mismatches"] != 0 or s["n_words"] != n or cf["n_words"] != n or (s["x"], s["s"], s["w"]) != (
            cf["x"], cf["s"], cf["w"])
        if bad and first_fail == NO_FAIL:
            first_fail = k
        found += [dict(check=k, reserved=0, word_index=r["word"], expected=r["expected"], actual=r["actual"],
                       host_value=call["host"][k][r["word"]] if r["word"] < n else 0)
                  for r in sorted(recs, key=lambda r: r["word"])]
    expect = chase_end(call["minor"], call["minor"], call["hops"])
    end, ns = call["chase_out"]
    if end != expect and first_fail == NO_FAIL:
        first_fail = CHECK_CHASE
    r = dict(status=OK if first_fail == NO_FAIL else ERR_CHECKSUM, first_fail=first_fail, bytes=call["bytes"],
             seed=list(call["seeds"]), check=checks, chase_hops=call["hops"], chase_end=end & 0xFFFFFFFF,
             chase_expect=expect, chase_minor=call["minor"], chase_ns=0 if end == U64 else ns)
    return r, found[:call["cap"]]


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
