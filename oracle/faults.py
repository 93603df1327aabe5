"""Restatement of the fault locator's verdict and annotations (cro_locate_faults, cro_emit_fault_annotations_json).

Pure Python over a report given as plain values, so the emitter can be held to it without a GPU.  A report is a dict:
  {"n_passes": int, "pass": [{"mismatches": int, "granules": int}, ...], "bit_flips": [64 ints]}
and words a list of (word_index, expected, actual).

Verdict rule (include/croprobe.h, CRO_FAULTS_*): a retest pass (1 or 2) that ran and found a mismatch makes the
faults persistent; otherwise mismatches in pass 0 are "not reproduced" when a retest ran and "unclassified" when none
did; no mismatch anywhere is "none".  Only the first min(n_passes, 3) passes count.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

from oracle import go_marshal_string_map

PASSES = 3
NONE, UNCLASSIFIED, NOT_REPRODUCED, PERSISTENT = 0, 1, 2, 3
VERDICT_TEXT = {NONE: "none", UNCLASSIFIED: "unclassified", NOT_REPRODUCED: "not-reproduced", PERSISTENT: "persistent"}
WORDS_SHOWN = 8


def verdict(report: Dict) -> int:
    np_ = min(report["n_passes"], PASSES)
    if any(report["pass"][p]["mismatches"] for p in range(1, np_)):
        return PERSISTENT
    if np_ == 0 or report["pass"][0]["mismatches"] == 0:
        return NONE
    return NOT_REPRODUCED if np_ > 1 else UNCLASSIFIED


def annotations(report: Dict, words: Sequence[Tuple[int, int, int]]) -> Dict[str, str]:
    np_ = min(report["n_passes"], PASSES)
    m = {
        "cohdi.io/probe-fault-verdict": VERDICT_TEXT[verdict(report)],
        "cohdi.io/probe-fault-mismatches": ",".join("%d:%d" % (p, report["pass"][p]["mismatches"]) for p in range(np_)),
        "cohdi.io/probe-fault-granules": ",".join("%d:%d" % (p, report["pass"][p]["granules"]) for p in range(np_)),
    }
    bits = [str(b) for b in range(64) if report["bit_flips"][b]]
    if bits:
        m["cohdi.io/probe-fault-bits"] = ",".join(bits)
    if words:
        m["cohdi.io/probe-fault-words"] = ",".join("%x:%016x" % (w, e ^ a) for w, e, a in words[:WORDS_SHOWN])
    return m


def annotations_json(report: Dict, words: Sequence[Tuple[int, int, int]]) -> bytes:
    """The bytes json.Marshal of the annotation map gives (keys sorted)."""
    return go_marshal_string_map(annotations(report, words)).encode()
