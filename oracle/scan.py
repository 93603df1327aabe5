"""Restatement of the whole-HBM scan's verdict, health bits and annotations (cro_scan_hbm, scan_health,
cro_emit_scan_annotations_json), and of what a stuck-at force does to the scan's two compare passes.

Pure Python over a report given as plain values, so the emitter can be held to it without a GPU.  A report is a dict:
  {"status": int, "cuda_error": int, "health": int, "seed": int, "covered_bytes": int, "free_bytes": int,
   "element_ns": [int] * 4, "pass": [{"mismatches": int, "granules": int, "bit_flips": [int] * 64}] * 2,
   "before": health, "after": health}
with health = {"nvml": int, "ecc_corrected": int, "ecc_uncorrected": int, "remap_corrected": int,
               "remap_uncorrected": int, "remap_pending": int, "remap_failure": int, "histogram": [int] * 5}

Rules (include/croprobe.h, "whole-HBM scan"): the verdict is "ok" for status 0, "corrupt" for CRO_ERR_CHECKSUM,
"cuda-error:<cuda_error>" for CRO_ERR_CUDA, else "error"; GB/s is 4 * covered_bytes // (sum of element ns), 0 when that
sum is 0; an NVML field prints only when the read that fills it answered (both reads for a delta, which wraps mod 2^64).
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np

from oracle import go_marshal_string_map, pattern_words_np

OK, ERR_CUDA, ERR_CHECKSUM = 0, -4, -6
ECC_CORRECTED_DURING, ECC_UNCORRECTED_DURING, REMAP_PENDING, REMAP_FAILURE = 1, 2, 4, 8
HEALTH_NAMES = ["ecc-corrected", "ecc-uncorrected", "remap-pending", "remap-failure"]
NVML_ECC_CORRECTED, NVML_ECC_UNCORRECTED, NVML_REMAP, NVML_HISTOGRAM = 1, 2, 4, 8
GRANULE_BYTES = 2 << 20
U64 = (1 << 64) - 1


def health_bits(before: Dict, after: Dict) -> int:
    """CRO_SCAN_HEALTH_* of the NVML reads before E0 and after E3."""
    h = 0
    both = before["nvml"] & after["nvml"]
    if both & NVML_ECC_CORRECTED and after["ecc_corrected"] > before["ecc_corrected"]:
        h |= ECC_CORRECTED_DURING
    if both & NVML_ECC_UNCORRECTED and after["ecc_uncorrected"] > before["ecc_uncorrected"]:
        h |= ECC_UNCORRECTED_DURING
    r = after if after["nvml"] & NVML_REMAP else before      # the latest remap state NVML gave
    if r["nvml"] & NVML_REMAP and r["remap_pending"]:
        h |= REMAP_PENDING
    if r["nvml"] & NVML_REMAP and r["remap_failure"]:
        h |= REMAP_FAILURE
    return h


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/hbm-scan-"
    st = r["status"]
    m = {p + "verdict": "ok" if st == OK else "corrupt" if st == ERR_CHECKSUM else
         "cuda-error:%d" % r["cuda_error"] if st == ERR_CUDA else "error"}
    m[p + "covered-bytes"] = str(r["covered_bytes"])
    m[p + "free-bytes"] = str(r["free_bytes"])
    m[p + "seed"] = "%016x" % r["seed"]
    m[p + "mismatches"] = "%d,%d" % (r["pass"][0]["mismatches"], r["pass"][1]["mismatches"])
    m[p + "granules"] = "%d,%d" % (r["pass"][0]["granules"], r["pass"][1]["granules"])
    ns = sum(r["element_ns"]) & U64
    m[p + "gbs"] = str(r["covered_bytes"] * 4 // ns if ns else 0)
    bits = [b for b in range(64) if r["pass"][0]["bit_flips"][b] or r["pass"][1]["bit_flips"][b]]
    if bits:
        m[p + "bits"] = ",".join(map(str, bits))
    names = [HEALTH_NAMES[b] for b in range(4) if r["health"] >> b & 1]
    if names:
        m[p + "health"] = ",".join(names)
    B, A = r["before"], r["after"]
    if B["nvml"] & A["nvml"] & NVML_ECC_CORRECTED:
        m[p + "ecc-corrected"] = str((A["ecc_corrected"] - B["ecc_corrected"]) & U64)
    if B["nvml"] & A["nvml"] & NVML_ECC_UNCORRECTED:
        m[p + "ecc-uncorrected"] = str((A["ecc_uncorrected"] - B["ecc_uncorrected"]) & U64)
    if A["nvml"] & NVML_REMAP:
        m[p + "remapped"] = "%d,%d" % (A["remap_corrected"], A["remap_uncorrected"])
    if A["nvml"] & NVML_HISTOGRAM:
        m[p + "remap-histogram"] = ",".join(map(str, A["histogram"]))
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")


def forced_mismatches(seed: int, first: int, count: int, and_mask: int, or_mask: int) -> List[Dict]:
    """What the scan's two compare passes see in scan words [first, first + count) forced to (w & and) | or after each
    fill: per pass (0 against P, 1 against ~P) the mismatching words as {"word", "expected", "actual"}, the exact count,
    the bit-flip counters and the 2 MiB granules touched."""
    words = pattern_words_np(seed, first, count)
    out = []
    for inv in (np.uint64(0), np.uint64(U64)):
        exp = words ^ inv
        act = (exp & np.uint64(and_mask)) | np.uint64(or_mask)
        bad = np.nonzero(exp != act)[0]
        d = exp[bad] ^ act[bad]
        flips = [int(((d >> np.uint64(b)) & np.uint64(1)).sum()) for b in range(64)]
        idx = bad.astype(np.uint64) + np.uint64(first)
        out.append({"mismatches": int(bad.size), "bit_flips": flips,
                    "granules": len(set((int(i) * 8) // GRANULE_BYTES for i in idx)),
                    "words": [{"word": int(i), "expected": int(e), "actual": int(a)}
                              for i, e, a in zip(idx, exp[bad], act[bad])]})
    return out
