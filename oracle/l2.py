"""Restatement of the L2 probe (cro_probe_l2, l2_kernels.cu, l2_probe.cu): its rotation map, the words each element
reads and writes, A1's closed forms, the classification and the annotation emitter.

Pure Python (numpy for A1) over plain values, so the library can be held to it without a GPU.

A result for `classify` and `annotations` is a dict with the cro_l2_result fields they read:
  {"status", "verdict", "cuda_error", "sm_count", "sms_covered", "unpublished", "fold_ok", "mismatches" (6 ints),
   "overflow", "bytes", "iterations", "march_bytes", "march_ns", "health", "bad_sms", "bad_sm" (the first 16),
   "bad_lines", "bad_line" (the first 8), "a1_bad", "a2_bad", "a2_holes", "a1_bad_counter" (8), "a2_bad_counter" (8)}
An SM entry is {"smid", "mismatches" (6 ints), "last", "words_read" (6 ints)}; a record {"element", "iteration", "smid", "word"}.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import go_marshal_string_map

OK, ERR_CUDA, ERR_CHECKSUM = 0, -4, -6
NONE, SM, LINE, ATOMIC, ALL = 0, 1, 2, 3, 4
PERSISTENT, INTERMITTENT = 1, 2
BLOCK_WORDS = 16384 // 8
HEALTH_NAMES = ["sram-corrected", "sram-uncorrected", "l2-corrected", "l2-uncorrected", "threshold-exceeded", "l2-bucket"]
STRIDE = 0xD1B54A32D192ED03
U64 = (1 << 64) - 1


def pattern(seed: int, i: int) -> int:
    z = (seed + i + 0x9E3779B97F4A7C15) & U64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & U64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & U64
    return z ^ (z >> 31)


def delta(G: int) -> int:
    """The rotation step: 0 when G < 5 (no step puts M1 .. M5 of a word on five CTAs)."""
    return 0 if G < 5 else G // 5


def owner(block: int, element: int, G: int) -> int:
    """The CTA that handles `block` in `element`."""
    return (block + element * delta(G)) % G


def blocks_of(cta: int, element: int, blocks: int, G: int) -> List[int]:
    return [b for b in range(blocks) if owner(b, element, G) == cta]


def words_read(cta: int, element: int, blocks: int, G: int) -> int:
    """Words CTA `cta` reads in `element` (0 for M0, which reads nothing)."""
    return 0 if element == 0 else len(blocks_of(cta, element, blocks, G)) * BLOCK_WORDS


def expected_read(seed: int, element: int, w: int) -> int:
    """What element 1 .. 5 reads at word w: P in M1, M3, M5 and Q = ~P in M2, M4."""
    p = pattern(seed, w)
    return p ^ U64 if element in (2, 4) else p


def written(seed: int, element: int, w: int) -> int:
    """What element 0 .. 4 writes at word w: P in M0, M2, M4 and Q in M1, M3."""
    p = pattern(seed, w)
    return p ^ U64 if element in (1, 3) else p


def m5_fold(checksum, seed: int, n_words: int, iterations: int) -> Tuple[int, int, int]:
    """The CTAs' M5 folds combined: `iterations` times the checksum (the C oracle's COracle().checksum) of
    pattern_word(seed, 0 .. n_words)."""
    x, s, w = checksum(seed, 0, n_words)
    return (x if iterations % 2 else 0, s * iterations & U64, w * iterations & U64)


def _pattern_np(seed: int, idx: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + idx + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def a1_counters(seed_atomic: int, n: int, G: int) -> Tuple[np.ndarray, np.ndarray]:
    """(sum, xor) every A1 counter i < n ends at: over CTAs j < G of pattern_word(seed_atomic, j * n + i)."""
    i = np.arange(n, dtype=np.uint64)
    s = np.zeros(n, dtype=np.uint64)
    x = np.zeros(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for j in range(G):
            v = _pattern_np(seed_atomic, np.uint64(j * n) + i)
            s += v
            x ^= v
    return s, x


def classify(r: Dict, sms: List[Dict], faults: List[Dict]) -> Dict:
    """verdict, status, bad_sms, bad_sm, bad_lines, bad_line, the SMs' marks (by smid) and the records' line flags.

    `all` (a common cause) when a CTA did not publish, when every SM that read words in an element where a read went
    wrong saw a wrong word itself, when the fold failed with every compare passing, or when mismatches were counted but
    none recorded."""
    readers: Dict[int, set] = {}
    for f in faults:
        readers.setdefault(f["word"], set()).add(f["smid"])
    lines = sorted(w for w, s in readers.items() if len(s) >= 2)
    bad = sorted({next(iter(s)) for s in readers.values() if len(s) == 1})
    failed_el = [any(s["mismatches"][e] for s in sms) for e in range(6)]
    total = sum(sum(s["mismatches"]) for s in sms)
    every, marks = total > 0, {}
    for s in sms:
        any_ = sum(s["mismatches"])
        if any(failed_el[e] and s["words_read"][e] for e in range(6)) and not any_:
            every = False          # it read in an element where a read went wrong, and read everything right
        marks[s["smid"]] = PERSISTENT if s["last"] else INTERMITTENT if any_ else 0
    all_ = r["unpublished"] > 0 or every or (not r["fold_ok"] and r["mismatches"][5] == 0) or (total > 0 and not faults)
    verdict = ALL if all_ else LINE if lines else SM if bad else ATOMIC if (r["a1_bad"] or r["a2_bad"]) else NONE
    return {"verdict": verdict, "status": OK if verdict == NONE else ERR_CHECKSUM, "bad_sms": len(bad),
            "bad_sm": (bad[:16] + [0] * 16)[:16], "bad_lines": len(lines),
            "bad_line": ([8 * w for w in lines[:8]] + [0] * 8)[:8], "marks": marks,
            "line": [1 if len(readers[f["word"]]) >= 2 else 0 for f in faults]}


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-l2-"
    names = {SM: "sm", LINE: "line", ATOMIC: "atomic", ALL: "all"}
    st = r["status"]
    if st == OK:
        verdict = "ok"
    elif st == ERR_CHECKSUM and r["verdict"] in names:
        verdict = names[r["verdict"]]
    elif st == ERR_CUDA:
        verdict = "cuda-error:%d" % r["cuda_error"]
    else:
        verdict = "error"
    m = {p + "verdict": verdict, p + "sms": "%d/%d" % (r["sms_covered"], r["sm_count"]), p + "bytes": str(r["bytes"]),
         p + "iterations": str(r["iterations"]),
         p + "march-gbs": str(r["march_bytes"] // r["march_ns"] if r["march_ns"] else 0)}
    if r["bad_sms"]:
        m[p + "bad-sms"] = ",".join(str(s) for s in r["bad_sm"][:min(r["bad_sms"], 16)])
    if r["bad_lines"]:
        m[p + "bad-lines"] = ",".join(str(o) for o in r["bad_line"][:min(r["bad_lines"], 8)])
    if r["a1_bad"]:
        m[p + "a1-bad-counters"] = ",".join(str(c) for c in r["a1_bad_counter"][:min(r["a1_bad"], 8)])
    if r["a2_bad"]:
        m[p + "a2-bad-counters"] = ",".join(str(c) for c in r["a2_bad_counter"][:min(r["a2_bad"], 8)])
    if r["a2_holes"]:
        m[p + "a2-holes"] = str(r["a2_holes"])
    if r["overflow"]:
        m[p + "overflow"] = "1"
    flags = [HEALTH_NAMES[b] for b in range(6) if r["health"] >> b & 1]
    if flags:
        m[p + "health"] = ",".join(flags)
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
