"""Restatement of the fault locator's verdict and annotations (cro_locate_faults, cro_emit_fault_annotations_json).

Pure Python over a report given as plain values, so the emitter can be held to it without a GPU.  A report is a dict:
  {"n_passes": int, "pass": [{"mismatches": int, "granules": int}, ...], "bit_flips": [64 ints]}
and words a list of (word_index, expected, actual).

Verdict rule (include/croprobe.h, CRO_FAULTS_*): a retest pass (1 or 2) that ran and found a mismatch makes the
faults persistent; otherwise mismatches in pass 0 are "not reproduced" when a retest ran and "unclassified" when none
did; no mismatch anywhere is "none".  Only the first min(n_passes, 3) passes count.

collect() restates the report cro_locate_faults makes from what its compare kernels wrote (cro_selftest_locate_collect).
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

from oracle import checksum_np, go_marshal_string_map, pattern_word

PASSES = 3
RECORDS = 4096
OK, ERR_CHECKSUM = 0, -6
U64 = (1 << 64) - 1
NONE, UNCLASSIFIED, NOT_REPRODUCED, PERSISTENT = 0, 1, 2, 3


def complement_fold(f: Tuple[int, int, int], n: int) -> Tuple[int, int, int]:
    """The closed form of the complement of a pattern over n words from the pattern's: ~p = -1 - p, and the weights
    2i + 1 of n words sum to n^2."""
    return f[0] ^ (U64 if n & 1 else 0), (-n - f[1]) & U64, (-n * n - f[2]) & U64


def deltas(records, index) -> Tuple[int, int, int]:
    """What the records change in a fold: xor, sum and weighted sum of actual - expected, each record at the position
    index(word) of its own sweep."""
    dx = ds = dw = 0
    for r in records:
        d = (r["actual"] - r["expected"]) & U64
        dx ^= r["actual"] ^ r["expected"]
        ds = (ds + d) & U64
        dw = (dw + d * (2 * index(r["word"]) + 1)) & U64
    return dx, ds, dw


# ---- faults in a pattern region, seen by the fold and word by word ----------------------------------------------------
# A fault is (first, count, and_mask, or_mask, xor_mask): words [first, first + count) of the region become
# ((w & and_mask) | or_mask) ^ xor_mask.  The probe's test hooks place exactly these: an XOR run (CRO_F_TEST_INJECT,
# CRO_SELFTEST_F_XOR) and a stuck-at run (the and / or force).
def xor_run(first: int, mask: int, count: int = 1) -> Tuple[int, int, int, int, int]:
    return (first, count, U64, 0, mask)


def stuck_run(first: int, count: int, bit: int, value: int) -> Tuple[int, int, int, int, int]:
    """Bit `bit` of every word of the run stuck at `value` (0 or 1)."""
    return (first, count, U64 ^ (1 << bit), value << bit, 0)


def fault_records(seed: int, faults) -> List[Dict]:
    """The words the faults change in the pattern of `seed` (word i = pattern_word(seed, i)), applied in list order,
    each to the word as the earlier ones left it: one {"word", "expected", "actual"} per word that ends up differing."""
    now = {}
    for first, count, and_mask, or_mask, xor_mask in faults:
        for i in range(first, first + count):
            w = now.get(i, pattern_word(seed, i))
            now[i] = ((w & and_mask) | or_mask) ^ xor_mask
    recs = [dict(word=i, expected=pattern_word(seed, i), actual=a) for i, a in sorted(now.items())]
    return [r for r in recs if r["actual"] != r["expected"]]


def faulted_fold(seed: int, n_words: int, faults) -> Tuple[int, int, int]:
    """The fold (xor, sum, weighted sum) of words [0, n_words) of the pattern with the faults applied."""
    x, s, w = checksum_np(seed, 0, n_words)
    dx, ds, dw = deltas([r for r in fault_records(seed, faults) if r["word"] < n_words], lambda i: i)
    return x ^ dx, (s + ds) & U64, (w + dw) & U64


def word_mismatches(seed: int, n_words: int, faults) -> int:
    """What a word-by-word compare of words [0, n_words) counts."""
    return sum(1 for r in fault_records(seed, faults) if r["word"] < n_words)


def flip_direction(seed: int, i: int, bit: int) -> int:
    """+1 when flipping bit `bit` of pattern word i adds 2^bit to it (the bit is 0), -1 when it subtracts."""
    return -1 if pattern_word(seed, i) >> bit & 1 else 1


def find_directions(seed: int, bit: int, dirs: Sequence[int], start: int = 0, stride: int = 1, limit: int = 1 << 16) -> int:
    """The first a >= start, below start + limit, at which flipping bit `bit` of words a, a + stride, a + 2 stride, ...
    goes in the directions dirs (+1 / -1 each).  XOR runs placed there take the fold-blind shapes of DESIGN.md §3."""
    for a in range(start, start + limit):
        if all(flip_direction(seed, a + m * stride, bit) == d for m, d in enumerate(dirs)):
            return a
    raise ValueError("no run of directions %s for bit %d in [%d, %d)" % (list(dirs), bit, start, start + limit))


def explained(slot: Dict, cf: Tuple[int, int, int], d: Tuple[int, int, int]) -> bool:
    """The fold in `slot` is the closed form cf changed by exactly the deltas d."""
    return (slot["x"] ^ cf[0], (slot["s"] - cf[1]) & U64, (slot["w"] - cf[2]) & U64) == d


def merge(records_by_pass, chunk_of=lambda w: 0) -> List[Dict]:
    """Every recorded word once, by index: expected and actual from the first record of it (in pass order), bit p of
    passes for each pass that recorded it, reserved = chunk_of(word)."""
    words = {}
    for p, recs in enumerate(records_by_pass):
        for r in recs:
            w = words.setdefault(r["word"], dict(word_index=r["word"], expected=r["expected"], actual=r["actual"], passes=0,
                                                 reserved=chunk_of(r["word"])))
            w["passes"] |= 1 << p
    return [words[k] for k in sorted(words)]


def collect(call: Dict) -> Tuple[Dict, List[Dict]]:
    """The report and word list cro_locate_faults makes of its passes.  call: {"sweep_bytes", "passes": [{"halves",
    "skipped", "seed": [2], "invert"}] (one per pass), "counters": [{"mismatches", "claims", "bits": [64]}],
    "records": [[{"word", "expected", "actual"}]] (the first min(claims, RECORDS) of each pass), "granules": [[words]],
    "slots": [9 slots {"x", "s", "w", "t0", "t1", "n_words", ...}], "cap"}.

    From include/croprobe.h: half h of the region holds words [h * n, (h + 1) * n), n = S / 8, and word i of a half
    is compared with pattern_word(seed[h], i) ^ invert.  The device's slots are [2p + h] for the compare of half h in
    pass p, then one closed form per distinct seed of a compared half, in pass then half order; a pass with invert
    compares against the complement's closed form.  complete: every pass recorded all its mismatches, each compared
    half's fold differs from its closed form by exactly its records' deltas (weights from the half's start), and the
    caller's list holds every located word."""
    n = call["sweep_bytes"] // 8
    np_ = len(call["passes"])
    seeds = []
    for P in call["passes"]:
        for h in range(2):
            if P["halves"] >> h & 1 and P["seed"][h] not in seeds:
                seeds.append(P["seed"][h])
    complete = True
    bit_flips = [0] * 64
    passes = []
    for p, (P, c, recs) in enumerate(zip(call["passes"], call["counters"], call["records"])):
        recorded = min(c["claims"], RECORDS)
        assert len(recs) == recorded
        complete &= recorded == c["mismatches"]
        bit_flips = [(a + b) & U64 for a, b in zip(bit_flips, c["bits"])]
        out = dict(halves=P["halves"], skipped=P["skipped"], seed=list(P["seed"]), invert=P["invert"], words_scanned=0,
                   mismatches=c["mismatches"], recorded=recorded, granules=sum(bin(g).count("1") for g in call["granules"][p]),
                   scan_ns=0, fold_xor=[0, 0], fold_sum=[0, 0], fold_wsum=[0, 0])
        for h in range(2):
            if not P["halves"] >> h & 1:
                continue
            s = call["slots"][2 * p + h]
            out["words_scanned"] = (out["words_scanned"] + s["n_words"]) & U64
            out["scan_ns"] = (out["scan_ns"] + s["t1"] - s["t0"]) & U64
            out["fold_xor"][h], out["fold_sum"][h], out["fold_wsum"][h] = s["x"], s["s"], s["w"]
            c_ = call["slots"][2 * PASSES + seeds.index(P["seed"][h])]
            cf = (c_["x"], c_["s"], c_["w"])
            if P["invert"]:
                cf = complement_fold(cf, n)
            mine = [r for r in recs if (r["word"] >= n) == (h == 1)]
            complete &= explained(s, cf, deltas(mine, lambda w: w - h * n))
        passes.append(out)
    blank = dict(halves=0, skipped=0, seed=[0, 0], invert=0, words_scanned=0, mismatches=0, recorded=0, granules=0,
                 scan_ns=0, fold_xor=[0, 0], fold_sum=[0, 0], fold_wsum=[0, 0])
    passes += [dict(blank) for _ in range(PASSES - np_)]
    words = merge(call["records"])
    listed = words[:call["cap"]]
    r = dict(status=ERR_CHECKSUM if any(P["mismatches"] for P in passes[:np_]) else OK, n_passes=np_,
             complete=int(complete and len(listed) == len(words)), sweep_bytes=call["sweep_bytes"], retest_seed=0,
             located=len(words), recorded=len(listed), flip_or=sum(1 << b for b in range(64) if bit_flips[b]),
             bit_flips=bit_flips, pass_=passes)
    r["verdict"] = verdict(dict(n_passes=np_, **{"pass": passes}))
    return r, listed
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
