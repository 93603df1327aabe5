"""Restatement of the register-file probe's pattern, fold closed form, classification and annotations (include/croprobe.h
"register file"; closed_form, take_regfile_round, close_regfile_call and regfile_annotations in the library).

Pure Python over plain values, so the library can be held to it without a GPU.

  word(seed, i, t, k)         P_i(t, k): the low 32 bits of pattern_word(seed + i * STRIDE, t * SLOTS + k)
  fold(seed, iterations)      the closed form of every CTA's fold: the last iteration's E1 words ~P over every thread
                              and slot, as (xor, sum, sum of v * (2k + 1)) mod 2^64
  classify(call)              the result, SM entries and sorted records of a call's rounds and records
  annotations(r)              the cohdi.io/probe-regfile-* map of a result
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import go_marshal_string_map, pattern_word, pattern_words_np

OK, ERR_CUDA, ERR_CHECKSUM, ERR_UNSUPPORTED = 0, -4, -6, -10
NONE, SM, ALL = 0, 1, 2
PERSISTENT, INTERMITTENT = 1, 2
SLOTS, THREADS, ELEMENTS, RECORDS, MAX_SMS = 224, 256, 2, 4096, 256
STRIDE = 0xD1B54A32D192ED03
SEED_OFFSET, SEEDS_PER_CALL = 1 << 56, 4096
HEALTH_NAMES = ["corrected", "uncorrected", "threshold-exceeded"]
NVML_ECC_CORRECTED, NVML_ECC_UNCORRECTED = 1, 2
U32, U64 = (1 << 32) - 1, (1 << 64) - 1


def call_seed(seed_dev: int, k: int) -> int:
    """The seed of call k on a device of seed seed_dev: iteration i of it uses call_seed + i * STRIDE."""
    return (seed_dev + SEED_OFFSET + SEEDS_PER_CALL * k * STRIDE) & U64


def iteration_seed(seed: int, i: int) -> int:
    return (seed + i * STRIDE) & U64


def word(seed: int, i: int, t: int, k: int) -> int:
    """P_i(t, k), before the complement E1 applies."""
    return pattern_word(iteration_seed(seed, i), t * SLOTS + k) & U32


def words(seed: int, i: int) -> np.ndarray:
    """P_i as a THREADS x SLOTS uint32 array."""
    return (pattern_words_np(iteration_seed(seed, i), 0, THREADS * SLOTS) & np.uint64(U32)).astype(np.uint32).reshape(THREADS, SLOTS)


def fold(seed: int, iterations: int) -> Tuple[int, int, int]:
    v = (~words(seed, iterations - 1)).astype(np.uint64)
    x = int(np.bitwise_xor.reduce(v.ravel()))
    s = int(v.sum(dtype=np.uint64))
    wt = np.arange(SLOTS, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    w = int((v * wt).sum(dtype=np.uint64))      # each product < 2^41, the sum < 2^57: no wrap
    return x, s & U64, w & U64


def _blank(call: Dict) -> Dict:
    x, s, w = fold(call["seed"], call["iterations"])
    return {"status": OK, "verdict": NONE, "seed": call["seed"], "call": call["call"], "sm_count": call["sm_count"],
            "nsmid": 0, "iterations": call["iterations"], "rounds": 0, "sms_covered": 0, "complete": 0, "ctas": 0,
            "unpublished": 0, "failed_sms": 0, "bad_sms": 0, "bad_sm": [], "mismatches": [0, 0], "fold_mismatches": 0,
            "bits_checked": 0, "timer_ns": 0, "fold": (0, 0, 0), "expect": (x, s, w)}


def classify(call: Dict) -> Tuple[Dict, List[Dict], List[Dict]]:
    """call = {"seed", "call", "iterations", "sm_count", "rounds": [[cta] * sm_count], "claims", "records": [rec]} with
    cta = {"stamp", "t0", "t1", "cycles", "count": [2], "last", "fold": (x, s, w), "smid", "nsmid"} and rec a dict of
    the cro_regfile_fault fields.  Returns (result, SM entries by smid, records sorted), or a blanked result of status
    ERR_UNSUPPORTED for a %nsmid above MAX_SMS."""
    r = _blank(call)
    per_sm: Dict[int, Dict] = {}
    last: Dict[int, int] = {}
    fold_sm = None
    for rnd in call["rounds"]:
        r["rounds"] += 1
        r["ctas"] += len(rnd)
        t0, t1 = None, 0
        for x in rnd:
            if x["stamp"] != call["call"]:
                r["unpublished"] += 1
                continue
            if x["nsmid"] > MAX_SMS:
                b = _blank(call)
                b["status"] = ERR_UNSUPPORTED
                b["expect"] = (0, 0, 0)
                return b, [], []
            r["nsmid"] = x["nsmid"]
            t0 = x["t0"] if t0 is None else min(t0, x["t0"])
            t1 = max(t1, x["t1"])
            S = per_sm.setdefault(x["smid"], {"smid": x["smid"], "mark": 0, "mismatches": [0, 0], "fold_mismatches": 0,
                                               "ns": 0, "cycles": 0, "ctas": 0})
            S["ctas"] += 1
            for e in range(ELEMENTS):
                S["mismatches"][e] = (S["mismatches"][e] + x["count"][e]) & U64
                r["mismatches"][e] = (r["mismatches"][e] + x["count"][e]) & U64
            last[x["smid"]] = (last.get(x["smid"], 0) + x["last"]) & U64
            S["ns"] = (S["ns"] + (x["t1"] - x["t0"] if x["t1"] > x["t0"] else 0)) & U64
            S["cycles"] = (S["cycles"] + x["cycles"]) & U64
            r["bits_checked"] += 32 * SLOTS * THREADS * ELEMENTS * call["iterations"]
            bad = tuple(x["fold"]) != r["expect"]
            S["fold_mismatches"] += bad
            r["fold_mismatches"] += bad
            if fold_sm is None or x["smid"] < fold_sm:
                fold_sm = x["smid"]
                r["fold"] = tuple(x["fold"])
        if t0 is not None and t1 > t0:
            r["timer_ns"] += t1 - t0
        r["sms_covered"] = len(per_sm)
    r["complete"] = int(r["sms_covered"] >= r["sm_count"])
    sms = [per_sm[s] for s in sorted(per_sm)]
    for S in sms:
        anyf = S["fold_mismatches"] + S["mismatches"][0] + S["mismatches"][1]
        S["mark"] = PERSISTENT if last[S["smid"]] else INTERMITTENT if anyf else 0
        if S["mark"]:
            r["bad_sms"] += 1
            if len(r["bad_sm"]) < 16:
                r["bad_sm"].append(S["smid"])
    r["failed_sms"] = r["bad_sms"]
    recs = sorted(call["records"][:min(call["claims"], RECORDS)],
                  key=lambda q: (q["smid"], q["iteration"], q["element"], q["warp"], q["lane"], q["slot"]))
    every = r["unpublished"] or (r["failed_sms"] and r["failed_sms"] == r["sms_covered"])
    anyf = r["unpublished"] or r["failed_sms"]
    r["verdict"] = ALL if every else SM if anyf else NONE
    r["status"] = ERR_CHECKSUM if anyf else OK
    return r, sms, recs


def annotations(r: Dict) -> Dict[str, str]:
    """r = {"status", "verdict", "cuda_error", "sms_covered", "sm_count", "bad_sms", "bad_sm" (the first min(bad_sms,
    16)), "slots", "threads", "regs_per_sm", "iterations", "health", "before", "after"}, health = {"nvml",
    "ecc_corrected", "ecc_uncorrected", ...}."""
    p = "cohdi.io/probe-regfile-"
    st = r["status"]
    names = {SM: "sm", ALL: "all"}
    if st == OK:
        verdict = "ok"
    elif st == ERR_CHECKSUM and r["verdict"] in names:
        verdict = names[r["verdict"]]
    elif st == ERR_CUDA:
        verdict = "cuda-error:%d" % r["cuda_error"]
    else:
        verdict = "error"
    m = {p + "verdict": verdict, p + "sms": "%d/%d" % (r["sms_covered"], r["sm_count"])}
    if r["bad_sms"]:
        m[p + "bad-sms"] = ",".join(str(s) for s in r["bad_sm"][:min(r["bad_sms"], 16)])
    m[p + "regs"] = "%d/%d" % (r["slots"] * r["threads"], r["regs_per_sm"])
    m[p + "iterations"] = str(r["iterations"])
    flags = [HEALTH_NAMES[b] for b in range(3) if r["health"] >> b & 1]
    if flags:
        m[p + "health"] = ",".join(flags)
    B, A = r["before"], r["after"]
    if B["nvml"] & A["nvml"] & NVML_ECC_CORRECTED:
        m[p + "ecc-corrected"] = str((A["ecc_corrected"] - B["ecc_corrected"]) & U64)
    if B["nvml"] & A["nvml"] & NVML_ECC_UNCORRECTED:
        m[p + "ecc-uncorrected"] = str((A["ecc_uncorrected"] - B["ecc_uncorrected"]) & U64)
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
