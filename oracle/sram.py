"""Restatement of the SRAM probe's health bits, annotations and M5 closed form (sram_health,
cro_emit_sram_annotations_json, closed_form in sram_probe.cu).

Pure Python over a result given as plain values, so the emitter can be held to it without a GPU.  A result is a dict:
  {"status": int, "verdict": int, "cuda_error": int, "sm_count": int, "legs": int, "bytes_per_sm": int, "health": int,
   "sms_covered": [int] * 2, "bad_sm": [int] (the first min(bad_sms, 16)), "bad_sms": int,
   "bad_pair": [(from, owner, direction)] (the first min(bad_pairs, 8)), "bad_pairs": int, "before": health,
   "after": health}
with health = {"nvml": int, "threshold_exceeded": int, "ecc_corrected": int, "ecc_uncorrected": int}.

classify() restates the probe's classification of a call's rounds and records (cro_selftest_sram_classify).

Rules (include/croprobe.h, "SRAM"): the verdict is "ok" for status 0, "sm" / "link" / "all" for CRO_ERR_CHECKSUM with
that verdict, "cuda-error:<cuda_error>" for CRO_ERR_CUDA, else "error"; -sms is the least coverage over the legs run;
an ECC delta prints only when both reads answered it (it wraps mod 2^64).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Tuple

from oracle import go_marshal_string_map

OK, ERR_CUDA, ERR_CHECKSUM = 0, -4, -6
NONE, SM, LINK, ALL = 0, 1, 2, 3
DIR_LOCAL, DIR_READ, DIR_WRITE = 0, 1, 2
ERR_UNSUPPORTED = -10
SMEM, DSMEM, LEGS, ELEMENTS, RECORDS, MAX_SMS, MAX_PAIRS = 0, 1, 2, 6, 4096, 256, 8
PERSISTENT, INTERMITTENT = 1, 2
SILENT = 0xFFFFFFFF
CORRECTED_DURING, UNCORRECTED_DURING, THRESHOLD_EXCEEDED = 1, 2, 4
HEALTH_NAMES = ["corrected", "uncorrected", "threshold-exceeded"]
NVML_ECC_CORRECTED, NVML_ECC_UNCORRECTED, NVML_STATUS = 1, 2, 4
U64 = (1 << 64) - 1


def health_bits(before: Dict, after: Dict) -> int:
    """CRO_SRAM_HEALTH_* of the NVML reads before the first leg and after the last."""
    h = 0
    both = before["nvml"] & after["nvml"]
    if both & NVML_ECC_CORRECTED and after["ecc_corrected"] > before["ecc_corrected"]:
        h |= CORRECTED_DURING
    if both & NVML_ECC_UNCORRECTED and after["ecc_uncorrected"] > before["ecc_uncorrected"]:
        h |= UNCORRECTED_DURING
    if after["nvml"] & NVML_STATUS and after["threshold_exceeded"]:
        h |= THRESHOLD_EXCEEDED
    return h


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-sram-"
    st = r["status"]
    names = {SM: "sm", LINK: "link", ALL: "all"}
    if st == OK:
        verdict = "ok"
    elif st == ERR_CHECKSUM and r["verdict"] in names:
        verdict = names[r["verdict"]]
    elif st == ERR_CUDA:
        verdict = "cuda-error:%d" % r["cuda_error"]
    else:
        verdict = "error"
    m = {p + "verdict": verdict}
    run = [r["sms_covered"][leg] for leg in range(2) if r["legs"] >> leg & 1]
    m[p + "sms"] = "%d/%d" % (min(run) if run else 0, r["sm_count"])
    if r["bad_sms"]:
        m[p + "bad-sms"] = ",".join(str(s) for s in r["bad_sm"][:min(r["bad_sms"], 16)])
    if r["bad_pairs"]:
        m[p + "bad-pairs"] = ",".join("%d-%d:%s" % (f, o, "r" if d == DIR_READ else "w")
                                      for f, o, d in r["bad_pair"][:min(r["bad_pairs"], 8)])
    m[p + "bytes-per-sm"] = str(r["bytes_per_sm"])
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


def m5_fold(checksum, seed: int, n_words: int, iterations: int) -> Tuple[int, int, int]:
    """The fold every CTA of the local leg publishes: M5 reads pattern_word(seed, 0 .. n_words) once per iteration, the
    iterations' xors xored and sums summed.  `checksum` is the C oracle's (COracle().checksum)."""
    x, s, w = checksum(seed, 0, n_words)
    return (x if iterations % 2 else 0, s * iterations & U64, w * iterations & U64)


LEG_FIELDS = ("iterations", "rounds", "bytes", "ns", "timer_ns", "sms_covered", "complete", "mismatches", "fold_mismatches",
              "recorded", "failed_sms", "unpublished", "ctas", "cluster", "fold_xor", "fold_sum", "fold_wsum", "expect_xor",
              "expect_sum", "expect_wsum")


def _blank(call: Dict, legs: int) -> Dict:
    leg = []
    for _ in range(LEGS):
        L = dict.fromkeys(LEG_FIELDS, 0)
        L["mismatches"] = [0] * ELEMENTS
        leg.append(L)
    return {"status": OK, "verdict": NONE, "seed": call["seed"], "call": call["call"], "sm_count": call["sm_count"],
            "legs": legs, "nsmid": 0, "bytes_per_sm": 8 * call["n_words"], "bad_sms": 0, "bad_sm": [0] * 16, "bad_pairs": 0,
            "bad_pair": [(0, 0, 0)] * MAX_PAIRS, "leg": leg}


def classify(call: Dict, checksum: Callable) -> Tuple[Dict, List[Dict], List[Dict]]:
    """The result, the SM list (by SM id) and the faults (by leg, element, smid, iteration, word) the SRAM probe reports
    for a call given as
      {"legs": int (0: both), "iterations": int, "n_words": int, "seed": int, "cluster": int, "sm_count": int,
       "net_grid": int, "call": int, "rounds": per leg, a list of rounds, each a list of CTA dicts (stamp, t0, t1,
       cycles, count[6], last, fold_x, fold_s, fold_w, smid, nsmid, rank, block), "claims": [int] * 2,
       "records": per leg, the record dicts the device kept (element, iteration, smid, peer_block, round, word,
       expected, actual)}.
    `checksum` is the C oracle's (COracle().checksum), for the local leg's M5 closed form (m5_fold)."""
    legs = call["legs"] or 3
    k, it, n_words, cluster = call["call"], call["iterations"], call["n_words"], call["cluster"]
    r = _blank(call, legs)
    per_sm: Dict[int, Dict] = {}
    last = [dict(), dict()]                       # per leg and SM: failed compares of the last iteration
    block_smid: List[List[int]] = []              # network leg, per round: blockIdx.x -> %smid (SILENT: no record)
    kept: List[List[Dict]] = [[], []]
    for leg in range(LEGS):
        if not legs >> leg & 1:
            continue
        net = leg == DSMEM
        L = r["leg"][leg]
        L["iterations"], L["cluster"] = it, cluster if net else 0
        if not net:
            L["expect_xor"], L["expect_sum"], L["expect_wsum"] = m5_fold(checksum, call["seed"], n_words, it)
        moved = 8 * n_words * it * (cluster + 2 if net else 10)
        grid = call["net_grid"] if net else call["sm_count"]
        seen, fold_sm = set(), None
        for ctas in call["rounds"][leg]:
            L["rounds"] += 1
            L["ctas"] += grid
            L["bytes"] = (L["bytes"] + moved * grid) & U64
            if net:
                block_smid.append([SILENT] * grid)
            t0, t1 = None, None
            for j, x in enumerate(ctas):
                if x["stamp"] != k:
                    L["unpublished"] += 1
                    continue
                if x["nsmid"] > MAX_SMS:
                    out = _blank(call, legs)
                    out["status"] = ERR_UNSUPPORTED
                    return out, [], []
                r["nsmid"] = x["nsmid"]
                t0 = x["t0"] if t0 is None else min(t0, x["t0"])
                t1 = x["t1"] if t1 is None else max(t1, x["t1"])
                if net:
                    block_smid[-1][j] = x["smid"]
                seen.add(x["smid"])
                s = per_sm.setdefault(x["smid"], {"smid": x["smid"], "reserved": 0, "leg": [
                    {"mismatches": [0] * ELEMENTS, "fold_mismatches": 0, "ns": 0, "cycles": 0, "ctas": 0, "mark": 0}
                    for _ in range(LEGS)]})
                SL = s["leg"][leg]
                SL["ctas"] += 1
                for e in range(ELEMENTS):
                    SL["mismatches"][e] = (SL["mismatches"][e] + x["count"][e]) & U64
                    L["mismatches"][e] = (L["mismatches"][e] + x["count"][e]) & U64
                last[leg][x["smid"]] = (last[leg].get(x["smid"], 0) + x["last"]) & U64
                SL["ns"] = (SL["ns"] + max(x["t1"] - x["t0"], 0)) & U64
                SL["cycles"] = (SL["cycles"] + x["cycles"]) & U64
                if net:
                    continue
                bad = (x["fold_x"], x["fold_s"], x["fold_w"]) != (L["expect_xor"], L["expect_sum"], L["expect_wsum"])
                SL["fold_mismatches"] += bad
                L["fold_mismatches"] += bad
                if fold_sm is None or x["smid"] < fold_sm:
                    fold_sm = x["smid"]
                    L["fold_xor"], L["fold_sum"], L["fold_wsum"] = x["fold_x"], x["fold_s"], x["fold_w"]
            if t0 is not None and t1 > t0:
                L["timer_ns"] = (L["timer_ns"] + t1 - t0) & U64
            L["sms_covered"] = len(seen)
        L["complete"] = 1 if L["sms_covered"] >= call["sm_count"] else 0
        L["recorded"] = min(call["claims"][leg], RECORDS)
        kept[leg] = call["records"][leg][:L["recorded"]]
        for smid in sorted(per_sm):
            SL = per_sm[smid]["leg"][leg]
            if not SL["ctas"]:
                continue
            failed = SL["fold_mismatches"] + sum(SL["mismatches"])
            SL["mark"] = PERSISTENT if last[leg].get(smid) else INTERMITTENT if failed else 0
            L["failed_sms"] += 1 if SL["mark"] else 0

    faults = []
    for leg in range(LEGS):
        for q in kept[leg]:
            f = {"leg": leg, "element": q["element"], "iteration": q["iteration"], "smid": q["smid"], "word": q["word"],
                 "reserved": 0, "expected": q["expected"], "actual": q["actual"]}
            if leg == SMEM:
                f["peer_smid"], f["direction"] = q["smid"], DIR_LOCAL
            else:
                f["direction"] = DIR_READ if q["element"] == 1 else DIR_WRITE
                known = q["round"] < len(block_smid) and q["peer_block"] < len(block_smid[q["round"]])
                f["peer_smid"] = block_smid[q["round"]][q["peer_block"]] if known else SILENT
            faults.append(f)
    faults.sort(key=lambda f: (f["leg"], f["element"], f["smid"], f["iteration"], f["word"]))

    sms = [per_sm[s] for s in sorted(per_sm)]
    local_bad = [s["smid"] for s in sms if s["leg"][SMEM]["mark"]]
    pairs = set()
    for f in faults:
        if f["leg"] != DSMEM or f["smid"] in local_bad or f["peer_smid"] in local_bad:
            continue
        reader_or_writer = f["smid"] if f["direction"] == DIR_READ else f["peer_smid"]
        owner = f["peer_smid"] if f["direction"] == DIR_READ else f["smid"]
        pairs.add((f["direction"], reader_or_writer, owner))
    pairs = sorted(pairs)
    ran = [r["leg"][l] for l in range(LEGS) if legs >> l & 1]
    every = any(L["unpublished"] or (L["failed_sms"] and L["failed_sms"] == L["sms_covered"]) for L in ran)
    some = any(L["unpublished"] or L["failed_sms"] for L in ran)
    r["bad_sms"] = len(local_bad)
    r["bad_sm"] = (local_bad[:16] + [0] * 16)[:16]
    r["bad_pairs"] = len(pairs)
    listed = [(a & 0xFFFF, o & 0xFFFF, d) for d, a, o in pairs[:MAX_PAIRS]]
    r["bad_pair"] = (listed + [(0, 0, 0)] * MAX_PAIRS)[:MAX_PAIRS]
    r["verdict"] = ALL if every else SM if local_bad else LINK if some else NONE
    r["status"] = ERR_CHECKSUM if some else OK
    return r, sms, faults
