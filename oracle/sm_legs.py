"""Restatement of the per-SM arithmetic probes' classification (cro_probe_compute, cro_probe_precision): what each round's
CTA records add to a leg and to its SMs, the marks, the slowest SM, the verdict, the bad-SM list and the fault order.

Written from include/croprobe.h ("SM compute", cro_compute_leg, cro_compute_sm_leg, cro_compute_result and
cro_selftest_sm_legs_classify), not from csrc/sm_legs.hpp.  oracle/compute.py and oracle/precision.py give it their leg
counts and operation counts; everything is plain Python over dicts.

A call is a dict:
  {"legs": int (0: all), "iterations": [int] * n_legs, "grid": int, "call": int,
   "rounds": per leg, [(ctas, bits)] with ctas a list of grid CTA dicts (stamp, t0, t1, cycles, mismatches,
             fold_mismatches, fold, smid, nsmid) and bits the leg's coverage bitmap words after the round,
   "claims": [int] * n_legs, "records": per leg, the fault dicts the device kept (leg, smid, row, col, ...)}
classify() returns (result, sms, faults) as dicts shaped like the C structs.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

OK, ERR_CHECKSUM, ERR_UNSUPPORTED = 0, -6, -10
NONE, SM, ALL = 0, 1, 2
PERSISTENT, INTERMITTENT = 1, 2
MAX_SMS, MAX_BAD_SMS = 256, 16
U64 = (1 << 64) - 1
U32 = (1 << 32) - 1

LEG_FIELDS = ("iterations", "rounds", "ops", "ns", "timer_ns", "sms_covered", "complete", "mismatches", "fold_mismatches",
              "recorded", "failed_sms", "unpublished", "ctas", "slowest_sm", "slow_permille", "reserved", "fold",
              "expect_fold")
SM_LEG_FIELDS = ("mismatches", "fold_mismatches", "ns", "cycles", "ctas", "mark")


def blank(n_legs: int, call: int = 0, sm_count: int = 0, legs: int = 0) -> Dict:
    """A result of zeroes but for the call number, SM count and legs."""
    return {"status": OK, "verdict": NONE, "seed": 0, "call": call, "sm_count": sm_count, "legs": legs, "host_ref_ns": 0,
            "nsmid": 0, "bad_sms": 0, "bad_sm": [0] * MAX_BAD_SMS, "leg": [dict.fromkeys(LEG_FIELDS, 0) for _ in range(n_legs)]}


def median(values: Sequence[int]) -> int:
    """The (n / 2)-th of n values sorted ascending, from 0: the upper median for an even n."""
    v = sorted(values)
    return v[len(v) // 2]


def slowest(per_iter: Dict[int, int]) -> Tuple[int, int]:
    """(slowest SM, slow_permille) over {smid: cycles per iteration}: the most cycles, the lowest SM id on a tie, against
    the median (0 when the median is 0)."""
    worst = min(per_iter, key=lambda s: (-per_iter[s], s))
    m = median(list(per_iter.values()))
    return worst, (min(per_iter[worst] * 1000 // m, U32) if m else 0)


def classify(call: Dict, n_legs: int, ops_per_iteration: Sequence[int], max_records: int) -> Tuple[Dict, List[Dict], List[Dict]]:
    """The result, the SM list (by SM id) and the faults (by leg, smid, row, col) the probe reports for `call`."""
    legs = call["legs"] or (1 << n_legs) - 1
    grid, k = call["grid"], call["call"]
    r = blank(n_legs, k, grid, legs)
    per_sm: Dict[int, Dict] = {}
    faults: List[Dict] = []
    for leg in range(n_legs):
        if not legs >> leg & 1:
            continue
        R = r["leg"][leg]
        it = call["iterations"][leg]
        R["iterations"] = it
        fold_sm = None
        for ctas, bits in call["rounds"][leg]:
            R["rounds"] += 1
            R["ctas"] += grid
            R["ops"] = (R["ops"] + ops_per_iteration[leg] * it * grid) & U64
            t0, t1 = None, None
            for x in ctas:
                if x["stamp"] != k:
                    R["unpublished"] += 1
                    continue
                if x["nsmid"] > MAX_SMS:                    # more SM ids than the bitmaps hold: nothing is reported
                    out = blank(n_legs, k, grid, legs)
                    out["status"] = ERR_UNSUPPORTED
                    return out, [], []
                r["nsmid"] = x["nsmid"]
                t0 = x["t0"] if t0 is None else min(t0, x["t0"])
                t1 = x["t1"] if t1 is None else max(t1, x["t1"])
                s = per_sm.setdefault(x["smid"], {"smid": x["smid"], "reserved": 0,
                                                  "leg": [dict.fromkeys(SM_LEG_FIELDS, 0) for _ in range(n_legs)]})
                SL = s["leg"][leg]
                SL["ctas"] += 1
                SL["mismatches"] = (SL["mismatches"] + x["mismatches"]) & U64
                SL["fold_mismatches"] = (SL["fold_mismatches"] + x["fold_mismatches"]) & U64
                SL["ns"] = (SL["ns"] + max(x["t1"] - x["t0"], 0)) & U64
                SL["cycles"] = (SL["cycles"] + x["cycles"]) & U64
                R["mismatches"] = (R["mismatches"] + x["mismatches"]) & U64
                R["fold_mismatches"] = (R["fold_mismatches"] + x["fold_mismatches"]) & U64
                if fold_sm is None or x["smid"] < fold_sm:  # the first CTA to publish on the lowest SM id
                    fold_sm, R["fold"] = x["smid"], x["fold"]
            if t0 is not None and t1 > t0:
                R["timer_ns"] = (R["timer_ns"] + t1 - t0) & U64
            R["sms_covered"] = sum(bin(w).count("1") for w in bits)
        R["complete"] = 1 if R["sms_covered"] >= grid else 0
        R["recorded"] = min(call["claims"][leg], max_records)
        faults.extend(call["records"][leg][:R["recorded"]])
        per_iter = {}
        for smid in sorted(per_sm):
            SL = per_sm[smid]["leg"][leg]
            if not SL["ctas"]:
                continue
            SL["mark"] = PERSISTENT if SL["mismatches"] else INTERMITTENT if SL["fold_mismatches"] else 0
            R["failed_sms"] += 1 if SL["mark"] else 0
            per_iter[smid] = SL["cycles"] // (SL["ctas"] * it)
        if per_iter:
            R["slowest_sm"], R["slow_permille"] = slowest(per_iter)
    ran = [r["leg"][l] for l in range(n_legs) if legs >> l & 1]
    every = any(R["unpublished"] or (R["failed_sms"] and R["failed_sms"] == R["sms_covered"]) for R in ran)
    some = any(R["unpublished"] or R["failed_sms"] for R in ran)
    sms = [per_sm[s] for s in sorted(per_sm)]
    bad = [s["smid"] for s in sms if any(SL["mark"] for SL in s["leg"])]
    r["bad_sms"] = len(bad)
    r["bad_sm"] = (bad[:MAX_BAD_SMS] + [0] * MAX_BAD_SMS)[:MAX_BAD_SMS]
    faults.sort(key=lambda f: (f["leg"], f["smid"], f["row"], f["col"]))
    r["verdict"] = ALL if every else SM if some else NONE
    r["status"] = ERR_CHECKSUM if some else OK
    return r, sms, faults
