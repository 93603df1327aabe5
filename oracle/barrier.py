"""Restatement of the barrier probe (cro_probe_barrier): the call's table from the seed, every check each thread makes
in the device's order (with what a clean run reads), the fold's closed form, the records an injection makes, and the
classification and annotations (the cross-lane probe's, three legs, and the LINK pairs)."""
from __future__ import annotations

from typing import Dict, List, Tuple

from oracle import go_marshal_string_map, pattern_word

U64 = (1 << 64) - 1
M32 = 0xFFFFFFFF
LEGS, THREADS, WARPS = 3, 256, 8
BAR, MBAR, CLUSTER = range(3)
OPS = [64, 8, 17]
NAMES = ["bar", "mbar", "cluster"]
STRIDE = 0xD1B54A32D192ED03
SEED_OFFSET = 1 << 52
CBAR_ROWS = 2
(POPC, AND, OR, ARRIVE, TICKET, COUNT, DROP, TX, CBAR, ST_B32, ST_B64, ST_V2, ST_V4, RED_ADD, RED_ADD64, RED_MIN, RED_MAX,
 RED_MINS, RED_MAXS, RED_AND, RED_OR, RED_XOR, RED_INC, RED_DEC) = range(24)
VALUE, EARLY, TICKET_KIND, TIMEOUT = range(4)
NONE, SM, ALL, LINK = 0, 1, 2, 3


def call_seed(seed_dev: int, k: int) -> int:
    return (seed_dev + SEED_OFFSET + k * STRIDE) & U64


def word(seed, leg, row, k, t):
    return pattern_word(seed, ((((leg * 256 + row) * 4 + k) << 8) | t) & U64)


def warp_order(seed, leg, row):
    perm = list(range(8))
    for i in range(7, 0, -1):
        j = word(seed, leg, row, 2, i) % (i + 1)
        perm[i], perm[j] = perm[j], perm[i]
    return perm


def mask_of(perm, a, b):
    return sum(1 << perm[i] for i in range(a, b))


def members(warps):
    return [t for t in range(THREADS) if warps >> (t >> 5) & 1]


def s32(x):
    x &= M32
    return x - (1 << 32) if x >> 31 else x


def blank_row():
    return {"form": 0, "bar": 0, "count": 0, "warps": 0, "producers": 0, "phases": 0, "held": 0, "arriver": 0, "expect": 0,
            "pred": [0] * 8, "next_rank": [0] * 8, "slot_init": [0] * 8, "slot_expect": [0] * 8}


def row(leg, seed, r, cluster=2):
    """(row dict, words[thread] = [w0, w1]) of row r of leg."""
    R, w = blank_row(), [[0, 0] for _ in range(THREADS)]
    if leg == BAR:
        perm = warp_order(seed, leg, r)
        R["form"], R["bar"] = POPC + r // 16, r % 16
        if R["form"] == ARRIVE:
            nw = 2 + r % 7
            np_ = 1 + word(seed, leg, r, 3, 1) % (nw - 1)
            R["producers"], R["warps"], R["count"] = mask_of(perm, 0, np_), mask_of(perm, np_, nw), 32 * nw
            for t in members(R["producers"]):
                w[t][0] = (word(seed, leg, r, 0, t) & 0xFFFFFF00) | (r + 1)
            return R, w
        nw = 1 + r % 8
        R["warps"], R["count"] = mask_of(perm, 0, nw), 32 * nw
        kind = r % 5
        one = members(R["warps"])[word(seed, leg, r, 3, 0) % R["count"]]
        ones = 0
        for t in members(R["warps"]):
            p = [1, 0, int(t == one), int(t != one), word(seed, leg, r, 1, t) & 1][kind]
            R["pred"][t >> 5] |= p << (t & 31)
            ones += p
        R["expect"] = ones if R["form"] == POPC else int(ones == R["count"]) if R["form"] == AND else int(ones > 0)
        return R, w
    if leg == MBAR:
        perm = warp_order(seed, leg, r)
        R["form"] = TICKET + r // 2
        nw = 1 + word(seed, leg, r, 3, 0) % 8
        n = 32 * nw
        R["warps"] = mask_of(perm, 0, nw)
        part = members(R["warps"])
        R["held"] = part[word(seed, leg, r, 3, 1) % n]
        R["phases"] = 1
        if R["form"] == TICKET:
            R["held"], R["count"] = word(seed, leg, r, 3, 1) % THREADS, n + 1
        elif R["form"] == COUNT:
            R["phases"] = 2 + word(seed, leg, r, 3, 2) % 7
            for t in part:
                w[t][0] = 1 + word(seed, leg, r, 0, t) % 4
                R["count"] += w[t][0]
        elif R["form"] == DROP:
            R["phases"], R["count"] = 2, n
            for t in part:
                if t != R["held"]:
                    w[t][0] = word(seed, leg, r, 0, t) & 1
        else:
            R["phases"] = 1 + word(seed, leg, r, 3, 2) % 4
            R["count"], R["arriver"] = 1, word(seed, leg, r, 3, 3) % THREADS
            for t in part:
                w[t][0] = 1 + word(seed, leg, r, 0, t) % 64
                R["expect"] += w[t][0]
        return R, w
    R["form"] = CBAR if r < CBAR_ROWS else ST_B32 + (r - CBAR_ROWS)
    f = R["form"]
    if f == CBAR:
        R["next_rank"] = [(k + 1) % cluster if k < cluster else 0 for k in range(8)]
        for t in range(THREADS):
            w[t][0] = (word(seed, CLUSTER, r, 0, t) & 0xFFFFFF00) | (r + 1)
        return R, w
    if f <= ST_V4:
        R["count"] = THREADS * [4, 8, 8, 16][f - ST_B32]
        for t in range(THREADS):
            a, b = word(seed, CLUSTER, r, 0, t), word(seed, CLUSTER, r, 1, t)
            w[t] = [a & M32 if f == ST_B32 else a, b if f == ST_V4 else 0]
        return R, w
    slots = 1 + word(seed, CLUSTER, r, 3, 0) % 8
    wide = f == RED_ADD64
    R["arriver"], R["count"] = slots, THREADS * (8 if wide else 4)
    per = [sum(1 for t in range(THREADS) if t % slots == s) for s in range(8)]
    bound = 2000 + word(seed, CLUSTER, r, 3, 1) % 1000
    for s in range(slots):
        x = word(seed, CLUSTER, r, 1, s)
        R["slot_init"][s] = x % 1000 if f == RED_INC else per[s] + x % 1000 if f == RED_DEC else x if wide else x & M32
    d = list(R["slot_init"])
    for t in range(THREADS):
        a, b = word(seed, CLUSTER, r, 0, t), word(seed, CLUSTER, r, 2, t) & M32
        v = a if wide else a & M32
        if f == RED_AND:
            v |= b
        if f == RED_OR:
            v &= b
        if f in (RED_INC, RED_DEC):
            v = bound
        w[t][0] = v
        s, o = t % slots, d[t % slots]
        d[s] = {RED_ADD: lambda: (o + v) & M32, RED_ADD64: lambda: (o + v) & U64, RED_MIN: lambda: min(o, v), RED_MAX: lambda: max(o, v),
                RED_MINS: lambda: min(s32(o), s32(v)) & M32, RED_MAXS: lambda: max(s32(o), s32(v)) & M32, RED_AND: lambda: o & v,
                RED_OR: lambda: o | v, RED_XOR: lambda: o ^ v, RED_INC: lambda: 0 if o >= v else o + 1,
                RED_DEC: lambda: v if (o == 0 or o > v) else o - 1}[f]()
    R["slot_expect"] = d
    return R, w


def table(leg, seed, cluster=2):
    return [row(leg, seed, r, cluster) for r in range(OPS[leg])]


def checks(leg, R, w, t, rank=0):
    """Thread t's checks of row R in the device's order: (kind, bar, phase, slot, expected, folded)."""
    f = R["form"]
    part = R["warps"] >> (t >> 5) & 1
    if f == ARRIVE:
        return [(EARLY, R["bar"], 0, p, w[p][0], True) for p in members(R["producers"])] if part else []
    if f in (POPC, AND, OR):
        return [(VALUE, R["bar"], 0, 0, R["expect"], True)] if part else []
    if f == CBAR:
        return [(EARLY, f, 0, 0, w[t][0], True), (VALUE, f, 0, 1, R["next_rank"][rank], False)]
    if leg == MBAR:
        out = []
        for j in range(R["phases"]):
            if f == TICKET and part:
                out += [(TICKET_KIND, f, j, 0, 1, True), (TICKET_KIND, f, j, 1, t, True)]
            out += [(EARLY, f, j, 2, 0, True), (VALUE, f, j, 3, 1, True), (VALUE, f, j, 4, 1, True)]
        return out
    out = [(VALUE, f, 0, 2, 1, True)]
    if f <= ST_V4:
        out += [(VALUE, f, 0, 0, w[t][0], True), (VALUE, f, 0, 1, w[t][1], True)]
    elif t < R["arriver"]:
        out.append((VALUE, f, 0, 0, R["slot_expect"][t], True))
    return out


def fold(leg, seed, cluster=2) -> Tuple[int, int, int]:
    x = s = wt = 0
    for op, (R, w) in enumerate(table(leg, seed, cluster)):
        for t in range(THREADS):
            for c in checks(leg, R, w, t):
                if c[5]:
                    x ^= c[4]
                    s += c[4]
                    wt += c[4] * (2 * op + 1)
    return x, s & U64, wt & U64


def injected(leg, seed, op, w_, l, mask, cluster=2, rank=0):
    """The records an injection of mask into row op of thread (w_, l) makes, as (kind, bar, phase, slot, expected,
    actual), in the order the thread keeps them.  rank: the CTA's cluster rank, which only the CBAR rows' getctarank
    check depends on (the device does not report it, so a caller matching a CLUSTER CTA's records tries each rank)."""
    R, w = row(leg, seed, op, cluster)
    return [(k, b, p, s, e, e ^ mask) for k, b, p, s, e, _f in checks(leg, R, w, 32 * w_ + l, rank)]


# ---- classification and annotations: the cross-lane probe's rules for three legs, then the barrier probe's own ------
OK, ERR_CUDA, ERR_CHECKSUM, ERR_UNSUPPORTED = 0, -4, -6, -10
PERSISTENT, INTERMITTENT = 1, 2
THREAD_RECORDS, RECORDS, MAX_SMS = 4, 4096, 256


def _blank(call):
    return {"status": OK, "verdict": NONE, "seed": call["seed"], "call": call["call"], "sm_count": call["sm_count"],
            "legs": call["legs"], "nsmid": 0, "iterations": call["iterations"], "rounds": 0, "sms_covered": 0, "complete": 0,
            "ctas": 0, "unpublished": 0, "threads_unpublished": 0, "failed_sms": 0, "bad_sms": 0, "failed_legs": 0,
            "bad_sm": [], "mismatches": [0] * LEGS, "ops_checked": [0] * LEGS, "fold_mismatches": [0] * LEGS,
            "fold": [(0, 0, 0)] * LEGS, "timer_ns": 0, "timeouts": 0, "cluster_sms": 0, "bad_pairs": 0, "bad_pair": []}


def classify(call: Dict, expect: Dict[int, Tuple[int, int, int]]):
    """call = {"legs", "seed", "call", "iterations", "sm_count", "rounds": {leg: [(ctas, threads, records)]}} with
    dicts of the cro_barrier_cta / _thread / _fault fields; expect[leg] the leg's closed form.  Returns (result, SM
    entries by smid, the records sorted and capped), or a blanked result of status ERR_UNSUPPORTED."""
    r = _blank(call)
    per_sm, last, seen, fold_sm, kept = {}, {}, {leg: set() for leg in range(LEGS)}, {}, []
    k = call["call"]
    for leg in range(LEGS):
        if not call["legs"] >> leg & 1:
            continue
        for ctas, threads, records in call["rounds"][leg]:
            r["rounds"] += 1
            r["ctas"] += len(ctas)
            t0, t1 = None, 0
            for j, x in enumerate(ctas):
                if x["stamp"] != k:
                    r["unpublished"] += 1
                    r["failed_legs"] |= 1 << leg
                    continue
                if x["nsmid"] > MAX_SMS:
                    b = _blank(call)
                    b["status"] = ERR_UNSUPPORTED
                    return b, [], []
                r["nsmid"] = x["nsmid"]
                t0 = x["t0"] if t0 is None else min(t0, x["t0"])
                t1 = max(t1, x["t1"])
                seen[leg].add(x["smid"])
                S = per_sm.setdefault(x["smid"], {"smid": x["smid"], "mark": 0, "failed_legs": 0, "ctas": 0,
                                                  "mismatches": [0] * LEGS, "fold_mismatches": 0, "ns": 0, "cycles": 0})
                S["ctas"] += 1
                S["ns"] += x["t1"] - x["t0"] if x["t1"] > x["t0"] else 0
                S["cycles"] = (S["cycles"] + x["cycles"]) & U64
                fx = fs = fw = n = 0
                silent = False
                for q in range(THREADS):
                    e = threads[j * THREADS + q]
                    if e["stamp"] != k:
                        r["threads_unpublished"] += 1
                        silent = True
                        continue
                    n += e["count"]
                    last[x["smid"]] = last.get(x["smid"], 0) + e["last"]
                    fx ^= e["fold_x"]
                    fs = (fs + e["fold_s"]) & U64
                    fw = (fw + e["fold_w"]) & U64
                    base = (j * THREADS + q) * THREAD_RECORDS
                    kept += records[base:base + min(e["count"], THREAD_RECORDS)]
                S["mismatches"][leg] += n
                r["mismatches"][leg] += n
                r["ops_checked"][leg] += OPS[leg] * THREADS * call["iterations"]
                bad = not silent and (fx, fs, fw) != tuple(expect[leg])
                S["fold_mismatches"] += bad
                r["fold_mismatches"][leg] += bad
                if n or bad or silent:
                    S["failed_legs"] |= 1 << leg
                    r["failed_legs"] |= 1 << leg
                if leg not in fold_sm or x["smid"] < fold_sm[leg]:
                    fold_sm[leg] = x["smid"]
                    r["fold"][leg] = (fx, fs, fw)
            if t0 is not None and t1 > t0:
                r["timer_ns"] += t1 - t0
    # coverage: the CTA-local legs' when one ran (a cluster cannot use every SM), else the CLUSTER leg's
    local = [leg for leg in (BAR, MBAR) if call["legs"] >> leg & 1]
    ran = local or ([CLUSTER] if call["legs"] >> CLUSTER & 1 else [])
    r["sms_covered"] = min(len(seen[leg]) for leg in ran) if ran else 0
    r["complete"] = int(r["sms_covered"] >= r["sm_count"])
    r["cluster_sms"] = len(seen[CLUSTER])
    sms = [per_sm[s] for s in sorted(per_sm)]
    for S in sms:
        S["mark"] = PERSISTENT if last.get(S["smid"], 0) else INTERMITTENT if S["failed_legs"] else 0
        if S["mark"]:
            r["bad_sms"] += 1
            if len(r["bad_sm"]) < 16:
                r["bad_sm"].append(S["smid"])
    r["failed_sms"] = r["bad_sms"]
    r["timeouts"] = sum(1 for q in kept if q["kind"] == TIMEOUT)
    pairs = sorted({(q["smid"], q["peer_smid"]) for q in kept if q["leg"] == CLUSTER})
    r["bad_pairs"], r["bad_pair"] = len(pairs), pairs[:16]
    recs = sorted(kept, key=lambda q: (q["leg"], q["smid"], q["iteration"], q["op"], q["warp"], q["lane"]))[:RECORDS]
    silent = r["unpublished"] or r["threads_unpublished"]
    every = silent or (r["failed_sms"] and r["failed_sms"] == len(per_sm))
    anyf = silent or r["failed_sms"]
    r["verdict"] = ALL if every else SM if anyf else NONE
    if r["verdict"] == SM and all(S["failed_legs"] == 1 << CLUSTER for S in sms if S["mark"]):
        r["verdict"] = LINK
    r["status"] = ERR_CHECKSUM if anyf else OK
    return r, sms, recs


def annotations(r: Dict) -> Dict[str, str]:
    """r = {"status", "verdict", "cuda_error", "sms_covered", "sm_count", "bad_sms", "bad_sm" (the first min(bad_sms,
    16)), "failed_legs", "iterations", "bad_pairs", "bad_pair" (the first min(bad_pairs, 16))}."""
    p = "cohdi.io/probe-barrier-"
    st = r["status"]
    names = {SM: "sm", ALL: "all", LINK: "link"}
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
    legs = [NAMES[b] for b in range(LEGS) if r["failed_legs"] >> b & 1]
    if legs:
        m[p + "legs"] = ",".join(legs)
    m[p + "iterations"] = str(r["iterations"])
    if r["bad_pairs"]:
        m[p + "bad-pairs"] = ",".join("%d>%d" % q for q in r["bad_pair"][:min(r["bad_pairs"], 16)])
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
