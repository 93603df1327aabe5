"""Restatement of the cross-lane probe (include/croprobe.h "cross-lane"): each leg's operands, the results the PTX ISA
defines for them, the fold's closed form, what a test injection does, the classification and the annotations.

Pure Python over plain values, written from the PTX ISA's definitions of shfl.sync, vote.sync, match.sync,
redux.sync and atom.shared, so the library's cro_xlane_expected and classification can be held to it without a GPU.

  expected(leg, seed, it, w)       [op * 32 + lane] of warp w in iteration it
  fold(leg, seed, iterations)      the closed form of every CTA's fold of the leg
  injected(leg, seed, it, op, w, l, mask)
                                   {(warp, lane): (expected, actual, peer)}: the records an injection into lane l of
                                   warp w in op `op` of iteration `it` makes, over the whole CTA
  classify(call), annotations(r)
"""
from __future__ import annotations

from typing import Dict, List, Tuple

from oracle import go_marshal_string_map, pattern_word

OK, ERR_CUDA, ERR_CHECKSUM, ERR_UNSUPPORTED = 0, -4, -6, -10
NONE, SM, ALL = 0, 1, 2
PERSISTENT, INTERMITTENT = 1, 2
SHFL, VOTE, MATCH, REDUX, ATOMS = range(5)
LEGS, THREADS, WARPS, THREAD_RECORDS, RECORDS, MAX_SMS = 5, 256, 8, 4, 4096, 256
OPS = [177, 384, 64, 1296, 60]
NAMES = ["shfl", "vote", "match", "redux", "atoms"]
STRIDE = 0xD1B54A32D192ED03
SEED_OFFSET, SEEDS_PER_CALL = 1 << 54, 4096
NO_PEER = 0xFFFFFFFF
U32, U64 = (1 << 32) - 1, (1 << 64) - 1


def call_seed(seed_dev: int, k: int) -> int:
    return (seed_dev + SEED_OFFSET + SEEDS_PER_CALL * k * STRIDE) & U64


def iteration_seed(seed: int, i: int) -> int:
    return (seed + i * STRIDE) & U64


def word(s: int, leg: int, op: int, w: int, l: int) -> int:
    return pattern_word(s, (leg << 22) | (op << 10) | (w << 6) | l)


def s32(x: int) -> int:
    return x - (1 << 32) if x & 0x80000000 else x


# ---- SHFL -----------------------------------------------------------------------------------------------------------
def shfl_ops() -> List[Tuple[str, int, int]]:
    """(mode, b, width) per op; for idx b is the offset r (the source lane is lane + r)."""
    ops = [("idx", r, 32) for r in range(32)]
    for mode in ("up", "down"):
        for width in (32, 16, 8, 4, 2):
            ops += [(mode, d, width) for d in range(1, width)]
    ops += [("bfly", m, 32) for m in range(1, 32)]
    assert len(ops) == OPS[SHFL]
    return ops


SHFL_OPS = shfl_ops()


def shfl_source(op: int, lane: int) -> Tuple[int, bool]:
    """The lane whose value `lane` receives and the predicate: a source outside the lane's segment of `width` lanes
    leaves the lane its own value and the predicate false."""
    mode, b, width = SHFL_OPS[op]
    lo = lane - lane % width
    if mode == "idx":
        return (lane + b) % 32, True
    j = lane - b if mode == "up" else lane + b if mode == "down" else lane ^ b
    ok = lo <= j < lo + width
    return (j, True) if ok else (lane, False)


def shfl_operand(s, op, w, l):
    return word(s, SHFL, op, w, l) & U32


# ---- VOTE -----------------------------------------------------------------------------------------------------------
def vote_pred_bit(row: int, l: int):
    if row == 0:
        return 0
    if row == 1:
        return 1
    if row < 34:
        return int(l == row - 2)
    if row < 66:
        return int(l != row - 34)
    return None


def vote_operand(s, row, w, l):
    x = word(s, VOTE, row, w, l) & U32
    b = vote_pred_bit(row, l)
    return x if b is None else (x & ~1 & U32) | b


def vote_results(preds: List[int]) -> List[int]:
    ballot = sum(p << l for l, p in enumerate(preds))
    return [ballot, int(any(preds)), int(all(preds)), int(all(preds) or not any(preds))]


# ---- MATCH ----------------------------------------------------------------------------------------------------------
def match_values(s, row, w) -> Tuple[List[int], List[int]]:
    n = [1, 2, 3, 32][row] if row < 4 else 1 + (word(s, MATCH, row, 8, 0) & U32) % 32
    cls = [l if n == 32 else (word(s, MATCH, row, w, l) & U32) % n for l in range(32)]
    v32 = [word(s, MATCH, row, w, 32 + c) & U32 for c in cls]
    hi = lambda c: word(s, MATCH, row, 8 + w, c & ~1) & U32
    lo = lambda c: word(s, MATCH, row, 8 + w, 32 + (c & ~2)) & U32
    v64 = [(hi(c) << 32) | lo(c) for c in cls]
    return v32, v64


def match_results(v: List[int]) -> List[Tuple[int, int]]:
    """(any, all) of every lane: any = the mask of lanes holding its value; all = the full mask with the predicate
    (bit 32) when every lane holds one value, else 0."""
    same = all(x == v[0] for x in v)
    return [(sum(1 << j for j in range(32) if v[j] == v[l]), (1 << 33) - 1 if same else 0) for l in range(32)]


# ---- REDUX ----------------------------------------------------------------------------------------------------------
def redux_operand(s, row, w, l):
    x = word(s, REDUX, row, w, l) & U32
    if row >= 128:
        return x
    j, k = row % 32, row // 32
    if k == 0:
        return 0 if l == j else x | (1 << j) | 1
    if k == 1:
        return U32 if l == j else x & ~(1 << j) & ~1 & U32
    if k == 2:
        return 0x80000000 if l == j else x & 0x7FFFFFFF
    return 0x7FFFFFFF if l == j else x | 0x80000000


def redux_results(v: List[int]) -> List[int]:
    sv = [s32(x) for x in v]
    x = o = 0
    an = U32
    for y in v:
        an &= y
        o |= y
        x ^= y
    return [sum(v) & U32, sum(sv) & U32, min(v), max(v), min(sv) & U32, max(sv) & U32, an, o, x]


# ---- ATOMS ----------------------------------------------------------------------------------------------------------
KINDS = ["add", "inc", "dec", "min.u32", "max.u32", "min.s32", "max.s32", "and", "or", "xor", "exch.b32", "exch.b64",
         "cas.b32", "cas.b64", "add.u64"]
WIDE = {"exch.b64", "cas.b64", "add.u64"}


def atoms_groups(shape: int) -> List[List[Tuple[int, int]]]:
    """Each group's members (warp, lane) in rank order."""
    if shape == 0:
        return [[(t >> 5, t & 31) for t in range(THREADS)]]
    if shape == 1:
        return [[(w, l) for l in range(32)] for w in range(WARPS)]
    if shape == 2:
        return [[(w, l) for w in range(WARPS)] for l in range(32)]
    return [[(t >> 5, t & 31)] for t in range(THREADS)]


def atoms_group_of(shape, w, l) -> int:
    return [0, w, l, 32 * w + l][shape]


def atoms_init(s, op, g):
    v = word(s, ATOMS, op, 8 + (g >> 6), g & 63)
    kind = KINDS[op // 4]
    if kind == "inc":
        return v & 0x3FFFFFFF
    if kind == "dec":
        return (v & 0x3FFFFFFF) | 0x40000000
    return v if kind in WIDE else v & U32


def atoms_value(s, op, w, l, rank, g):
    kind = KINDS[op // 4]
    x = word(s, ATOMS, op, w, l)
    if kind.startswith("exch"):
        v = atoms_init(s, op, g) ^ (rank + 1)
        return v if kind in WIDE else v & U32
    if kind == "inc":
        return (x | 0xC0000000) & U32
    if kind == "dec":
        return (x | 0x80000000) & U32
    return x if kind in WIDE else x & U32


def atoms_group_results(kind: str, init: int, vals: List[int]) -> List[int]:
    """What each member checks after every member's atom ran, in whatever order: the final word for the
    order-independent kinds; for inc / dec the final word (bits 32..63) and its ticket's presence (bit 0); for exch
    whether its own value's presence slot was marked by the old value someone got back or by the final word."""
    n = len(vals)
    if kind.startswith("exch"):
        # the old values returned and the final word are the initial word and every value, each once, in any order
        return [int((init ^ (r + 1)) in vals) for r in range(n)]
    if kind == "inc":
        return [((init + n) << 32) | 1] * n
    if kind == "dec":
        return [((init - n) << 32) | 1] * n
    acc = init
    for v in vals:
        if kind in ("add", "cas.b32"):
            acc = (acc + v) & U32
        elif kind in ("add.u64", "cas.b64"):
            acc = (acc + v) & U64
        elif kind == "min.u32":
            acc = min(acc, v)
        elif kind == "max.u32":
            acc = max(acc, v)
        elif kind == "min.s32":
            acc = min(acc, v, key=s32)
        elif kind == "max.s32":
            acc = max(acc, v, key=s32)
        elif kind == "and":
            acc &= v
        elif kind == "or":
            acc |= v
        else:
            acc ^= v
    return [acc] * n


def atoms_op(s, op, inj=None, mask=0) -> Dict[Tuple[int, int], int]:
    """{(warp, lane): result} of op `op`, with `mask` XORed into the value of member inj = (warp, lane)."""
    kind, shape = KINDS[op // 4], op % 4
    out = {}
    for g, members in enumerate(atoms_groups(shape)):
        init = atoms_init(s, op, g)
        vals = []
        for r, (w, l) in enumerate(members):
            v = atoms_value(s, op, w, l, r, g)
            if (w, l) == inj:
                v = (v ^ mask) & (U64 if kind in WIDE else U32)
            vals.append(v)
        for (w, l), res in zip(members, atoms_group_results(kind, init, vals)):
            out[(w, l)] = res
    return out


# ---- every leg ------------------------------------------------------------------------------------------------------
def _warp_results(leg, s, w, inj_lane=None, inj_op=None, mask=0) -> List[Tuple[int, int]]:
    """[(result, peer)] by op * 32 + lane of warp w, with mask XORed into lane inj_lane's operand of op inj_op."""
    m = lambda op, l: mask if (op == inj_op and l == inj_lane) else 0
    out = [None] * (OPS[leg] * 32)
    if leg == SHFL:
        for op in range(OPS[SHFL]):
            for l in range(32):
                j, p = shfl_source(op, l)
                out[op * 32 + l] = (((shfl_operand(s, op, w, j) ^ m(op, j)) & U32) | (int(p) << 32), j)
    elif leg == VOTE:
        for row in range(OPS[VOTE] // 4):
            x = [vote_operand(s, row, w, l) for l in range(32)]
            for f in range(4):
                op = row * 4 + f
                r = vote_results([(x[l] ^ m(op, l)) & 1 for l in range(32)])[f]
                for l in range(32):
                    out[op * 32 + l] = (r, NO_PEER)
    elif leg == MATCH:
        for row in range(OPS[MATCH] // 4):
            v32, v64 = match_values(s, row, w)
            for f in range(4):
                op = row * 4 + f
                v = [(v32[l] ^ m(op, l)) & U32 for l in range(32)] if f < 2 else [(v64[l] ^ m(op, l)) & U64 for l in range(32)]
                res = match_results(v)
                for l in range(32):
                    out[op * 32 + l] = (res[l][f % 2], NO_PEER)
    elif leg == REDUX:
        for row in range(OPS[REDUX] // 9):
            x = [redux_operand(s, row, w, l) for l in range(32)]
            for f in range(9):
                op = row * 9 + f
                r = redux_results([(x[l] ^ m(op, l)) & U32 for l in range(32)])[f]
                for l in range(32):
                    out[op * 32 + l] = (r, NO_PEER)
    else:
        for op in range(OPS[ATOMS]):
            res = atoms_op(s, op)
            for l in range(32):
                out[op * 32 + l] = (res[(w, l)], NO_PEER)
    return out


def expected(leg: int, seed: int, it: int, w: int) -> List[int]:
    return [r for r, _ in _warp_results(leg, iteration_seed(seed, it), w)]


def fold(leg: int, seed: int, iterations: int) -> Tuple[int, int, int]:
    x = s = wt = 0
    for w in range(WARPS):
        e = expected(leg, seed, iterations - 1, w)
        for i, v in enumerate(e):
            x ^= v
            s += v
            wt += v * (2 * (i // 32) + 1)
    return x, s & U64, wt & U64


def injected(leg: int, seed: int, it: int, op: int, w: int, l: int, mask: int) -> Dict[Tuple[int, int], Tuple[int, int, int]]:
    """The records of an injection: {(warp, lane): (expected, actual, peer)} over the CTA, for op `op`."""
    s = iteration_seed(seed, it)
    out = {}
    if leg == ATOMS:
        clean, bad = atoms_op(s, op), atoms_op(s, op, (w, l), mask)
        return {k: (clean[k], bad[k], NO_PEER) for k in clean if clean[k] != bad[k]}
    clean = _warp_results(leg, s, w)
    bad = _warp_results(leg, s, w, l, op, mask)
    for lane in range(32):
        (e, peer), (a, _) = clean[op * 32 + lane], bad[op * 32 + lane]
        if e != a:
            out[(w, lane)] = (e, a, peer)
    return out


# ---- classification and annotations --------------------------------------------------------------------------------
def _blank(call):
    return {"status": OK, "verdict": NONE, "seed": call["seed"], "call": call["call"], "sm_count": call["sm_count"],
            "legs": call["legs"], "nsmid": 0, "iterations": call["iterations"], "rounds": 0, "sms_covered": 0, "complete": 0,
            "ctas": 0, "unpublished": 0, "threads_unpublished": 0, "failed_sms": 0, "bad_sms": 0, "failed_legs": 0,
            "bad_sm": [], "mismatches": [0] * LEGS, "ops_checked": [0] * LEGS, "fold_mismatches": [0] * LEGS,
            "fold": [(0, 0, 0)] * LEGS, "timer_ns": 0}


def classify(call: Dict, expect: Dict[int, Tuple[int, int, int]]) -> Tuple[Dict, List[Dict], List[Dict]]:
    """call = {"legs", "seed", "call", "iterations", "sm_count", "rounds": {leg: [(ctas, threads, records)]}} with
    dicts of the cro_xlane_cta / _thread / _fault fields; expect[leg] the leg's closed form.  Returns (result, SM
    entries by smid, the records sorted and capped), or a blanked result of status ERR_UNSUPPORTED."""
    r = _blank(call)
    per_sm, last, seen, fold_sm, recs = {}, {}, {leg: set() for leg in range(LEGS)}, {}, []
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
                    recs += records[base:base + min(e["count"], THREAD_RECORDS)]
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
    ran = [leg for leg in range(LEGS) if call["legs"] >> leg & 1]
    r["sms_covered"] = min(len(seen[leg]) for leg in ran) if ran else 0
    r["complete"] = int(r["sms_covered"] >= r["sm_count"])
    sms = [per_sm[s] for s in sorted(per_sm)]
    for S in sms:
        S["mark"] = PERSISTENT if last.get(S["smid"], 0) else INTERMITTENT if S["failed_legs"] else 0
        if S["mark"]:
            r["bad_sms"] += 1
            if len(r["bad_sm"]) < 16:
                r["bad_sm"].append(S["smid"])
    r["failed_sms"] = r["bad_sms"]
    recs = sorted(recs, key=lambda q: (q["leg"], q["smid"], q["iteration"], q["op"], q["warp"], q["lane"]))[:RECORDS]
    silent = r["unpublished"] or r["threads_unpublished"]
    every = silent or (r["failed_sms"] and r["failed_sms"] == len(per_sm))
    anyf = silent or r["failed_sms"]
    r["verdict"] = ALL if every else SM if anyf else NONE
    r["status"] = ERR_CHECKSUM if anyf else OK
    return r, sms, recs


def annotations(r: Dict) -> Dict[str, str]:
    """r = {"status", "verdict", "cuda_error", "sms_covered", "sm_count", "bad_sms", "bad_sm" (the first min(bad_sms,
    16)), "failed_legs", "iterations"}."""
    p = "cohdi.io/probe-xlane-"
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
    legs = [NAMES[b] for b in range(LEGS) if r["failed_legs"] >> b & 1]
    if legs:
        m[p + "legs"] = ",".join(legs)
    m[p + "iterations"] = str(r["iterations"])
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
