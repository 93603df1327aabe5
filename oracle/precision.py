"""Restatement of the SM precision probe (cro_probe_precision): operands, answers, each leg's encoding of the answer and
the fold over it, and the annotation emitter (cro_emit_precision_annotations_json).

Independent of csrc/precision_probe.cu: numpy over the header's rules (include/croprobe.h, "SM precision").  An emitter
input is a dict shaped as oracle/compute.py's, with 7 legs.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

import sm_legs
from oracle import go_marshal_string_map, pattern_words_np

WIDE, SMALL128, SMALL, NARROW = range(4)
SHAPE = {WIDE: (128, 64, 128), SMALL128: (128, 256, 128), SMALL: (128, 256, 256), NARROW: (128, 256, 256)}
BOUND = {WIDE: 1 << 45, SMALL128: 16 * 128, SMALL: 16 * 256, NARROW: 4 * 256}     # sum over k of |a * b|
LEG_NAMES = ["f64", "dfma", "tf32", "f16", "f16acc", "e5m2", "hfma2"]
LEG_ANSWER = [WIDE, WIDE, SMALL128, SMALL, NARROW, SMALL, NARROW]
LEG_BITS = [64, 64, 32, 32, 16, 32, 16]
LEGS, RECORDS = 7, 4096
RATE_LEGS = [(0, "f64-gflops"), (2, "tf32-gflops"), (3, "f16-gflops"), (4, "f16acc-gflops"), (5, "e5m2-gflops")]
OK, ERR_CHECKSUM = 0, -6
NONE, SM, ALL = 0, 1, 2
U64 = (1 << 64) - 1


def operands(answer: int, seed: int):
    """(A as M x K, B as K x N) int64 arrays of the answer's reading of the operands of `seed`."""
    m, n, k = SHAPE[answer]
    count = m * k + k * n
    if answer == WIDE:
        w = pattern_words_np(seed, 0, count).astype(np.uint64)
        low = (w & np.uint64(0xFFFFF)).astype(np.int64)
        v = np.where(low >= 1 << 19, low - (1 << 20), low)
    else:
        b = pattern_words_np(seed, 0, count // 8).astype("<u8").view(np.uint8).astype(np.int64)
        v = (b & 3) - 2 if answer == NARROW else (b & 7) - 4
    return v[:m * k].reshape(m, k), v[m * k:].reshape(k, n)


def answer(answer_kind: int, seed: int) -> np.ndarray:
    a, b = operands(answer_kind, seed)
    return a @ b


def abs_sum(answer_kind: int, seed: int) -> np.ndarray:
    """Per element, sum over k of |A[m][k] * B[k][n]|: a bound on every partial sum in any order."""
    a, b = operands(answer_kind, seed)
    return np.abs(a) @ np.abs(b)


def encode(leg: int, tile: np.ndarray) -> np.ndarray:
    """The leg's type's bit pattern of every value (uint64, zero-extended), -0 taken as 0."""
    bits = LEG_BITS[leg]
    if bits == 64:
        raw = tile.astype(np.float64).view(np.uint64)
    elif bits == 32:
        raw = tile.astype(np.float32).view(np.uint32).astype(np.uint64)
    else:
        raw = tile.astype(np.float16).view(np.uint16).astype(np.uint64)
    return np.where(raw == np.uint64(1 << (bits - 1)), np.uint64(0), raw)


def cta_fold(leg: int, tile: np.ndarray, iterations: int = 1) -> int:
    """Sum over every element e of canon(value) * (2e + 1) mod 2^64, times iterations: a clean CTA's fold."""
    v = encode(leg, tile).ravel()
    w = 2 * np.arange(v.size, dtype=np.uint64) + np.uint64(1)
    with np.errstate(over="ignore"):
        return (int((v * w).sum(dtype=np.uint64)) * iterations) & U64


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-precision-"
    if r["status"] == OK:
        verdict = "ok"
    elif r["status"] == ERR_CHECKSUM and r["verdict"] in (SM, ALL):
        verdict = "sm" if r["verdict"] == SM else "all"
    else:
        verdict = "error"
    ran = [i for i in range(7) if (r["legs"] >> i) & 1]
    legs = r["leg"]
    covered = min((legs[i]["sms_covered"] for i in ran), default=0)
    m = {p + "verdict": verdict, p + "sms": "%d/%d" % (covered, r["sm_count"])}
    if r["bad_sms"]:
        m[p + "bad-sms"] = ",".join(str(x) for x in r["bad_sm"][:min(r["bad_sms"], 16)])
    failed = [LEG_NAMES[i] for i in ran
              if legs[i]["mismatches"] or legs[i]["fold_mismatches"] or legs[i]["unpublished"]]
    if failed:
        m[p + "failed-legs"] = ",".join(failed)
    for i, key in RATE_LEGS:
        m[p + key] = str(legs[i]["ops"] // legs[i]["ns"] if legs[i]["ns"] else 0)
    if ran:
        worst = ran[0]
        for i in ran:
            if legs[i]["slow_permille"] > legs[worst]["slow_permille"]:
                worst = i
        m[p + "slowest-sm"] = "%d %d" % (legs[worst]["slowest_sm"], legs[worst]["slow_permille"])
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode()


def classify(call: Dict):
    """The classification of a call's rounds and records (oracle/sm_legs.py): leg l computes its answer's M x N x K."""
    ops = [2 * SHAPE[a][0] * SHAPE[a][1] * SHAPE[a][2] for a in LEG_ANSWER]
    return sm_legs.classify(call, LEGS, ops, RECORDS)
