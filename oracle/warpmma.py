"""Restatement of the SM warp-MMA probe (cro_probe_warpmma): the answers (the compute and precision probes' for the
arithmetic legs, the block-transposed tile for MOVE), each leg's encoding of its answer and the fold over it, the wrong
row a fragment-address substitution must give, and the annotation emitter (cro_emit_warpmma_annotations_json).

Independent of csrc/warpmma_probe.cu: numpy over the header's rules (include/croprobe.h, "SM warp-MMA").  An emitter
input is a dict shaped as oracle/compute.py's, with 6 legs.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

import compute
import precision
import sm_legs
from oracle import go_marshal_string_map, pattern_words_np

S8, SMALL, SMALL128, NARROW, MOVE = range(5)
M, N = 128, 256
K = {S8: 256, SMALL: 256, SMALL128: 128, NARROW: 256}
LEG_NAMES = ["s8", "f16", "bf16", "tf32", "f16acc", "move"]
LEG_ANSWER = [S8, SMALL, SMALL, SMALL128, NARROW, MOVE]
LEG_ELEM = [1, 2, 2, 4, 2, 2]                                     # operand bytes of an arithmetic leg; MOVE: a word
LEG_BITS = [32, 32, 32, 32, 16, 16]
LEGS, RECORDS = 6, 4096
RATE_LEGS = [(0, "s8-gops"), (1, "f16-gflops"), (2, "bf16-gflops"), (3, "tf32-gflops"), (4, "f16acc-gflops"),
             (5, "move-gelems")]
OK, ERR_CHECKSUM = 0, -6
NONE, SM, ALL = 0, 1, 2
U64 = (1 << 64) - 1


def source_tile(seed: int) -> np.ndarray:
    """MOVE's source S: M x N 16-bit words, S[r][c] halfword e % 4 of pattern_word(seed, e // 4), e = r * N + c."""
    return pattern_words_np(seed, 0, M * N // 4).astype("<u8").view("<u2").astype(np.int64).reshape(M, N)


def operands(answer: int, seed: int):
    """(A as M x K, B as K x N) of an arithmetic answer: the compute probe's (S8, SMALL) or precision probe's."""
    if answer in (S8, SMALL):
        return compute.operands(answer, seed)
    return precision.operands(precision.SMALL128 if answer == SMALL128 else precision.NARROW, seed)


def answer(answer_kind: int, seed: int) -> np.ndarray:
    if answer_kind == MOVE:
        s = source_tile(seed)
        return s.reshape(M // 8, 8, N // 8, 8).transpose(0, 3, 2, 1).reshape(M, N)    # E[8a + i][8b + j] = S[8a + j][8b + i]
    a, b = operands(answer_kind, seed)
    return a @ b


def k_steps(leg: int) -> int:
    """16-byte K segments of an A row of an arithmetic leg: the k-steps a substitution may name."""
    return K[LEG_ANSWER[leg]] * LEG_ELEM[leg] // 16


def substituted_row(leg: int, seed: int, row: int, kstep: int) -> np.ndarray:
    """Row `row` of the answer when the A ldmatrix of k-step `kstep` reads row ^ 1 for that 16-byte segment: D[R][n] +
    sum over its k of (A[R ^ 1][k] - A[R][k]) * B[k][n].  Every other row is unchanged."""
    a, b = operands(LEG_ANSWER[leg], seed)
    per = 16 // LEG_ELEM[leg]
    ks = slice(kstep * per, (kstep + 1) * per)
    return a[row] @ b + (a[row ^ 1, ks] - a[row, ks]) @ b[ks]


def substituted_partial_bound(leg: int, seed: int, row: int, kstep: int) -> int:
    """Sum over k of |a'[k] * B[k][n]| of the substituted row, the largest over n: a bound on every partial sum."""
    a, b = operands(LEG_ANSWER[leg], seed)
    per = 16 // LEG_ELEM[leg]
    r = a[row].copy()
    r[kstep * per:(kstep + 1) * per] = a[row ^ 1, kstep * per:(kstep + 1) * per]
    return int((np.abs(r) @ np.abs(b)).max())


def encode(leg: int, tile: np.ndarray) -> np.ndarray:
    """The value's bits in the leg's type (uint64): int32 for S8, f32 for F16 / BF16 / TF32, f16 for F16ACC (both with
    -0 taken as 0), the raw 16-bit word for MOVE."""
    if leg == 0:
        return tile.astype(np.int64).astype(np.uint32).astype(np.uint64)
    if leg == 5:
        return (tile.astype(np.int64) & 0xFFFF).astype(np.uint64)
    bits = LEG_BITS[leg]
    raw = tile.astype(np.float16).view(np.uint16) if bits == 16 else tile.astype(np.float32).view(np.uint32)
    raw = raw.astype(np.uint64)
    return np.where(raw == np.uint64(1 << (bits - 1)), np.uint64(0), raw)


def cta_fold(leg: int, tile: np.ndarray, iterations: int = 1) -> int:
    """Sum over every element e of canon(value) * (2e + 1) mod 2^64, times iterations: a clean CTA's fold."""
    v = encode(leg, tile).ravel()
    w = 2 * np.arange(v.size, dtype=np.uint64) + np.uint64(1)
    with np.errstate(over="ignore"):
        return (int((v * w).sum(dtype=np.uint64)) * iterations) & U64


def value_bits(leg: int, v: int) -> int:
    """The raw bits a thread holds for the integer v (zero-extended)."""
    if leg == 0:
        return v & 0xFFFFFFFF
    if leg == 5:
        return v & 0xFFFF
    if LEG_BITS[leg] == 16:
        return int(np.array([v], dtype=np.float16).view(np.uint16)[0])
    return int(np.array([v], dtype=np.float32).view(np.uint32)[0])


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-warpmma-"
    if r["status"] == OK:
        verdict = "ok"
    elif r["status"] == ERR_CHECKSUM and r["verdict"] in (SM, ALL):
        verdict = "sm" if r["verdict"] == SM else "all"
    else:
        verdict = "error"
    ran = [i for i in range(LEGS) if (r["legs"] >> i) & 1]
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


def ops(leg: int) -> int:
    """Operations per CTA and iteration: 2 M N K, MOVE the M N elements it moves."""
    return M * N if leg == 5 else 2 * M * N * K[LEG_ANSWER[leg]]


def classify(call: Dict):
    """The classification of a call's rounds and records (oracle/sm_legs.py) with this probe's six legs."""
    return sm_legs.classify(call, LEGS, [ops(l) for l in range(LEGS)], RECORDS)
