"""Restatement of the SM sparse probe (cro_probe_sparse): the compressed A, B and pair of every group, the answers, each
leg's encoding of the answer and the fold over it, the wrong answer a metadata substitution must give, and the
annotation emitter (cro_emit_sparse_annotations_json).

Independent of csrc/sparse_probe.cu: numpy over the header's rules (include/croprobe.h, "SM sparse").  An emitter input
is a dict shaped as oracle/compute.py's, with 6 legs.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

import sm_legs
from oracle import go_marshal_string_map, pattern_words_np

S8, SMALL, SMALL256, SMALL128 = range(4)
M, N = 128, 256
K = {S8: 512, SMALL: 512, SMALL256: 256, SMALL128: 128}          # logical K
GROUP = {S8: 4, SMALL: 4, SMALL256: 4, SMALL128: 2}              # K positions per group
PAIRS4 = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]         # the pair order of a 2:4 group
PAIRS2 = [(0,), (1,)]                                             # ... of a TF32 1:2 group
NIBBLE4 = [i | j << 2 for i, j in PAIRS4]
NIBBLE2 = [0x4, 0xE]
LEG_NAMES = ["s8", "e4m3", "e5m2", "bf16", "f16", "tf32"]
LEG_ANSWER = [S8, SMALL, SMALL, SMALL256, SMALL256, SMALL128]
LEGS, RECORDS = 6, 4096
RATE_LEGS = [(0, "s8-gops"), (1, "e4m3-gflops"), (2, "e5m2-gflops"), (3, "bf16-gflops"), (4, "f16-gflops"), (5, "tf32-gflops")]
OK, ERR_CHECKSUM = 0, -6
NONE, SM, ALL = 0, 1, 2
U64 = (1 << 64) - 1


def pairs(answer: int):
    return PAIRS2 if GROUP[answer] == 2 else PAIRS4


def groups(answer: int) -> int:
    return K[answer] // GROUP[answer]


def _bytes(seed: int, count: int) -> np.ndarray:
    return pattern_words_np(seed, 0, (count + 7) // 8).astype("<u8").view(np.uint8).astype(np.int64)[:count]


def operands(answer: int, seed: int):
    """(compressed A as M x K/2, B as K x N, pair index of every group as M x K/G) of the operands of `seed`."""
    k, g = K[answer], GROUP[answer]
    p = len(pairs(answer))
    kc, ng = k // 2, k // g
    blocks = -(-ng // p)
    b = _bytes(seed, M * kc + k * N + M * blocks)
    if answer == S8:
        v = np.where(b >= 128, b - 256, b)
        a = v[:M * kc]
        a = np.where(a == 0, 1, a)
    else:
        v = (b & 7) - 4
        a = v[:M * kc]
        a = np.where(a >= 0, a + 1, a)
    bm = v[M * kc:M * kc + k * N].reshape(k, N)
    rot = b[M * kc + k * N:].reshape(M, blocks)
    gi = np.arange(ng)
    pair = (gi[None, :] + rot[:, gi // p]) % p
    return a.reshape(M, kc), bm, pair


def logical_a(answer: int, seed: int, pair: Optional[np.ndarray] = None) -> np.ndarray:
    """The logical M x K A: each kept value at its pair's K position, zeros elsewhere (pair: the operands' by default)."""
    ac, _, own = operands(answer, seed)
    pair = own if pair is None else pair
    g = GROUP[answer]
    kept = len(pairs(answer)[0])
    idx = np.array(pairs(answer))[pair]                   # M x groups x kept
    a = np.zeros((M, K[answer]), dtype=np.int64)
    rows = np.arange(M)[:, None, None]
    cols = g * np.arange(groups(answer))[None, :, None] + idx
    a[np.broadcast_to(rows, cols.shape), cols] = ac.reshape(M, groups(answer), kept)
    return a


def answer(answer_kind: int, seed: int) -> np.ndarray:
    _, b, _ = operands(answer_kind, seed)
    return logical_a(answer_kind, seed) @ b


def abs_sum(answer_kind: int, seed: int) -> np.ndarray:
    """Per element, sum over k of |A[m][k] * B[k][n]|: a bound on every partial sum in any order."""
    _, b, _ = operands(answer_kind, seed)
    return np.abs(logical_a(answer_kind, seed)) @ np.abs(b)


def substituted(answer_kind: int, seed: int, row: int, group: int) -> np.ndarray:
    """The answer tile when group `group` of row `row` takes the next legal pair, its kept values unchanged: what a
    metadata substitution of that (row, group) must make the tensor core compute."""
    _, b, pair = operands(answer_kind, seed)
    pair = pair.copy()
    pair[row, group] = (pair[row, group] + 1) % len(pairs(answer_kind))
    return logical_a(answer_kind, seed, pair) @ b


def encode(leg: int, tile: np.ndarray) -> np.ndarray:
    """The accumulator's 32 bits of every value (uint64): int32 for S8, f32 otherwise with -0 taken as 0."""
    if LEG_ANSWER[leg] == S8:
        return tile.astype(np.int64).astype(np.uint32).astype(np.uint64)
    raw = tile.astype(np.float32).view(np.uint32).astype(np.uint64)
    return np.where(raw == np.uint64(1 << 31), np.uint64(0), raw)


def cta_fold(leg: int, tile: np.ndarray, iterations: int = 1) -> int:
    """Sum over every element e of canon(value) * (2e + 1) mod 2^64, times iterations: a clean CTA's fold."""
    v = encode(leg, tile).ravel()
    w = 2 * np.arange(v.size, dtype=np.uint64) + np.uint64(1)
    with np.errstate(over="ignore"):
        return (int((v * w).sum(dtype=np.uint64)) * iterations) & U64


def value_bits(leg: int, v: int) -> int:
    """The raw 32 bits the accumulator holds for the integer v."""
    if LEG_ANSWER[leg] == S8:
        return v & 0xFFFFFFFF
    return int(np.array([v], dtype=np.float32).view(np.uint32)[0])


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-sparse-"
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


def classify(call: Dict):
    """The classification of a call's rounds and records (oracle/sm_legs.py): leg l's ops are 2 M N K of its logical K."""
    ops = [2 * M * N * K[a] for a in LEG_ANSWER]
    return sm_legs.classify(call, LEGS, ops, RECORDS)
