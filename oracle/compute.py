"""Restatement of the SM compute probe (cro_probe_compute): operands, answers, the per-thread fold, and the annotation
emitter (cro_emit_compute_annotations_json).

Independent of csrc/compute.cpp and of compute_oracle.c: numpy over the header's rules (include/croprobe.h, "SM
compute").  An emitter input is a dict:
  {"status": int, "verdict": int, "sm_count": int, "legs": int, "bad_sms": int, "bad_sm": [int] * 16,
   "leg": [{"ops": int, "ns": int, "sms_covered": int, "mismatches": int, "fold_mismatches": int, "unpublished": int,
            "slowest_sm": int, "slow_permille": int}] * 5}
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict

import numpy as np

import sm_legs
from oracle import go_marshal_string_map, pattern_words_np

M, N, K = 128, 256, 256
S8, SMALL = 0, 1
LEG_NAMES = ["s8", "bf16", "e4m3", "ffma", "imad"]
LEG_ANSWER = [S8, SMALL, SMALL, SMALL, S8]
LEGS, RECORDS = 5, 4096
OK, ERR_CHECKSUM = 0, -6
NONE, SM, ALL = 0, 1, 2
U64 = (1 << 64) - 1


def operand_bytes(seed: int) -> np.ndarray:
    """The M*K + K*N operand bytes of `seed`: byte e is byte e % 8 (little-endian) of pattern_word(seed, e // 8)."""
    words = pattern_words_np(seed, 0, (M * K + K * N) // 8)
    return words.astype("<u8").view(np.uint8)


def operands(answer: int, seed: int):
    """(A as M x K, B as K x N) int64 arrays of the s8 (answer 0) or small-int (answer 1) reading."""
    b = operand_bytes(seed)
    v = b.view(np.int8).astype(np.int64) if answer == S8 else (b & 7).astype(np.int64) - 4
    return v[:M * K].reshape(M, K), v[M * K:].reshape(K, N)


def answer(answer_kind: int, seed: int) -> np.ndarray:
    a, b = operands(answer_kind, seed)
    return a @ b


def max_partial_sum(answer_kind: int, seed: int) -> int:
    """Largest |sum over k < k1 of A[m][k] * B[k][n]| over every m, n and prefix k1: the exactness bound on real data."""
    a, b = operands(answer_kind, seed)
    acc = np.zeros((M, N), dtype=np.int64)
    best = 0
    for k in range(K):
        acc += np.outer(a[:, k], b[k, :])
        best = max(best, int(np.abs(acc).max()))
    return best


def fragment():
    """(rows, cols): 256 x 128 arrays, the element of accumulator value j of thread t (the wgmma m64n256 fragment)."""
    t = np.arange(256)[:, None]
    j = np.arange(128)[None, :]
    rows = 64 * (t // 128) + 16 * ((t // 32) % 4) + (t % 32) // 4 + 8 * ((j // 2) % 2)
    cols = 8 * (j // 4) + 2 * (t % 4) + j % 2
    return rows, cols


def thread_folds(tile: np.ndarray) -> np.ndarray:
    """Per thread: sum_j tile[row(t, j)][col(t, j)] * (2j + 1) mod 2^64, as uint64."""
    rows, cols = fragment()
    v = tile[rows, cols].astype(np.int64).astype(np.uint64)
    w = (2 * np.arange(128, dtype=np.uint64) + 1)[None, :]
    with np.errstate(over="ignore"):
        return (v * w).sum(axis=1, dtype=np.uint64)


def cta_fold(tile: np.ndarray, iterations: int = 1) -> int:
    return (int(thread_folds(tile).sum(dtype=np.uint64)) * iterations) & U64


class CComputeOracle:
    """ctypes over oracle/libcompute_oracle.so (built by __graft_entry__.build_oracle from compute_oracle.c)."""

    def __init__(self, path: str = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libcompute_oracle.so")):
        L = ctypes.CDLL(path)
        L.oracle_compute_operand.restype = ctypes.c_int
        L.oracle_compute_operand.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_uint32]
        L.oracle_compute_answer.restype = ctypes.c_int
        L.oracle_compute_answer.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.POINTER(ctypes.c_int32)]
        self.lib = L

    def operand(self, answer_kind: int, seed: int, e: int) -> int:
        return self.lib.oracle_compute_operand(answer_kind, seed, e)

    def answer(self, answer_kind: int, seed: int) -> np.ndarray:
        out = (ctypes.c_int32 * (M * N))()
        assert self.lib.oracle_compute_answer(answer_kind, seed, out) == 0
        return np.frombuffer(out, dtype=np.int32).reshape(M, N).copy()


def annotations(r: Dict) -> Dict[str, str]:
    p = "cohdi.io/probe-compute-"
    if r["status"] == OK:
        verdict = "ok"
    elif r["status"] == ERR_CHECKSUM and r["verdict"] in (SM, ALL):
        verdict = "sm" if r["verdict"] == SM else "all"
    else:
        verdict = "error"
    ran = [i for i in range(5) if (r["legs"] >> i) & 1]
    legs = r["leg"]
    covered = min((legs[i]["sms_covered"] for i in ran), default=0)
    m = {p + "verdict": verdict, p + "sms": "%d/%d" % (covered, r["sm_count"])}
    if r["bad_sms"]:
        m[p + "bad-sms"] = ",".join(str(x) for x in r["bad_sm"][:min(r["bad_sms"], 16)])
    failed = [LEG_NAMES[i] for i in ran
              if legs[i]["mismatches"] or legs[i]["fold_mismatches"] or legs[i]["unpublished"]]
    if failed:
        m[p + "failed-legs"] = ",".join(failed)
    for i, key in ((0, "s8-gops"), (1, "bf16-gflops"), (2, "e4m3-gflops")):
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
    """The classification of a call's rounds and records (oracle/sm_legs.py): every leg computes one M x N x K tile."""
    return sm_legs.classify(call, LEGS, [2 * M * N * K] * LEGS, RECORDS)
