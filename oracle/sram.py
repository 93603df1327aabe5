"""Restatement of the SRAM probe's health bits, annotations and M5 closed form (sram_health,
cro_emit_sram_annotations_json, closed_form in sram_probe.cu).

Pure Python over a result given as plain values, so the emitter can be held to it without a GPU.  A result is a dict:
  {"status": int, "verdict": int, "cuda_error": int, "sm_count": int, "legs": int, "bytes_per_sm": int, "health": int,
   "sms_covered": [int] * 2, "bad_sm": [int] (the first min(bad_sms, 16)), "bad_sms": int,
   "bad_pair": [(from, owner, direction)] (the first min(bad_pairs, 8)), "bad_pairs": int, "before": health,
   "after": health}
with health = {"nvml": int, "threshold_exceeded": int, "ecc_corrected": int, "ecc_uncorrected": int}.

Rules (include/croprobe.h, "SRAM"): the verdict is "ok" for status 0, "sm" / "link" / "all" for CRO_ERR_CHECKSUM with
that verdict, "cuda-error:<cuda_error>" for CRO_ERR_CUDA, else "error"; -sms is the least coverage over the legs run;
an ECC delta prints only when both reads answered it (it wraps mod 2^64).
"""
from __future__ import annotations

from typing import Dict, Tuple

from oracle import go_marshal_string_map

OK, ERR_CUDA, ERR_CHECKSUM = 0, -4, -6
NONE, SM, LINK, ALL = 0, 1, 2, 3
DIR_READ, DIR_WRITE = 1, 2
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
