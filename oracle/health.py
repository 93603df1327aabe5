"""Restatement of the health check's stop and status rules (cro_selftest_health_classify) and of its annotations
(cro_emit_health_annotations_json), written from include/croprobe.h ("health").

Checks, bit c in run order: compute, precision, sram, l2, link, scan.  Rules:
  * a check that returns CRO_ERR_CUDA is the last to run; every later selected check is not run;
  * the call's status is CRO_ERR_CHECKSUM when any check returned it, else the first other non-OK status in run order,
    else CRO_OK.

A result is a dict:
  {"status": int, "ran": int, "failed": int, "errored": int, "not_run": int, "incomplete": int, "check_ns": [int] * 6,
   "check_status": [int] * 6, "helper_ns": int, and for each check that ran, under its name, the dict its own
   restatement (compute.py, precision.py, sram.py, l2.py, link.py, scan.py) takes}.
The annotations are every ran check's own, unchanged, and cohdi.io/probe-health-*: -verdict ("ok", "fail" for
CRO_ERR_CHECKSUM, "cuda-error:<cuda_error of the check that returned CRO_ERR_CUDA>" with 0 for the checks whose result
carries none, else "error"), -failed, -errors, -not-run, -incomplete (check names in run order, each only when there is
one) and -ms (helper_ns, or the checks' summed ns when helper_ns is 0, integer ms).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import compute
import l2
import link
import precision
import scan
import sram
from oracle import go_marshal_string_map

OK, ERR_CUDA, ERR_CHECKSUM = 0, -4, -6
NAMES = ["compute", "precision", "sram", "l2", "link", "scan"]
MODULES = [compute, precision, sram, l2, link, scan]
ALL = (1 << len(NAMES)) - 1
HAS_CUDA_ERROR = {"sram", "l2", "scan"}


def classify(checks: int, statuses: List[int]) -> Tuple[Dict, int]:
    """The summary after the first len(statuses) checks to run returned `statuses`, and the bit of the check to run
    next (0: none).  ValueError for bits outside ALL or more statuses than the rules let run."""
    checks = checks or ALL
    if checks & ~ALL:
        raise ValueError("unknown check bits")
    order = [c for c in range(len(NAMES)) if checks >> c & 1]
    s = {"checks": checks, "ran": 0, "failed": 0, "errored": 0, "not_run": 0, "check_status": [0] * len(NAMES)}
    returned = []
    nxt = 0
    for c in order:
        if returned and returned[-1] == ERR_CUDA:
            s["not_run"] |= 1 << c
        elif len(returned) == len(statuses):
            nxt = 1 << c
            break
        else:
            st = statuses[len(returned)]
            returned.append(st)
            s["ran"] |= 1 << c
            s["check_status"][c] = st
            if st == ERR_CHECKSUM:
                s["failed"] |= 1 << c
            elif st != OK:
                s["errored"] |= 1 << c
    if len(returned) < len(statuses):
        raise ValueError("more statuses than checks that run")
    other = [st for st in returned if st not in (OK, ERR_CHECKSUM)]
    s["status"] = ERR_CHECKSUM if ERR_CHECKSUM in returned else other[0] if other else OK
    return s, nxt


def names(mask: int) -> str:
    return ",".join(NAMES[c] for c in range(len(NAMES)) if mask >> c & 1)


def annotations(r: Dict) -> Dict[str, str]:
    m: Dict[str, str] = {}
    for c, mod in enumerate(MODULES):
        if r["ran"] >> c & 1:
            m.update(mod.annotations(r[NAMES[c]]))
    p = "cohdi.io/probe-health-"
    st = r["status"]
    verdict = "ok" if st == OK else "fail" if st == ERR_CHECKSUM else "error"
    if st == ERR_CUDA:
        for c, name in enumerate(NAMES):
            if r["ran"] >> c & 1 and r["check_status"][c] == ERR_CUDA:
                verdict = "cuda-error:%d" % (r[name]["cuda_error"] if name in HAS_CUDA_ERROR else 0)
                break
    m[p + "verdict"] = verdict
    for key, field in (("failed", "failed"), ("errors", "errored"), ("not-run", "not_run"), ("incomplete", "incomplete")):
        if r[field]:
            m[p + key] = names(r[field])
    ns = r["helper_ns"] or sum(r["check_ns"])
    m[p + "ms"] = str(ns // 1000000)
    return m


def annotations_json(r: Dict) -> bytes:
    return go_marshal_string_map(annotations(r)).encode("utf-8")
