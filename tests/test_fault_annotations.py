"""The fault locator's C structs and annotation emitter, without a GPU.

The ctypes mirrors of cro_locate_opts / cro_fault_word / cro_locate_pass / cro_fault_report are held to the header as
gcc lays it out, and cro_emit_fault_annotations_json is held byte for byte to oracle/faults.py on crafted reports."""
import ctypes
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = {
    "cro_locate_opts": ("LocateOpts", ["flags", "reserved0", "test_force_first", "test_force_count", "test_force_and",
                                       "test_force_or"]),
    "cro_fault_word": ("FaultWord", ["word_index", "expected", "actual", "passes", "reserved"]),
    "cro_locate_pass": ("LocatePass", ["halves", "skipped", "seed", "invert", "words_scanned", "mismatches", "recorded",
                                       "granules", "scan_ns", "fold_xor", "fold_sum", "fold_wsum"]),
    "cro_fault_report": ("FaultReport", ["status", "verdict", "n_passes", "complete", "sweep_bytes", "retest_seed",
                                         "located", "recorded", "flip_or", "bit_flips", "pass"]),
}


def test_ctypes_layout_matches_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    got = {}
    for ln in subprocess.check_output([str(exe)], text=True).splitlines():
        name, field, v = ln.split()
        got[(name, field)] = int(v)
    for cname, (py, fields) in FIELDS.items():
        cls = getattr(cro, py)
        assert ctypes.sizeof(cls) == got[(cname, "sizeof")], cname
        for f in fields:
            assert getattr(cls, "pass_" if f == "pass" else f).offset == got[(cname, f)], (cname, f)


def make_report(cro, n_passes, mism, gran, bits):
    r = cro.FaultReport()
    r.n_passes = n_passes
    for p in range(len(mism)):
        r.pass_[p].mismatches = mism[p]
        r.pass_[p].granules = gran[p]
    for b, v in enumerate(bits):
        r.bit_flips[b] = v
    return r


def as_dict(r):
    return {"n_passes": r.n_passes, "pass": [{"mismatches": p.mismatches, "granules": p.granules} for p in r.pass_],
            "bit_flips": list(r.bit_flips)}


def crafted(cro):
    rng = random.Random(20261015)
    zero = [0] * 64
    yield make_report(cro, 1, [0, 0, 0], [0, 0, 0], zero), []                          # clean, no retest
    yield make_report(cro, 3, [0, 0, 0], [0, 0, 0], zero), []                          # clean with retest
    yield make_report(cro, 0, [0, 0, 0], [0, 0, 0], zero), []                          # empty report (a failed call)
    yield make_report(cro, 1, [1, 0, 0], [1, 0, 0], [1] + [0] * 63), [(7, 5, 4)]       # unclassified
    yield make_report(cro, 3, [1, 0, 0], [1, 0, 0], [1] + [0] * 63), [(7, 5, 4)]       # not reproduced
    yield make_report(cro, 3, [0, 2, 0], [0, 1, 0], zero[:63] + [2]), [(1, 0, 1 << 63), (2, 0, 1 << 63)]   # persistent
    yield make_report(cro, 3, [0, 0, 1], [0, 0, 1], zero), [(0, ~0 & (2**64 - 1), 0)]
    yield make_report(cro, 7, [3, 0, 0], [2, 0, 0], zero), []                          # n_passes past the array
    for _ in range(400):
        np_ = rng.choice([0, 1, 3, 2, 5])
        mism = [rng.choice([0, 0, 1, rng.randrange(1, 1 << 40), 2**64 - 1]) for _ in range(3)]
        gran = [rng.randrange(0, 40961) for _ in range(3)]
        bits = [rng.choice([0, 0, 0, rng.randrange(1, 1 << 33)]) for _ in range(64)]
        n = rng.choice([0, 1, 5, 8, 9, 40])        # more than 8 words: the list is truncated to 8
        words = sorted({(rng.randrange(0, 1 << 40), rng.getrandbits(64), rng.getrandbits(64)) for _ in range(n)})
        yield make_report(cro, np_, mism, gran, bits), words


def test_emitter_equals_the_restatement(cro):
    import faults
    seen = set()
    for rep, words in crafted(cro):
        arr = [cro.FaultWord(w, e, a, 1, 0) for w, e, a in words]
        got = cro.emit_fault_annotations_json(rep, arr).encode()
        want = faults.annotations_json(as_dict(rep), words)
        assert got == want, (got, want)
        seen.add(faults.verdict(as_dict(rep)))
    assert seen == {faults.NONE, faults.UNCLASSIFIED, faults.NOT_REPRODUCED, faults.PERSISTENT}


def test_emitter_rejects_bad_arguments(cro):
    buf = ctypes.create_string_buffer(64)
    n = ctypes.c_size_t()
    r = cro.FaultReport()
    assert cro.lib.cro_emit_fault_annotations_json(None, None, 0, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_emit_fault_annotations_json(ctypes.byref(r), None, 1, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_emit_fault_annotations_json(ctypes.byref(r), None, -1, buf, 64, ctypes.byref(n)) == cro.ERR_INVALID_ARG


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_locate_without_a_context_is_refused(cro):
    r = cro.FaultReport()
    n = ctypes.c_int(-1)
    words = (cro.FaultWord * 4)()
    assert cro.lib.cro_locate_faults(None, 0, None, ctypes.byref(r), words, 4, ctypes.byref(n)) == cro.ERR_INVALID_ARG
