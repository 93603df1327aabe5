"""The register-file probe without a GPU: the ctypes mirrors against the header as gcc lays it out, the kernel as ptxas
and cuobjdump built it (no spills; K registers loaded between two barriers and compared after the third), the emitter
and the classification against oracle/regfile.py, and the helper's argv and frame through a stand-in."""
import ctypes
import importlib.util
import json
import os
import random
import re
import shutil
import stat
import struct
import subprocess
import sys
import tempfile
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
LIB = os.path.join(ROOT, "composable-resource-operator_b200", "libcroprobe.so")
CLI = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
U = "GPU-5ca90000-0000-0000-0000-000000000003"
K, T = 224, 256

FIELDS = {
    "cro_regfile_opts": ("RegfileOpts", ["iterations", "max_rounds", "deadline_ms", "test_inject_sm", "test_inject_warp",
                                         "test_inject_lane", "test_inject_slot", "test_inject_element", "test_inject_iteration",
                                         "test_inject_mask"]),
    "cro_regfile_result": ("RegfileResult", ["status", "verdict", "seed", "call", "sm_count", "nsmid", "cuda_error", "health",
                                             "iterations", "rounds", "slots", "threads", "num_regs", "regs_per_sm",
                                             "sms_covered", "complete", "ctas", "unpublished", "failed_sms", "bad_sms", "bad_sm",
                                             "mismatches", "fold_mismatches", "recorded", "sms_listed", "reserved",
                                             "bits_checked", "ns", "timer_ns", "wall_ns", "helper_ns", "fold_xor", "fold_sum",
                                             "fold_wsum", "expect_xor", "expect_sum", "expect_wsum", "before", "after"]),
    "cro_regfile_sm": ("RegfileSm", ["smid", "mark", "mismatches", "fold_mismatches", "ns", "cycles", "ctas", "reserved"]),
    "cro_regfile_fault": ("RegfileFault", ["element", "iteration", "smid", "warp", "lane", "slot", "expected", "actual"]),
    "cro_regfile_cta": ("RegfileCta", ["stamp", "t0", "t1", "cycles", "count", "last", "fold_x", "fold_s", "fold_w", "smid",
                                       "nsmid", "block", "reserved"]),
}
CONSTANTS = ["CRO_REGFILE_SLOTS", "CRO_REGFILE_THREADS", "CRO_REGFILE_ELEMENTS", "CRO_REGFILE_RECORDS", "CRO_REGFILE_MAX_SMS",
             "CRO_REGFILE_MAX_ITERATIONS", "CRO_REGFILE_MAX_ROUNDS", "CRO_REGFILE_NONE", "CRO_REGFILE_SM", "CRO_REGFILE_ALL",
             "CRO_REGFILE_PERSISTENT", "CRO_REGFILE_INTERMITTENT"]


def test_ctypes_layout_and_constants_match_the_header(cro, tmp_path):
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "croprobe.h"', "int main(void) {"]
    for cname, (_py, fields) in FIELDS.items():
        src.append('printf("%s sizeof %%zu\\n", sizeof(%s));' % (cname, cname))
        for f in fields:
            src.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, f, cname, f))
    for k in CONSTANTS:
        src.append('printf("const %s %%lld\\n", (long long)(%s));' % (k, k))
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
        assert [f for f, *_ in cls._fields_] == fields, cname
        for f in fields:
            assert getattr(cls, f).offset == got[(cname, f)], (cname, f)
    for k in CONSTANTS:
        assert getattr(cro, k[len("CRO_"):]) == got[("const", k)], k


# ---- the kernel as the compiler built it ----------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not installed")
def test_the_kernel_holds_its_words_without_spilling():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC] + FLAGS + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "regfile_kernels.cu"), "-o",
                                             os.path.join(d, "r.o")], capture_output=True, text=True, check=True)
    text = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\S+)'", text)
    assert len(kernels) == 1 and "regfile_kernel" in kernels[0], kernels
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in text, text
    regs = int(re.search(r"Used (\d+) registers", text).group(1))
    assert regs >= 250, regs


INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")
REG = re.compile(r"(?<![\w.])R(\d+)(?![\w])")


def kernel_sass():
    """[(opcode, operand text)] of the register-file kernel in the built library."""
    out, on = [], False
    for ln in subprocess.check_output([CUOBJDUMP, "-sass", LIB], text=True).splitlines():
        if "Function : " in ln:
            on = "regfile_kernel" in ln
            continue
        m = INSN.search(ln)
        if on and m:
            out.append((m.group(3), m.group(4)))
    return out


def width(op):
    return 4 if ".128" in op else 2 if (".64" in op or ".WIDE" in op) else 1


def defs(op, args):
    """Registers an instruction writes: its first operand, unless it is a store, a barrier or a branch."""
    if op.split(".")[0] in ("ST", "STS", "STG", "STL", "RED", "BAR", "BRA", "EXIT", "MEMBAR", "WARPSYNC", "BSYNC", "BSSY",
                            "CALL", "RET", "NOP", "ERRBAR", "CGAERRBAR", "YIELD"):
        return set()
    first = args.split(",")[0]
    m = REG.search(first)
    if not m:
        return set()
    r = int(m.group(1))
    return set(range(r, r + width(op)))


def uses(op, args):
    """Registers an instruction reads (a 64-bit operand reads its pair)."""
    parts = args.split(",")
    srcs = parts if not defs(op, args) else parts[1:]
    out = set()
    for p in srcs:
        for m in REG.finditer(p):
            r = int(m.group(1))
            out |= {r, r + 1} if ("[" not in p and width(op) > 1) else {r}
    return out


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump is not installed")
def test_the_compared_words_are_held_in_registers_not_reloaded(cro):
    """Between the barrier before the loads and the barrier after them, the element's shared loads define exactly K
    distinct registers; no shared load of the source, local load or local store follows until the compares end; and
    every one of the K registers is read after the third barrier before anything writes it again."""
    sass = kernel_sass()
    assert sass
    assert not [op for op, _ in sass if op.split(".")[0] in ("LDL", "STL")], "local memory in the kernel"
    bars = [i for i, (op, _) in enumerate(sass) if op.startswith("BAR.SYNC")]
    # the load window: the first barrier followed by 16-byte shared loads
    b1 = next(b for b in bars if sass[b + 1][0].startswith("LDS.128") or sass[b + 2][0].startswith("LDS.128"))
    b2, b3 = [b for b in bars if b > b1][:2]
    loads = [(op, a) for op, a in sass[b1 + 1:b2] if op.startswith("LDS")]
    held = set()
    for op, a in loads:
        assert op.startswith("LDS.128"), op
        held |= defs(op, a)
    assert len(held) == K and len(loads) == K // 4
    base = {m.group(1) for _, a in loads for m in [re.search(r"\[(R\d+)", a)] if m}
    assert len(base) == 1, base
    # the compares end at the warp vote that decides whether any slot is recorded
    end = next(i for i in range(b3, len(sass)) if sass[i][0].startswith("VOTE.ANY"))
    for op, a in sass[b2 + 1:end]:
        assert op.split(".")[0] not in ("LDL", "STL"), op
        if op.startswith("LDS"):
            assert not set(re.findall(r"\[(R\d+)", a)) & base, ("a shared load of the source", op, a)
    # nothing writes a held register between the loads and the third barrier
    for op, a in sass[b2 + 1:b3]:
        assert not defs(op, a) & held, (op, a)
    # after the third barrier each held register is read before it is written
    pending = set(held)
    for op, a in sass[b3 + 1:end]:
        pending -= uses(op, a)
        assert not defs(op, a) & pending, ("redefined before it was compared", op, a, sorted(defs(op, a) & pending))
    assert not pending, sorted(pending)


# ---- the emitter against oracle/regfile.py --------------------------------------------------------------------------
def health_dict(h):
    return {"nvml": h.nvml, "threshold_exceeded": h.threshold_exceeded, "ecc_corrected": h.ecc_corrected,
            "ecc_uncorrected": h.ecc_uncorrected}


def as_dict(r):
    return {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sms_covered": r.sms_covered,
            "sm_count": r.sm_count, "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm[:min(r.bad_sms, 16)]), "slots": r.slots,
            "threads": r.threads, "regs_per_sm": r.regs_per_sm, "iterations": r.iterations, "health": r.health,
            "before": health_dict(r.before), "after": health_dict(r.after)}


def crafted(cro):
    rng = random.Random(20261017)
    for j in range(400):
        r = cro.RegfileResult()
        r.status = rng.choice([0, -6, -6, -4, -1, -10])
        r.verdict = rng.choice([0, 1, 2, 3])
        r.cuda_error = rng.choice([0, 214, 700])
        r.sm_count, r.sms_covered = 132, rng.choice([132, 131, 0])
        r.bad_sms = rng.choice([0, 1, 5, 16, 17, 132])
        for i in range(16):
            r.bad_sm[i] = rng.randrange(256)
        r.slots, r.threads, r.regs_per_sm = rng.choice([(224, 256, 65536), (0, 0, 0)])
        r.iterations = rng.choice([1, 64, 4096])
        r.health = rng.randrange(8)
        for h in (r.before, r.after):
            h.nvml = rng.randrange(8)
            h.threshold_exceeded = rng.randrange(2)
            h.ecc_corrected, h.ecc_uncorrected = rng.randrange(1 << 64), rng.choice([0, 3, (1 << 64) - 1])
        yield r


def test_emitter_equals_the_restatement(cro):
    import regfile
    for r in crafted(cro):
        assert cro.emit_regfile_annotations_json(r).encode() == regfile.annotations_json(as_dict(r)), as_dict(r)


def test_emitter_spells_the_keys(cro):
    r = cro.RegfileResult()
    r.status, r.verdict, r.sm_count, r.sms_covered, r.bad_sms = -6, 1, 132, 132, 2
    r.bad_sm[0], r.bad_sm[1] = 7, 40
    r.slots, r.threads, r.regs_per_sm, r.iterations = 224, 256, 65536, 64
    got = json.loads(cro.emit_regfile_annotations_json(r))
    assert got == {"cohdi.io/probe-regfile-verdict": "sm", "cohdi.io/probe-regfile-sms": "132/132",
                   "cohdi.io/probe-regfile-bad-sms": "7,40", "cohdi.io/probe-regfile-regs": "57344/65536",
                   "cohdi.io/probe-regfile-iterations": "64"}


# ---- the classification against oracle/regfile.py ------------------------------------------------------------------
def cta_dict(x):
    return {"stamp": x.stamp, "t0": x.t0, "t1": x.t1, "cycles": x.cycles, "count": list(x.count), "last": x.last,
            "fold": (x.fold_x, x.fold_s, x.fold_w), "smid": x.smid, "nsmid": x.nsmid}


def rec_dict(f):
    return {k: getattr(f, k) for k, _ in f._fields_}


def make_call(cro, rng, case):
    import regfile
    sm_count, iterations, call = rng.choice([(132, 1, 0), (132, 4, 3), (8, 2, 1), (1, 3, 9)])
    seed = rng.randrange(1 << 64)
    good = regfile.fold(seed, iterations)
    n_rounds = rng.choice([1, 1, 2, 3])
    smids = rng.sample(range(sm_count + 4), sm_count)
    rounds = []
    for _ in range(n_rounds):
        rnd = []
        for j in range(sm_count):
            x = cro.RegfileCta()
            x.stamp, x.t0, x.t1, x.cycles = call, 1000 + j, 2000 + rng.randrange(99), rng.randrange(1 << 30)
            x.fold_x, x.fold_s, x.fold_w = good
            x.smid, x.nsmid, x.block = smids[j] if rng.random() < 0.9 else rng.choice(smids), 140, j
            rnd.append(x)
        rounds.append(rnd)
    flat = [x for rnd in rounds for x in rnd]
    bad = flat if case == "every" else [rng.choice(flat)] if case in ("one", "fold", "overflow") else []
    for x in bad:
        if case == "fold":
            x.fold_s ^= 1
            continue
        e = rng.randrange(2)
        x.count[e] = rng.randrange(1, 5) if case != "overflow" else K * T
        x.last = rng.choice([0, x.count[e]])
    if case == "silent":
        rng.choice(flat).stamp = (1 << 64) - 1
    if case == "nsmid":
        rng.choice(flat).nsmid = 300
    claims = {"overflow": 5000, "every": rng.randrange(0, 50)}.get(case, rng.randrange(0, 4) if bad else 0)
    recs = []
    for _ in range(min(claims, cro.REGFILE_RECORDS)):
        f = cro.RegfileFault()
        f.element, f.iteration, f.smid = rng.randrange(2), rng.randrange(iterations), rng.choice(smids)
        f.warp, f.lane, f.slot = rng.randrange(8), rng.randrange(32), rng.randrange(K)
        f.expected, f.actual = rng.randrange(1 << 32), rng.randrange(1 << 32)
        recs.append(f)
    return dict(seed=seed, call=call, iterations=iterations, sm_count=sm_count, rounds=rounds, claims=claims, records=recs)


@pytest.mark.parametrize("case", ["clean", "one", "every", "fold", "silent", "overflow", "nsmid"])
def test_classification_equals_the_restatement(cro, case):
    import regfile
    rng = random.Random(hash(case) & 0xFFFF)
    for _ in range(6):
        c = make_call(cro, rng, case)
        r, sms, faults = cro.selftest_regfile_classify(c["iterations"], c["seed"], c["sm_count"], c["call"], c["rounds"],
                                                       c["claims"], c["records"])
        want, wsms, wrecs = regfile.classify(dict(c, rounds=[[cta_dict(x) for x in rnd] for rnd in c["rounds"]],
                                                  records=[rec_dict(f) for f in c["records"]]))
        assert r.status == want["status"], case
        if case == "nsmid":
            assert r.status == cro.ERR_UNSUPPORTED and not sms and not faults
            continue
        for k in ("verdict", "seed", "call", "sm_count", "nsmid", "iterations", "rounds", "sms_covered", "complete", "ctas",
                  "unpublished", "failed_sms", "bad_sms", "fold_mismatches", "bits_checked", "timer_ns"):
            assert getattr(r, k) == want[k], (case, k, getattr(r, k), want[k])
        assert list(r.bad_sm[:min(r.bad_sms, 16)]) == want["bad_sm"] and list(r.mismatches) == want["mismatches"]
        assert r.fold == want["fold"] and r.expect == want["expect"]
        assert [{k: getattr(s, k) if k != "mismatches" else list(s.mismatches) for k in w} for s, w in zip(sms, wsms)] == wsms
        assert len(sms) == len(wsms) == r.sms_listed
        assert [rec_dict(f) for f in faults] == wrecs and r.recorded == len(wrecs)
        if case == "every":
            assert r.verdict == cro.REGFILE_ALL
        if case in ("one", "fold", "overflow"):
            assert r.verdict in (cro.REGFILE_SM, cro.REGFILE_ALL) and r.status == cro.ERR_CHECKSUM
        if case == "silent":
            assert r.verdict == cro.REGFILE_ALL and r.unpublished == 1
        if case == "overflow":
            assert r.recorded == cro.REGFILE_RECORDS


def test_the_closed_form_is_the_last_iterations_complement(cro):
    import regfile
    from oracle import pattern_word
    seed = 0x1234_5678_9ABC_DEF0
    x = s = w = 0
    si = (seed + 2 * regfile.STRIDE) & regfile.U64
    for t in range(T):
        for k in range(K):
            v = ~pattern_word(si, t * K + k) & 0xFFFFFFFF
            x ^= v
            s += v
            w += v * (2 * k + 1)
    assert regfile.fold(seed, 3) == (x, s & regfile.U64, w & regfile.U64)
    r, _, _ = cro.selftest_regfile_classify(3, seed, 1, 0, [], 0, [])
    assert r.expect == (x, s & regfile.U64, w & regfile.U64)


def test_null_arguments_are_refused(cro):
    r, sms, faults = cro.RegfileResult(), (cro.RegfileSm * 4)(), (cro.RegfileFault * 4)()
    ks, k = ctypes.c_int(), ctypes.c_int()
    assert cro.lib.cro_emit_regfile_annotations_json(None, None, 0, None) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_regfile(None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                     ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_probe_regfile_uuid(None, None, None, ctypes.byref(r), sms, 4, ctypes.byref(ks), faults, 4,
                                          ctypes.byref(k)) == cro.ERR_INVALID_ARG
    for it in (0, cro.REGFILE_MAX_ITERATIONS + 1):
        assert cro.lib.cro_selftest_regfile_classify(it, 0, 1, 0, 0, None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks),
                                                     faults, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG
    assert cro.lib.cro_selftest_regfile_classify(1, 0, 0, 0, 0, None, 0, None, ctypes.byref(r), sms, 4, ctypes.byref(ks),
                                                 faults, 4, ctypes.byref(k)) == cro.ERR_INVALID_ARG


# ---- the helper wire: the table against cro_regfile_opts, and the argument count -------------------------------------
def test_wire_table_covers_the_options_and_round_trips(tmp_path):
    spec = importlib.util.spec_from_file_location("helper_wire_program", os.path.join(HERE, "test_helper_wire.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    body = ('    { const size_t at[] = {offsetof(cro_regfile_opts, deadline_ms)}, size[] = {sizeof(int32_t)}; '
            'check("regfile", &cro_wire_regfile, sizeof(cro_regfile_opts), at, size, 1); }')
    src = tmp_path / "wire.c"
    src.write_text(mod.PROGRAM.replace("@BODY@", body))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    assert "argc regfile-raw 14" in out.stdout


def test_cli_takes_exactly_its_argument_count():
    run = lambda k: subprocess.run([CLI, "regfile-raw", U] + ["0"] * (k - 3), capture_output=True, timeout=60).returncode
    assert run(13) == 64 and run(15) == 64
    assert run(14) != 64


# ---- the helper through a stand-in: argv, seed bases, frame, failures, deadline, refusals ----------------------------
def fake_helper(tmp_path, body):
    p = os.path.join(str(tmp_path), "fake-croprobe-cli")
    with open(p, "w") as f:
        f.write("#!%s\n" % sys.executable + body)
    os.chmod(p, os.stat(p).st_mode | stat.S_IXUSR)
    return p


HELPER = """
import os, struct, sys
assert sys.argv[1] == "regfile-raw" and os.environ["CUDA_VISIBLE_DEVICES"] == sys.argv[2] and len(sys.argv) == 14, sys.argv
open(%(log)r, "a").write(" ".join(sys.argv[1:]) + "\\n")
seed_base, iters, rounds, sm, warp, lane, slot, element, iteration, mask, cap = map(int, sys.argv[3:])
n = min(cap, 3)
r = bytearray(296)
struct.pack_into("<iIQQII", r, 0, -6, 1, 1234, 0, 132, 132)
struct.pack_into("<IIIIII", r, 40, iters, 1, 224, 256, 255, 65536)
struct.pack_into("<IIIIII", r, 64, 132, 1, 132, 0, 1, 1)
struct.pack_into("<H", r, 88, sm)
struct.pack_into("<QQQQ", r, 120, n, 0, 0, n)
struct.pack_into("<I", r, 152, %(listed)d)
sms = bytearray(256 * 56)
struct.pack_into("<II", sms, 0, 3, 0)
struct.pack_into("<II", sms, 56, sm, 1)
faults = b"".join(struct.pack("<8I", element, iteration, sm, warp, lane, slot + j, 5, 5 ^ mask) for j in range(n))
sys.stdout.buffer.write(bytes(r) + bytes(sms) + faults + b"%(extra)s")
sys.exit(1)
"""


def helper(tmp_path, listed=2, extra=""):
    log = str(tmp_path / "argv.log")
    return fake_helper(tmp_path, HELPER % {"log": log, "listed": listed, "extra": extra}), log


def test_helper_argv_frame_and_fresh_seed_bases(cro, tmp_path, monkeypatch):
    path, log = helper(tmp_path)
    monkeypatch.setenv("CRO_HELPER_PATH", path)
    r, sms, faults = cro.probe_regfile_uuid(None, U, iterations=3, inject=(9, 2, 17, 200, 1, 2, 1 << 31))
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.REGFILE_SM and r.seed == 1234 and r.num_regs == 255
    assert list(r.bad_sm[:r.bad_sms]) == [9] and r.helper_ns > 0 and r.recorded == 3 and r.sms_listed == 2
    assert [s.smid for s in sms] == [3, 9] and sms[1].mark == cro.REGFILE_PERSISTENT
    assert [(f.element, f.iteration, f.smid, f.warp, f.lane, f.slot, f.expected, f.actual) for f in faults] == \
        [(1, 2, 9, 2, 17, 200 + j, 5, 5 ^ (1 << 31)) for j in range(3)]
    r, sms, faults = cro.probe_regfile_uuid(None, U, cap=2)                    # the helper is asked for at most cap records
    assert len(faults) == 2 and r.recorded == 2
    lines = open(log).read().split("\n")[:2]
    a, b = (ln.split() for ln in lines)
    assert a[0] == "regfile-raw" and a[1] == U and a[3:] == ["3", "0", "9", "2", "17", "200", "1", "2", str(1 << 31), "256"]
    assert b[3:] == ["0", "0", "0", "0", "0", "0", "0", "0", "0", "2"]
    assert a[2] != b[2] and int(a[2]) & 0xFF == 0 and int(b[2]) & 0xFF == 0, (a[2], b[2])


def test_malformed_helper_frames_are_errors(cro, tmp_path, monkeypatch):
    for listed, extra in ((2, "x"), (cro.REGFILE_MAX_SMS + 1, "")):
        path, _ = helper(tmp_path, listed, extra)
        monkeypatch.setenv("CRO_HELPER_PATH", path)
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_regfile_uuid(None, U)
        assert e.value.code == cro.ERR_EXEC and "register-file helper for %s failed" % U in str(e.value)
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.stdout.buffer.write(b'short')\nsys.exit(1)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_regfile_uuid(None, U)
    assert e.value.code == cro.ERR_EXEC
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import sys\nsys.exit(3)\n"))
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_regfile_uuid(None, U)
    assert e.value.code == cro.ERR_NO_DEVICE


def test_wedged_helper_is_killed_at_its_deadline(cro, tmp_path, monkeypatch):
    marker = tmp_path / "pid"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "import os, time\nopen(%r, 'w').write(str(os.getpid()))\n"
                                                                  "time.sleep(60)\n" % str(marker)))
    t0 = time.monotonic()
    with pytest.raises(cro.ProbeError) as e:
        cro.probe_regfile_uuid(None, U, deadline_ms=300)
    assert e.value.code == cro.ERR_DEADLINE and "register-file helper" in str(e.value) and "was killed" in str(e.value)
    assert time.monotonic() - t0 < 5
    pid = int(marker.read_text())
    with pytest.raises(ProcessLookupError):
        os.kill(pid, 0)


def test_bad_options_are_refused_before_any_spawn(cro, tmp_path, monkeypatch):
    marker = tmp_path / "spawned"
    monkeypatch.setenv("CRO_HELPER_PATH", fake_helper(tmp_path, "open(%r, 'w').write('1')\n" % str(marker)))
    calls = [dict(iterations=cro.REGFILE_MAX_ITERATIONS + 1), dict(max_rounds=cro.REGFILE_MAX_ROUNDS + 1), dict(deadline_ms=-1),
             dict(inject=(256, 0, 0, 0, 0, 0, 1)), dict(inject=(0, 8, 0, 0, 0, 0, 1)), dict(inject=(0, 0, 32, 0, 0, 0, 1)),
             dict(inject=(0, 0, 0, 224, 0, 0, 1)), dict(inject=(0, 0, 0, 0, 2, 0, 1)),
             dict(inject=(0, 0, 0, 0, 0, 3, 1), iterations=3), dict(inject=(-2, 0, 0, 0, 0, 0, 1))]
    for kw in calls:
        with pytest.raises(cro.ProbeError) as e:
            cro.probe_regfile_uuid(None, U, **kw)
        assert e.value.code == cro.ERR_INVALID_ARG, kw
    assert not marker.exists()
