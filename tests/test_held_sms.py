"""Every per-SM probe on one H100 with part of the GPU held busy, against the restatements in oracle/ and the C oracle.

On an idle device round 1 of a probe covers every SM and each SM runs one CTA, so the coverage rounds, the per-SM CTA
counts of an SM that ran two CTAs of one launch and the short-coverage verdicts never run on a device.  Here
tests/sm_holder.cu keeps k SMs busy from this process and context (one CTA per SM asking for the whole opt-in shared
memory, so nothing else fits beside it) for at most HOLD_NS, and every probe is checked under that hold: it covers
exactly the SMs the holder left free, counts every CTA it ran, stays clean, names a free SM it was told to fail, and
cannot name a held one.  The holder is released in a `finally` after each call; a hold that cannot get all k CTAs
resident within 2 s fails the test.

Faults come only from the probes' software injection; nothing here repeats a call to catch a real one."""
import contextlib
import ctypes
import json
import os
import subprocess
import time

import numpy as np
import pytest

import test_compute_abi
import test_health_abi
import test_regfile_abi
import test_sram_abi
from test_alu_probe import INJECT as ALU_INJECT
from test_compute_probe import INT_MASK
from test_compute_probe import injected as compute_injected
from test_compute_probe import tiles as compute_tiles
from test_precision_probe import EXP_MASK as PRECISION_MASK
from test_precision_probe import answers as precision_answers
from test_sparse_probe import EXP_MASK as SPARSE_MASK
from test_sparse_probe import answers as sparse_answers
from test_warpmma_probe import EXP_MASK as WARPMMA_MASK
from test_warpmma_probe import answers as warpmma_answers
from test_xlane_probe import INJECT as XLANE_INJECT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOLDER_SRC = os.path.join(ROOT, "tests", "sm_holder.cu")
HOLD_NS = 2 * 10 ** 9              # the longest a hold lasts; every test releases it as soon as its call returns
K = 8
MIB = 1 << 20
gpu = pytest.mark.gpu
NONE, SM, ALL = 0, 1, 2            # the per-SM probes' verdicts (oracle/sm_legs.py, oracle/xlane.py, oracle/regfile.py)


def holder_cmd(out, *extra):
    import __graft_entry__ as g
    return [g._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
            "-cudart", "static", *extra, "-o", out, HOLDER_SRC]


def test_the_holder_compiles_for_sm_90a_without_spills(tmp_path):
    """A broken holder shows up without a GPU: it compiles, exports its entry points and its kernel does not spill."""
    out = str(tmp_path / "sm_holder.so")
    p = subprocess.run(holder_cmd(out, "-Xptxas", "-v"), capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert "hold_sm" in p.stderr and "Compiling entry function" in p.stderr, p.stderr
    assert " 0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in p.stderr, p.stderr
    lib = ctypes.CDLL(out)
    for name in ("holder_hold", "holder_release", "holder_smem_bytes", "holder_error"):
        assert hasattr(lib, name), name


class Holder:
    def __init__(self, so):
        self.lib = ctypes.CDLL(so)
        self.lib.holder_hold.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_uint)]
        self.lib.holder_error.restype = ctypes.c_char_p

    @contextlib.contextmanager
    def hold(self, k, hold_ns=HOLD_NS):
        smids = (ctypes.c_uint * k)()
        if self.lib.holder_hold(0, k, hold_ns, smids) != 0:
            pytest.fail("the SM holder failed: " + self.lib.holder_error().decode())
        try:
            H = set(smids)
            assert len(H) == k, ("two holding CTAs shared an SM: the shared-memory request did not fill it", list(smids))
            yield H
        finally:
            assert self.lib.holder_release() == 0, self.lib.holder_error().decode()


@pytest.fixture(scope="module")
def holder(tmp_path_factory, _built):
    out = str(tmp_path_factory.mktemp("holder") / "sm_holder.so")
    subprocess.check_call(holder_cmd(out))
    h = Holder(out)
    try:
        yield h
    finally:
        h.lib.holder_release()


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 * MIB, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def n(ctx):
    return ctx.own_devices()[0].sm_count


@pytest.fixture(scope="module")
def every_sm(ctx, n):
    """ALL: the SMs one clean call on the idle device covers."""
    _, sms, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1, legs=1)
    got = {s.smid for s in sms}
    assert len(got) == n
    return got


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def held(holder, k, fn):
    """fn() under a hold of k SMs: (H, fn's result, wall seconds of the call)."""
    with holder.hold(k) as H:
        out, t = timed(fn)
    return H, out, t


def report(name, k, H, rounds, covered, max_ctas, t_held, t_free):
    print("%s: k %d, H %s, rounds %d, sms_covered %d, max ctas %d, held %.1f ms, unheld %.1f ms"
          % (name, k, sorted(H), rounds, covered, max_ctas, t_held * 1e3, t_free * 1e3))


# ---- the four probes of oracle/sm_legs.py: compute, precision, sparse, warp-MMA -------------------------------------
def _sm_legs_probes(cro):
    import compute
    import precision
    import sparse
    import warpmma
    return {
        "compute": dict(call=lambda ctx, **kw: ctx.probe_compute(0, alu_iterations=2, **kw), leg=0, mask=INT_MASK, rc=(77, 133),
                        fold=lambda seed, leg, it: compute.cta_fold(compute_tiles(compute.CComputeOracle(), seed)[compute.LEG_ANSWER[leg]], it),
                        ops=lambda leg: 2 * compute.M * compute.N * compute.K, emit=cro.emit_compute_annotations_json, mod=compute),
        "precision": dict(call=lambda ctx, **kw: ctx.probe_precision(0, alu_iterations=2, **kw), leg=0, mask=PRECISION_MASK[0],
                          rc=(5, 7), fold=lambda seed, leg, it: precision.cta_fold(leg, precision_answers(seed)[precision.LEG_ANSWER[leg]], it),
                          ops=lambda leg: 2 * np.prod(precision.SHAPE[precision.LEG_ANSWER[leg]], dtype=object),
                          emit=cro.emit_precision_annotations_json, mod=precision),
        "sparse": dict(call=lambda ctx, **kw: ctx.probe_sparse(0, **kw), leg=0, mask=SPARSE_MASK, rc=(5, 7),
                       fold=lambda seed, leg, it: sparse.cta_fold(leg, sparse_answers(seed)[sparse.LEG_ANSWER[leg]], it),
                       ops=lambda leg: 2 * sparse.M * sparse.N * sparse.K[sparse.LEG_ANSWER[leg]],
                       emit=cro.emit_sparse_annotations_json, mod=sparse),
        "warpmma": dict(call=lambda ctx, **kw: ctx.probe_warpmma(0, **kw), leg=0, mask=WARPMMA_MASK[0], rc=(5, 7),
                        fold=lambda seed, leg, it: warpmma.cta_fold(leg, warpmma_answers(seed)[warpmma.LEG_ANSWER[leg]], it),
                        ops=lambda leg: warpmma.ops(leg), emit=cro.emit_warpmma_annotations_json, mod=warpmma),
    }


SM_LEGS = ["compute", "precision", "sparse", "warpmma"]
ITER = 2


def check_sm_legs_coverage(P, r, sms, H, every, n, k, leg, rounds):
    L = r.leg[leg]
    per = {s.smid: s.leg[leg].ctas for s in sms if s.leg[leg].ctas}
    assert set(per) == every - H and not set(per) & H, (sorted(set(per) & H), sorted(every - H - set(per)))
    assert L.sms_covered == n - k and L.complete == 0 and L.rounds == rounds
    assert L.ctas == n * rounds == sum(per.values()) and max(per.values()) >= 2 and L.unpublished == 0
    assert L.ops == P["ops"](leg) * L.iterations * L.ctas
    return per


@pytest.mark.parametrize("max_rounds", [1, 0], ids=["rounds1", "rounds-default"])
@pytest.mark.parametrize("name", SM_LEGS)
@gpu
def test_sm_legs_probe_covers_exactly_the_free_sms(cro, ctx, holder, n, every_sm, name, max_rounds):
    P = _sm_legs_probes(cro)[name]
    leg = P["leg"]
    (_, _, _), t_free = timed(lambda: P["call"](ctx, iterations=ITER, legs=1 << leg, max_rounds=max_rounds))
    H, (r, sms, faults), t = held(holder, K, lambda: P["call"](ctx, iterations=ITER, legs=1 << leg, max_rounds=max_rounds))
    rounds = max_rounds or 4
    per = check_sm_legs_coverage(P, r, sms, H, every_sm, n, K, leg, rounds)
    L = r.leg[leg]
    assert r.status == cro.OK and r.verdict == NONE and not faults and r.bad_sms == 0
    assert L.mismatches == L.fold_mismatches == L.recorded == L.failed_sms == 0
    assert L.fold == L.expect_fold == P["fold"](r.seed, leg, ITER)
    assert json.loads(P["emit"](r)) == P["mod"].annotations(test_compute_abi.as_dict(r))
    report(name, K, H, L.rounds, L.sms_covered, max(per.values()), t, t_free)


@pytest.mark.parametrize("where", ["free", "held", "every"])
@pytest.mark.parametrize("name", SM_LEGS)
@gpu
def test_sm_legs_injection_under_a_hold(cro, ctx, holder, n, every_sm, name, where):
    P = _sm_legs_probes(cro)[name]
    leg, (row, col) = P["leg"], P["rc"]
    with holder.hold(K) as H:
        smid = {"free": min(every_sm - H), "held": min(H), "every": -1}[where]
        r, sms, faults = P["call"](ctx, iterations=ITER, legs=1 << leg, inject=(leg, smid, ITER - 1, row, col, P["mask"]))
    per = check_sm_legs_coverage(P, r, sms, H, every_sm, n, K, leg, 4)
    L = r.leg[leg]
    if where == "held":              # the CTAs that would fail never ran there: a clean call whose coverage was short
        assert r.status == cro.OK and r.verdict == NONE and not faults and L.failed_sms == 0
        ann = json.loads(P["emit"](r))
        assert ann == P["mod"].annotations(test_compute_abi.as_dict(r))
        assert ann["cohdi.io/probe-%s-sms" % name] == "%d/%d" % (n - K, n)
        return
    if where == "every":
        assert r.status == cro.ERR_CHECKSUM and r.verdict == ALL
        assert L.failed_sms == L.sms_covered == n - K and L.mismatches == L.ctas
        return
    ctas = per[smid]
    assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and r.bad_sms == 1 and r.bad_sm[0] == smid
    assert L.failed_sms == 1 and L.mismatches == L.fold_mismatches == L.recorded == ctas
    assert [(f.leg, f.smid, f.row, f.col) for f in faults] == [(leg, smid, row, col)] * ctas
    if name == "compute":
        import compute
        v = int(compute_tiles(compute.CComputeOracle(), r.seed)[compute.LEG_ANSWER[leg]][row, col])
        assert [(f.expected, f.actual) for f in faults] == [(v, compute_injected(cro, leg, v, P["mask"]))] * ctas
    assert json.loads(P["emit"](r)) == P["mod"].annotations(test_compute_abi.as_dict(r))


# ---- the per-thread probes: cross-lane and ALU ------------------------------------------------------------------
def _lane_probes(cro):
    import alu
    import xlane
    return {
        "xlane": dict(call=lambda ctx, **kw: ctx.probe_xlane(0, **kw), ops=cro.XLANE_OPS, legs=cro.XLANE_LEGS,
                      fold=lambda seed, leg, it: xlane.fold(leg, seed, it), emit=cro.emit_xlane_annotations_json, mod=xlane,
                      inject=lambda leg, smid, it: (leg, smid, 3, 17, XLANE_INJECT[leg][0], it, XLANE_INJECT[leg][1]),
                      want=lambda r, leg, it: xlane.injected(leg, r.seed, it, XLANE_INJECT[leg][0], 3, 17, XLANE_INJECT[leg][1])),
        "alu": dict(call=lambda ctx, **kw: ctx.probe_alu(0, **kw), ops=cro.ALU_OPS, legs=cro.ALU_LEGS,
                    fold=lambda seed, leg, it: alu.fold(leg, seed), emit=cro.emit_alu_annotations_json, mod=alu,
                    inject=lambda leg, smid, it: (leg, smid, 3, 17, ALU_INJECT[leg][0], it, ALU_INJECT[leg][1], ALU_INJECT[leg][2]),
                    want=lambda r, leg, it: alu.injected(leg, r.seed, ALU_INJECT[leg][0], 3, 17, ALU_INJECT[leg][1], ALU_INJECT[leg][2])),
    }


def lane_dict(r):
    return {"status": r.status, "verdict": r.verdict, "cuda_error": r.cuda_error, "sms_covered": r.sms_covered,
            "sm_count": r.sm_count, "bad_sms": r.bad_sms, "bad_sm": list(r.bad_sm[:min(r.bad_sms, 16)]),
            "failed_legs": r.failed_legs, "iterations": r.iterations}


def check_lane_coverage(P, r, sms, H, every, n, k, legs, rounds):
    per = {s.smid: s.ctas for s in sms if s.ctas}
    assert set(per) == every - H and not set(per) & H, (sorted(set(per) & H), sorted(every - H - set(per)))
    assert r.sms_covered == n - k and r.complete == 0 and r.rounds == rounds * bin(legs).count("1")
    assert r.ctas == n * r.rounds == sum(per.values()) and max(per.values()) >= 2
    assert r.unpublished == 0 and r.threads_unpublished == 0
    for leg in range(P["legs"]):
        if legs >> leg & 1:       # every CTA that ran checked every op of its 256 threads each iteration, exactly
            assert r.ops_checked[leg] == P["ops"][leg] * 256 * r.iterations * n * rounds, leg
    return per


LANE_LEGS = [(name, leg) for name in ("xlane", "alu") for leg in range(5)]


@pytest.mark.parametrize("max_rounds", [1, 0], ids=["rounds1", "rounds-default"])
@pytest.mark.parametrize("name,leg", LANE_LEGS)
@gpu
def test_lane_probe_covers_exactly_the_free_sms(cro, ctx, holder, n, every_sm, name, leg, max_rounds):
    P = _lane_probes(cro)[name]
    (_, _, _), t_free = timed(lambda: P["call"](ctx, iterations=1, legs=1 << leg, max_rounds=max_rounds))
    H, (r, sms, faults), t = held(holder, K, lambda: P["call"](ctx, iterations=1, legs=1 << leg, max_rounds=max_rounds))
    rounds = max_rounds or 4
    per = check_lane_coverage(P, r, sms, H, every_sm, n, K, 1 << leg, rounds)
    assert r.status == cro.OK and r.verdict == NONE and not faults and r.bad_sms == 0 and r.failed_legs == 0
    assert r.mismatches[leg] == r.fold_mismatches[leg] == r.recorded == 0
    assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == P["fold"](r.seed, leg, 1)
    assert all(s.mark == 0 and s.fold_mismatches == 0 for s in sms)
    assert json.loads(P["emit"](r)) == P["mod"].annotations(lane_dict(r))
    report("%s leg %d" % (name, leg), K, H, r.rounds, r.sms_covered, max(per.values()), t, t_free)


@pytest.mark.parametrize("where", ["free", "held", "every"])
@pytest.mark.parametrize("name", ["xlane", "alu"])
@gpu
def test_lane_injection_under_a_hold(cro, ctx, holder, n, every_sm, name, where):
    P = _lane_probes(cro)[name]
    leg, iterations = 2, 2
    with holder.hold(K) as H:
        smid = {"free": max(every_sm - H), "held": max(H), "every": -1}[where]
        r, sms, faults = P["call"](ctx, iterations=iterations, legs=1 << leg, inject=P["inject"](leg, smid, iterations - 1),
                                   cap=4096)
    per = check_lane_coverage(P, r, sms, H, every_sm, n, K, 1 << leg, 4)
    if where == "held":
        assert r.status == cro.OK and r.verdict == NONE and not faults and r.failed_sms == 0
        ann = json.loads(P["emit"](r))
        assert ann == P["mod"].annotations(lane_dict(r)) and ann["cohdi.io/probe-%s-sms" % name] == "%d/%d" % (n - K, n)
        return
    if where == "every":
        assert r.status == cro.ERR_CHECKSUM and r.verdict == ALL and r.failed_sms == r.sms_covered == n - K
        return
    ctas = per[smid]
    assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and r.bad_sms == 1 and r.bad_sm[0] == smid
    assert r.failed_legs == 1 << leg and r.fold_mismatches[leg] == ctas and r.mismatches[leg] == ctas * len(_want_lanes(P, r, leg))
    got = {}
    for f in faults:
        assert (f.leg, f.smid, f.iteration) == (leg, smid, iterations - 1)
        got[(f.warp, f.lane)] = got.get((f.warp, f.lane), 0) + 1
    assert got == {wl: ctas for wl in _want_lanes(P, r, leg)}
    assert json.loads(P["emit"](r)) == P["mod"].annotations(lane_dict(r))


def _want_lanes(P, r, leg):
    """The (warp, lane) records one CTA makes for the injection: the restatement's injected(...)."""
    w = P["want"](r, leg, 1)
    return set(w) if isinstance(w, dict) else {(3, 17)}


# ---- the register-file probe --------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["none", "free", "held", "every"])
@gpu
def test_regfile_under_a_hold(cro, ctx, holder, n, every_sm, where):
    import regfile
    BIT = 1 << 19
    (_, _, _), t_free = timed(lambda: ctx.probe_regfile(0, iterations=1))
    with holder.hold(K) as H:
        smid = {"none": None, "free": min(every_sm - H), "held": min(H), "every": -1}[where]
        inj = None if smid is None else (smid, 3, 17, 100, 0, 0, BIT)
        (r, sms, faults), t = timed(lambda: ctx.probe_regfile(0, iterations=1, inject=inj))
    per = {s.smid: s.ctas for s in sms if s.ctas}
    assert set(per) == every_sm - H and r.sms_covered == n - K and r.complete == 0 and r.rounds == 4
    assert r.ctas == 4 * n == sum(per.values()) and max(per.values()) >= 2 and r.unpublished == 0
    assert r.bits_checked == 32 * 224 * 256 * 2 * r.iterations * r.ctas
    if where in ("none", "held"):
        assert r.status == cro.OK and r.verdict == NONE and not faults and r.failed_sms == 0
        assert r.fold == r.expect == regfile.fold(r.seed, 1)
        assert json.loads(cro.emit_regfile_annotations_json(r)) == regfile.annotations(test_regfile_abi.as_dict(r))
        report("regfile", K, H, r.rounds, r.sms_covered, max(per.values()), t, t_free)
    elif where == "every":
        assert r.status == cro.ERR_CHECKSUM and r.verdict == ALL and r.failed_sms == r.sms_covered == n - K
    else:
        assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and r.bad_sms == 1 and r.bad_sm[0] == smid
        assert sum(r.mismatches) == per[smid] and len(faults) == per[smid]
        e = regfile.word(r.seed, 0, 32 * 3 + 17, 100)
        assert all((f.element, f.iteration, f.smid, f.warp, f.lane, f.slot, f.expected, f.actual) == (0, 0, smid, 3, 17, 100, e, e ^ BIT)
                   for f in faults)


# ---- the SRAM probe: the local leg, and the network leg, whose clusters cannot use a held SM ---------------------------
@pytest.mark.parametrize("leg,cluster", [(0, 0), (1, 2), (1, 8)], ids=["local", "network-2", "network-8"])
@gpu
def test_sram_under_a_hold(cro, ctx, holder, coracle, n, every_sm, leg, cluster):
    import sram
    (r0, _, _), t_free = timed(lambda: ctx.probe_sram(0, legs=1 << leg, iterations=1, cluster=cluster))
    H, (r, sms, faults), t = held(holder, K, lambda: ctx.probe_sram(0, legs=1 << leg, iterations=1, cluster=cluster))
    L = r.leg[leg]
    per = {s.smid: s.leg[leg].ctas for s in sms if s.leg[leg].ctas}
    assert r.status == cro.OK and r.verdict == sram.NONE and not faults and r.bad_sms == 0 and r.bad_pairs == 0
    assert not set(per) & H and set(per) <= every_sm - H, sorted(set(per) & H)
    assert L.sms_covered == len(per) and L.complete == 0 and L.unpublished == 0 and L.rounds == 4
    assert L.ctas == sum(per.values()) and list(L.mismatches) == [0] * 6 and L.failed_sms == 0
    n_words = r.bytes_per_sm // 8
    if leg == 0:
        assert set(per) == every_sm - H and L.sms_covered == n - K and L.ctas == 4 * n and max(per.values()) >= 2
        assert L.fold == L.expect == sram.m5_fold(coracle.checksum, r.seed, n_words, 1)
        assert L.bytes == 80 * n_words * L.ctas
    else:
        assert L.cluster == cluster and L.ctas % cluster == 0 and L.sms_covered <= n - K
        assert L.bytes == 8 * n_words * (cluster + 2) * L.ctas
    assert json.loads(cro.emit_sram_annotations_json(r)) == sram.annotations(test_sram_abi.as_dict(r))
    report("sram %s" % ("local" if leg == 0 else "network %d" % cluster), K, H, L.rounds, L.sms_covered, max(per.values()), t,
           t_free)


# ---- one free SM: every CTA of every round runs there --------------------------------------------------------------
@pytest.mark.parametrize("inject", [False, True], ids=["clean", "inject"])
@pytest.mark.parametrize("name", ["compute", "alu"])
@gpu
def test_one_free_sm_runs_every_cta(cro, ctx, holder, n, every_sm, name, inject):
    """With one SM covered and failing, the rule of oracle/sm_legs.py and oracle/xlane.py (every covered SM failed)
    gives `all`, not `sm`: one SM cannot tell a bad SM from a common cause."""
    with holder.hold(n - 1) as H:
        (free,) = every_sm - H
        if name == "compute":
            inj = (0, free, 15, 77, 133, INT_MASK) if inject else None
            (r, sms, faults), t = timed(lambda: ctx.probe_compute(0, iterations=16, alu_iterations=1, legs=1, inject=inj))
        else:
            inj = (3, free, 3, 17, ALU_INJECT[3][0], 0, ALU_INJECT[3][1], ALU_INJECT[3][2]) if inject else None
            (r, sms, faults), t = timed(lambda: ctx.probe_alu(0, iterations=1, legs=1 << 3, inject=inj))
    if name == "compute":
        L = r.leg[0]
        covered, failed, ctas = L.sms_covered, L.failed_sms, L.ctas
        assert [(s.smid, s.leg[0].ctas) for s in sms] == [(free, 4 * n)] and L.rounds == 4 and L.complete == 0
    else:
        covered, failed, ctas = r.sms_covered, r.failed_sms, r.ctas
        assert [(s.smid, s.ctas) for s in sms] == [(free, 4 * n)] and r.rounds == 4 and r.complete == 0
        assert r.ops_checked[3] == cro.ALU_OPS[3] * 256 * 4 * n
    assert covered == 1 and ctas == 4 * n
    want = ALL if failed and failed == covered else SM if failed else NONE
    if inject:
        assert failed == 1 and want == ALL and r.verdict == want and r.status == cro.ERR_CHECKSUM
        assert list(r.bad_sm[:r.bad_sms]) == [free] and len(faults) == min(4 * n, 256)
    else:
        assert r.verdict == want == NONE and r.status == cro.OK and not faults
    print("%s one free SM %d: %d CTAs, verdict %d, %.1f ms" % (name, free, ctas, r.verdict, t * 1e3))


# ---- the L2 probe: no coverage rounds, but its readers' SMs are whatever SM a CTA landed on --------------------------
def l2_classify(r, sms, faults):
    import l2
    from test_l2_abi import as_dict
    return l2.classify(as_dict(r), [{"smid": s.smid, "mismatches": list(s.mismatches), "last": s.last,
                                     "words_read": list(s.words_read)} for s in sms],
                       [{"element": f.element, "iteration": f.iteration, "smid": f.smid, "word": f.word} for f in faults])


@pytest.mark.parametrize("size", ["min", "l2"])
@gpu
def test_l2_clean_under_a_hold(cro, ctx, holder, coracle, n, every_sm, size):
    import l2
    l2_bytes = ctx.probe_l2(0, bytes=cro.L2_MIN_BYTES, iterations=1)[0].l2_bytes
    nbytes = {"min": cro.L2_MIN_BYTES, "l2": l2_bytes // 16384 * 16384}[size]
    (_, _, _), t_free = timed(lambda: ctx.probe_l2(0, bytes=nbytes, iterations=1))
    H, (r, sms, faults), t = held(holder, K, lambda: ctx.probe_l2(0, bytes=nbytes, iterations=1))
    assert r.status == cro.OK and r.verdict == l2.NONE and not faults and r.unpublished == 0
    assert not {s.smid for s in sms} & H and sum(s.launches for s in sms) == 6 * n
    assert r.fold_ok == 1 and r.fold == r.expect == l2.m5_fold(coracle.checksum, r.seed, nbytes // 8, 1)
    for e in range(1, 6):
        assert sum(s.words_read[e] for s in sms) == nbytes // 8
    assert r.sms_covered <= n - K
    report("l2 %s" % size, K, H, 1, r.sms_covered, max(s.launches for s in sms), t, t_free)


@pytest.mark.parametrize("element", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("word", ["first", "middle", "last"])
@gpu
def test_l2_one_word_injection_names_its_reader_under_a_hold(cro, ctx, holder, every_sm, element, word):
    import l2
    W4 = 4 * MIB
    w = {"first": 0, "middle": W4 // 16 + 5, "last": W4 // 8 - 1}[word]
    with holder.hold(K) as H:
        r, sms, faults = ctx.probe_l2(0, bytes=W4, iterations=2, inject=(cro.L2_MARCH, -1, element, 1, w, 1 << 41))
    (f,) = faults
    G = r.ctas
    b = w // l2.BLOCK_WORDS
    assert (f.element, f.iteration, f.word, f.cta, f.writer_cta) == (element, 1, w, l2.owner(b, element, G), l2.owner(b, element - 1, G))
    assert f.smid in every_sm - H and f.writer_smid in every_sm - H
    want = l2_classify(r, sms, faults)
    assert (r.verdict, r.status, r.bad_sms, list(r.bad_sm)) == (want["verdict"], want["status"], want["bad_sms"], want["bad_sm"])
    assert r.verdict == l2.SM and list(r.bad_sm[:r.bad_sms]) == [f.smid] and f.line == want["line"][0] == 0


@gpu
def test_l2_a_word_every_reader_saw_wrong_under_a_hold(cro, ctx, holder, every_sm):
    """The five readers of a word are CTAs of five launches; under a hold two of them may share an SM.  The verdict
    and the records' line flags are what oracle/l2.py gives for the SMs the records name."""
    with holder.hold(K) as H:
        r, sms, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, inject=(cro.L2_MARCH, -1, -1, 0, 12345, 1 << 41))
    assert len(faults) == 5 and not {f.smid for f in faults} & H
    want = l2_classify(r, sms, faults)
    assert (r.verdict, r.bad_sms, r.bad_lines, list(r.bad_line)) == (want["verdict"], want["bad_sms"], want["bad_lines"], want["bad_line"])
    assert [f.line for f in faults] == want["line"]
    print("l2 line under a hold: readers on %d distinct SMs, verdict %d" % (len({f.smid for f in faults}), r.verdict))


# ---- the HBM path: no sweep kernel may need all its CTAs resident at once --------------------------------------------
@pytest.mark.parametrize("sweep", [64 * MIB, 64 * MIB + 12345 * 16], ids=["64MiB", "ragged"])
@gpu
def test_hbm_probe_under_a_hold(cro, holder, coracle, sweep):
    with cro.ProbeContext(sweep_bytes=sweep, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        c.probe_device(0)                                    # the region and the fill, outside the hold
        with holder.hold(K):
            p = c.probe_device(0)
            rep, words = c.locate_faults(0, retest=False)
        want = coracle.checksum(p.seed, 0, p.sweep_bytes // 8)
        assert p.sweep_bytes == sweep
        assert p.status == 0 and p.checksum == p.expect == want and p.copy_checksum == want
        assert p.copy_verified == p.copy_sweeps >= 1
        assert rep.status == 0 and rep.pass_[0].mismatches == 0 and not words


# ---- the health check: -incomplete lists exactly the SM checks that ran short -----------------------------------------
@gpu
def test_health_check_under_a_hold(cro, ctx, holder, n):
    import health
    opts = dict(compute=dict(iterations=2, alu_iterations=2), precision=dict(iterations=2, alu_iterations=2),
                sram=dict(iterations=1), l2=dict(bytes=4 * MIB, iterations=1), link=dict(bytes=64 * MIB),
                scan=dict(max_bytes=256 * MIB))
    (_, _), t_free = timed(lambda: ctx.check_health(0, **opts))
    H, (r, _), t = held(holder, K, lambda: ctx.check_health(0, **opts))
    assert r.status == cro.OK and r.failed == r.errored == r.not_run == 0
    cov = {0: min(L.sms_covered for i, L in enumerate(r.compute.leg) if r.compute.legs >> i & 1) < r.compute.sm_count,
           1: min(L.sms_covered for i, L in enumerate(r.precision.leg) if r.precision.legs >> i & 1) < r.precision.sm_count,
           2: min(L.sms_covered for i, L in enumerate(r.sram.leg) if r.sram.legs >> i & 1) < r.sram.sm_count,
           3: r.l2.sms_covered < r.l2.sm_count}
    short = sum(1 << c for c, s in cov.items() if s)
    assert r.incomplete == short and short & cro.HEALTH_COMPUTE          # compute runs first, inside the hold
    assert min(L.sms_covered for i, L in enumerate(r.compute.leg) if r.compute.legs >> i & 1) == n - K
    ann = json.loads(cro.emit_health_annotations_json(r))
    assert ann == health.annotations(test_health_abi.as_dict(r, cro))
    assert ann["cohdi.io/probe-health-incomplete"] == health.names(short)
    print("health under a hold: k %d, H %s, incomplete %s, held %.1f ms, unheld %.1f ms"
          % (K, sorted(H), health.names(short), t * 1e3, t_free * 1e3))
