"""Every probe option at the largest value include/croprobe.h accepts, run on one H100 against the restatements in
oracle/ and the C oracle.

The refusal tests check that max + 1 is refused; these check that the maximum itself works: iterations at their
limits (fold products that wrap mod 2^64, %clock64 sums past 2^32), the L2 probe's counter counts and buffer size at
both ends, 64 coverage rounds under a hold of part of the GPU, the whole-HBM scan's 128-chunk cap and the host link at
L = S and 2^24 hops.  Every row compares with a restatement exactly.

Faults come only from the probes' software injection and the scan's test force; nothing here repeats a call to catch a
real one.  The CPU guard at the end parses the header's option maxima and fails when one has no row here."""
import json
import os
import re
import time

import numpy as np
import pytest

import test_compute_abi
from test_compute_probe import FLOAT_MASK, INT_MASK
from test_compute_probe import injected as compute_injected
from test_compute_probe import is_float
from test_compute_probe import tiles as compute_tiles
from test_held_sms import HOLD_NS, Holder, holder_cmd, lane_dict
from test_held_sms import _lane_probes, _sm_legs_probes, check_lane_coverage, check_sm_legs_coverage
from test_precision_probe import EXP_MASK as PRECISION_MASK
from test_precision_probe import answers as precision_answers
from test_precision_probe import canon, expect_bits
from test_sparse_probe import EXP_MASK as SPARSE_MASK
from test_sparse_probe import answers as sparse_answers
from test_sram_probe import expected_word as sram_expected_word
from test_warpmma_probe import EXP_MASK as WARPMMA_MASK
from test_warpmma_probe import answers as warpmma_answers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "croprobe.h")
U64 = (1 << 64) - 1
MIB = 1 << 20
K = 8                              # SMs held in the 64-round rows
NONE, SM, ALL = 0, 1, 2
MIN_GHZ = 0.5                      # cycles / ns of an SM's CTAs: a %clock64 sum cut to 32 bits falls far below this
gpu = pytest.mark.gpu


def middle(it):
    """A middle iteration, past 4096 at 65536 (40000), proportionally below."""
    return it * 40000 // 65536


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=64 * MIB, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@pytest.fixture(scope="module")
def n(ctx):
    return ctx.own_devices()[0].sm_count


@pytest.fixture(scope="module")
def every_sm(ctx, n):
    _, sms, _ = ctx.probe_compute(0, iterations=1, alu_iterations=1, legs=1)
    got = {s.smid for s in sms}
    assert len(got) == n
    return got


@pytest.fixture(scope="module")
def holder(tmp_path_factory, _built):
    import subprocess
    out = str(tmp_path_factory.mktemp("holder") / "sm_holder.so")
    subprocess.check_call(holder_cmd(out))
    h = Holder(out)
    try:
        yield h
    finally:
        h.lib.holder_release()


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


# ---- 1. iterations at their maximum: the four tensor probes (oracle/sm_legs.py) --------------------------------------
def _tensor_probes(cro):
    import compute
    import precision
    import sparse
    import warpmma
    co = compute.CComputeOracle()
    return {
        "compute": dict(call=ctx_call("probe_compute"), legs=cro.COMPUTE_LEGS, mod=compute, emit=cro.emit_compute_annotations_json,
                        kw=dict(iterations=cro.COMPUTE_MAX_ITERATIONS, alu_iterations=cro.COMPUTE_MAX_ALU_ITERATIONS),
                        alu_legs=(cro.COMPUTE_LEG_FFMA, cro.COMPUTE_LEG_IMAD), rc=(77, 133),
                        tile=lambda seed, leg: compute_tiles(co, seed)[compute.LEG_ANSWER[leg]],
                        fold1=lambda leg, tile: compute.cta_fold(tile, 1), ops=lambda leg: 2 * compute.M * compute.N * compute.K,
                        mask=lambda leg: FLOAT_MASK if is_float(cro, leg) else INT_MASK,
                        record=lambda leg, f, v, mask: (f.expected, f.actual) == (v, compute_injected(cro, leg, v, mask))),
        "precision": dict(call=ctx_call("probe_precision"), legs=cro.PRECISION_LEGS, mod=precision,
                          emit=cro.emit_precision_annotations_json,
                          kw=dict(iterations=cro.PRECISION_MAX_ITERATIONS, alu_iterations=cro.PRECISION_MAX_ALU_ITERATIONS),
                          alu_legs=(cro.PRECISION_LEG_DFMA, cro.PRECISION_LEG_HFMA2), rc=(77, 45),
                          tile=lambda seed, leg: precision_answers(seed)[precision.LEG_ANSWER[leg]],
                          fold1=lambda leg, tile: precision.cta_fold(leg, tile, 1),
                          ops=lambda leg: 2 * int(np.prod(precision.SHAPE[precision.LEG_ANSWER[leg]], dtype=object)),
                          mask=lambda leg: PRECISION_MASK[leg],
                          record=lambda leg, f, v, mask: f.expected == v and canon(leg, f.actual_bits ^ mask) == expect_bits(leg, v)
                          and f.actual_bits >> precision.LEG_BITS[leg] == 0),
        "sparse": dict(call=ctx_call("probe_sparse"), legs=cro.SPARSE_LEGS, mod=sparse, emit=cro.emit_sparse_annotations_json,
                       kw=dict(iterations=cro.SPARSE_MAX_ITERATIONS), alu_legs=(), rc=(77, 45),
                       tile=lambda seed, leg: sparse_answers(seed)[sparse.LEG_ANSWER[leg]],
                       fold1=lambda leg, tile: sparse.cta_fold(leg, tile, 1),
                       ops=lambda leg: 2 * sparse.M * sparse.N * sparse.K[sparse.LEG_ANSWER[leg]], mask=lambda leg: SPARSE_MASK,
                       record=lambda leg, f, v, mask: (f.expected, f.actual_bits) == (v, sparse.value_bits(leg, v) ^ mask)),
        "warpmma": dict(call=ctx_call("probe_warpmma"), legs=cro.WARPMMA_LEGS, mod=warpmma, emit=cro.emit_warpmma_annotations_json,
                        kw=dict(iterations=cro.WARPMMA_MAX_ITERATIONS), alu_legs=(), rc=(77, 45),
                        tile=lambda seed, leg: warpmma_answers(seed)[warpmma.LEG_ANSWER[leg]],
                        fold1=lambda leg, tile: warpmma.cta_fold(leg, tile, 1), ops=lambda leg: warpmma.ops(leg),
                        mask=lambda leg: WARPMMA_MASK[leg],
                        record=lambda leg, f, v, mask: (f.expected, f.actual_bits) == (v, warpmma.value_bits(leg, v) ^ mask)),
    }


def ctx_call(method):
    return lambda ctx, **kw: getattr(ctx, method)(0, **kw)


def leg_iterations(P, leg):
    return P["kw"]["alu_iterations"] if leg in P["alu_legs"] else P["kw"]["iterations"]


TENSOR = ["compute", "precision", "sparse", "warpmma"]
TENSOR_LEGS = [(name, leg) for name, legs in (("compute", 5), ("precision", 7), ("sparse", 6), ("warpmma", 6))
               for leg in range(legs)]


@pytest.mark.parametrize("name", TENSOR)
@gpu
def test_tensor_probe_clean_at_its_iteration_maxima(cro, ctx, n, name):
    import sm_legs
    P = _tensor_probes(cro)[name]
    (r, sms, faults), t = timed(lambda: P["call"](ctx, **P["kw"]))
    assert r.status == cro.OK and r.verdict == NONE and not faults and r.bad_sms == 0 and r.sm_count == n
    assert [s.smid for s in sms] == sorted({s.smid for s in sms}) and len(sms) == n
    for leg in range(P["legs"]):
        L, it = r.leg[leg], leg_iterations(P, leg)
        assert L.iterations == it and L.rounds == 1 and L.ctas == n, leg
        assert L.sms_covered == n and L.complete == 1 and L.unpublished == 0, (leg, L.sms_covered, L.unpublished)
        assert L.mismatches == L.fold_mismatches == L.recorded == L.failed_sms == 0, leg
        once = P["fold1"](leg, P["tile"](r.seed, leg))
        assert L.fold == L.expect_fold == (it * once) & U64, (leg, hex(L.fold), hex(L.expect_fold), hex((it * once) & U64))
        assert L.ops == P["ops"](leg) * it * n, leg
        per_iter = {s.smid: s.leg[leg].cycles // (s.leg[leg].ctas * it) for s in sms}
        assert all(s.leg[leg].ctas == 1 and s.leg[leg].mark == 0 for s in sms), leg
        assert all(v > 0 for v in per_iter.values()), (leg, [s for s, v in per_iter.items() if not v])
        assert (L.slowest_sm, L.slow_permille) == sm_legs.slowest(per_iter), leg
    assert json.loads(P["emit"](r)) == P["mod"].annotations(test_compute_abi.as_dict(r))
    print("%s at %s: %.2f s, per leg %s ms" % (name, P["kw"], t, [round(r.leg[g].ns / 1e6, 1) for g in range(P["legs"])]))


@pytest.mark.parametrize("when", ["last", "middle"])
@pytest.mark.parametrize("name,leg", TENSOR_LEGS)
@gpu
def test_tensor_probe_injection_at_its_iteration_maxima(cro, ctx, every_sm, name, leg, when):
    P = _tensor_probes(cro)[name]
    it = leg_iterations(P, leg)
    iteration = it - 1 if when == "last" else middle(it)
    smid, (row, col), mask = min(every_sm), P["rc"], P["mask"](leg)
    r, sms, faults = P["call"](ctx, legs=1 << leg, inject=(leg, smid, iteration, row, col, mask), cap=4096, **P["kw"])
    assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and r.bad_sms == 1 and r.bad_sm[0] == smid
    (entry,) = [s for s in sms if s.smid == smid]
    ctas = entry.leg[leg].ctas
    L = r.leg[leg]
    assert ctas == 1 and L.iterations == it and L.sms_covered == len(every_sm) and L.unpublished == 0
    assert L.failed_sms == 1 and L.fold_mismatches == entry.leg[leg].fold_mismatches == ctas
    assert all(s.leg[leg].mark == 0 and s.leg[leg].mismatches == s.leg[leg].fold_mismatches == 0 for s in sms if s.smid != smid)
    if when == "last":
        v = int(P["tile"](r.seed, leg)[row, col])
        assert L.mismatches == L.recorded == ctas and entry.leg[leg].mark == cro.COMPUTE_PERSISTENT
        assert [(f.leg, f.smid, f.row, f.col) for f in faults] == [(leg, smid, row, col)] * ctas
        assert all(P["record"](leg, f, v, mask) for f in faults)
    else:
        assert L.mismatches == L.recorded == 0 and not faults and entry.leg[leg].mark == cro.COMPUTE_INTERMITTENT
    assert L.fold != L.expect_fold == (it * P["fold1"](leg, P["tile"](r.seed, leg))) & U64
    ann = json.loads(P["emit"](r))
    assert ann == P["mod"].annotations(test_compute_abi.as_dict(r)) and ann["cohdi.io/probe-%s-bad-sms" % name] == str(smid)


# ---- 1. iterations at their maximum: ALU and barrier, one leg per call ------------------------------------------------
def check_clock(sms):
    """Each SM's %clock64 sum over its %globaltimer window is a plausible SM clock: a sum cut to 32 bits is not."""
    for s in sms:
        assert s.cycles > 0 and s.cycles >= MIN_GHZ * s.ns, (s.smid, s.cycles, s.ns)


def check_lane_clean(cro, r, sms, faults, n, leg, it, ops, fold):
    assert r.status == cro.OK and r.verdict == NONE and not faults and r.bad_sms == 0 and r.failed_legs == 0
    assert r.iterations == it and r.legs == 1 << leg and r.recorded == 0
    assert r.mismatches[leg] == r.fold_mismatches[leg] == 0
    assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == fold, leg
    assert r.unpublished == 0 and r.threads_unpublished == 0
    assert r.ops_checked[leg] == ops * 256 * it * r.ctas
    assert [s.smid for s in sms] == sorted({s.smid for s in sms})
    assert all(s.mark == 0 and s.fold_mismatches == 0 and s.ctas >= 1 for s in sms)
    check_clock(sms)


@pytest.mark.parametrize("leg", range(5), ids=["logic", "shift", "iadd", "imul", "float"])
@gpu
def test_alu_clean_at_its_iteration_maximum(cro, ctx, n, leg):
    import alu
    it = cro.ALU_MAX_ITERATIONS
    r, sms, faults = ctx.probe_alu(0, iterations=it, legs=1 << leg)
    check_lane_clean(cro, r, sms, faults, n, leg, it, cro.ALU_OPS[leg], alu.fold(leg, r.seed))
    assert r.sms_covered == n and r.complete == 1 and r.rounds == 1 and r.ctas == n and len(sms) == n
    assert json.loads(cro.emit_alu_annotations_json(r)) == alu.annotations(lane_dict(r))
    print("alu leg %d at %d iterations: %.2f s of launches, %.2f s the call, max SM cycles %d"
          % (leg, it, r.ns / 1e9, r.wall_ns / 1e9, max(s.cycles for s in sms)))


@pytest.mark.parametrize("when", ["last", "middle"])
@gpu
def test_alu_injection_at_its_iteration_maximum(cro, ctx, every_sm, when):
    import alu
    from test_alu_probe import INJECT
    leg, warp, lane, it = cro.ALU_LEG_SHIFT, 7, 31, cro.ALU_MAX_ITERATIONS
    iteration = it - 1 if when == "last" else middle(it)
    smid = min(every_sm)
    op, operand, mask = INJECT[leg]
    r, sms, faults = ctx.probe_alu(0, iterations=it, legs=1 << leg, inject=(leg, smid, warp, lane, op, iteration, operand, mask),
                                   cap=cro.ALU_RECORDS)
    want = alu.injected(leg, r.seed, op, warp, lane, operand, mask)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid] and r.failed_legs == 1 << leg
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid and entry.failed_legs == 1 << leg and entry.ctas == 1
    assert entry.mark == (cro.ALU_PERSISTENT if when == "last" else cro.ALU_INTERMITTENT)
    assert r.mismatches[leg] == entry.ctas and r.fold_mismatches[leg] == (entry.ctas if when == "last" else 0)
    assert [(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, list(f.in_), tuple(f.expected), tuple(f.actual)) for f in faults] == \
        [(leg, op, iteration, smid, warp, lane) + tuple(want)] * entry.ctas


BARRIER_LEGS = [0, 1, 2]


@pytest.mark.parametrize("leg", BARRIER_LEGS, ids=["bar", "mbar", "cluster"])
@gpu
def test_barrier_clean_at_its_iteration_maximum(cro, ctx, n, leg):
    import barrier
    it = cro.BARRIER_MAX_ITERATIONS
    r, sms, faults = ctx.probe_barrier(0, iterations=it, legs=1 << leg)
    assert r.timeouts == 0 and r.bad_pairs == 0 and r.cluster == 2
    if leg == cro.BARRIER_LEG_CLUSTER:     # every CTA of a cluster checks every row: ops over the CTAs that ran
        assert r.cluster_sms == r.sms_covered == len(sms) > 0 and r.ctas % 2 == 0
    else:
        assert r.sms_covered == n and r.complete == 1 and r.rounds == 1 and r.ctas == n and len(sms) == n
    check_lane_clean(cro, r, sms, faults, n, leg, it, cro.BARRIER_OPS[leg], barrier.fold(leg, r.seed, 2))
    assert json.loads(cro.emit_barrier_annotations_json(r)) == barrier.annotations(barrier_dict(r))
    print("barrier leg %d at %d iterations: %.2f s of launches, %.2f s the call" % (leg, it, r.ns / 1e9, r.wall_ns / 1e9))


def barrier_dict(r):
    d = lane_dict(r)
    d["bad_pairs"] = r.bad_pairs
    d["bad_pair"] = [(p.smid, p.peer_smid) for p in r.bad_pair[:r.bad_pairs]]
    return d


@pytest.mark.parametrize("when", ["last", "middle"])
@gpu
def test_barrier_injection_at_its_iteration_maximum(cro, ctx, every_sm, when):
    import barrier
    from test_barrier_probe import INJECT, MASK
    leg, warp, lane, it = cro.BARRIER_LEG_MBAR, 7, 31, cro.BARRIER_MAX_ITERATIONS
    iteration = it - 1 if when == "last" else middle(it)
    smid, op = min(every_sm), INJECT[leg]
    r, sms, faults = ctx.probe_barrier(0, iterations=it, legs=1 << leg, inject=(leg, smid, warp, lane, op, iteration, MASK),
                                       cap=cro.BARRIER_RECORDS)
    want = barrier.injected(leg, r.seed, op, warp, lane, MASK)
    kept = min(len(want), cro.BARRIER_THREAD_RECORDS)
    assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid] and r.timeouts == 0
    (entry,) = [s for s in sms if s.mark]
    assert entry.smid == smid and entry.failed_legs == 1 << leg and entry.ctas == 1
    assert entry.mark == (cro.BARRIER_PERSISTENT if when == "last" else cro.BARRIER_INTERMITTENT)
    assert r.mismatches[leg] == len(want) * entry.ctas and r.fold_mismatches[leg] == (entry.ctas if when == "last" else 0)
    assert [(f.leg, f.op, f.iteration, f.smid, f.warp, f.lane, f.kind, f.bar, f.phase, f.slot, f.expected, f.actual)
            for f in faults] == [(leg, op, iteration, smid, warp, lane) + w for w in want[:kept]] * entry.ctas


# ---- 1. and 2. the L2 probe: iterations, counter counts and W at both ends --------------------------------------------
BIT = 1 << 41


def check_l2_clean(cro, coracle, r, sms, faults, nbytes, iterations):
    import l2
    G = r.ctas
    assert r.status == cro.OK and r.verdict == cro.L2_NONE and not faults, (r.status, r.verdict, r.a1_bad, r.a2_bad, r.a2_holes)
    assert r.bytes == nbytes and r.iterations == iterations and r.blocks == nbytes // cro.L2_BLOCK_BYTES and r.unpublished == 0
    assert list(r.mismatches) == [0] * 6 and sum(s.launches for s in sms) == 6 * iterations * G
    assert r.fold_ok == 1 and r.fold == r.expect == l2.m5_fold(coracle.checksum, r.seed, nbytes // 8, iterations)
    for e in range(1, 6):
        assert sum(s.words_read[e] for s in sms) == iterations * nbytes // 8, e
    assert r.a1_bad == r.a2_bad == r.a2_holes == 0 and r.a2_tickets == 32 * G


@gpu
def test_l2_at_its_iteration_maximum(cro, ctx, coracle):
    import l2
    it = cro.L2_MAX_ITERATIONS
    r, sms, faults = ctx.probe_l2(0, iterations=it)
    check_l2_clean(cro, coracle, r, sms, faults, r.bytes, it)
    w = 4 * MIB // 8 - 1
    r, sms, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=it, inject=(cro.L2_MARCH, -1, 3, it - 1, w, BIT))
    (f,) = faults
    b = w // l2.BLOCK_WORDS
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and list(r.bad_sm[:r.bad_sms]) == [f.smid]
    assert (f.element, f.iteration, f.word, f.cta, f.writer_cta) == (3, it - 1, w, l2.owner(b, 3, r.ctas), l2.owner(b, 2, r.ctas))
    assert f.expected == l2.expected_read(r.seed, 3, w) and f.actual == f.expected ^ BIT
    assert list(r.mismatches) == [0, 0, 0, 1, 0, 0] and r.fold_ok == 1


A1_COUNTS = [1, 7, 65537, 1 << 20]
A2_COUNTS = [1, 33, 8192]


@pytest.mark.parametrize("count", A1_COUNTS)
@gpu
def test_l2_a1_counter_counts(cro, ctx, coracle, count):
    r, sms, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, a1_counters=count)
    assert r.a1_counters == count
    check_l2_clean(cro, coracle, r, sms, faults, 4 * MIB, 1)
    for counter in sorted({0, count - 1}):
        r, _, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, a1_counters=count, inject=(cro.L2_A1, -1, 0, 0, counter, BIT))
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ATOMIC and not faults, counter
        assert (r.a1_bad, r.a1_bad_counter[0], r.a2_bad, r.a2_holes) == (1, counter, 0, 0), counter


@pytest.mark.parametrize("count", A2_COUNTS)
@gpu
def test_l2_a2_counter_counts(cro, ctx, coracle, count):
    r, sms, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, a2_counters=count)
    assert r.a2_counters == count
    check_l2_clean(cro, coracle, r, sms, faults, 4 * MIB, 1)
    for counter in sorted({0, count - 1}):
        r, _, faults = ctx.probe_l2(0, bytes=4 * MIB, iterations=1, a2_counters=count, inject=(cro.L2_A2, -1, 0, 0, counter, 1))
        assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_ATOMIC and not faults, counter
        assert (r.a2_bad, r.a2_bad_counter[0], r.a2_holes, r.a1_bad) == (1, counter, 1, 0), counter


@pytest.mark.parametrize("size", ["top", "l2+block"])
@gpu
def test_l2_buffer_size_ends(cro, ctx, coracle, size):
    import l2
    l2_bytes = ctx.probe_l2(0, bytes=cro.L2_MIN_BYTES, iterations=1)[0].l2_bytes
    nbytes = {"top": cro.L2_MAX_L2_MULTIPLE * l2_bytes // cro.L2_BLOCK_BYTES * cro.L2_BLOCK_BYTES,
              "l2+block": l2_bytes // cro.L2_BLOCK_BYTES * cro.L2_BLOCK_BYTES + cro.L2_BLOCK_BYTES}[size]
    r, sms, faults = ctx.probe_l2(0, bytes=nbytes, iterations=1)
    check_l2_clean(cro, coracle, r, sms, faults, nbytes, 1)
    w = nbytes // 8 - 1
    r, sms, faults = ctx.probe_l2(0, bytes=nbytes, iterations=1, inject=(cro.L2_MARCH, -1, 5, 0, w, BIT))
    (f,) = faults
    b = w // l2.BLOCK_WORDS
    assert r.status == cro.ERR_CHECKSUM and r.verdict == cro.L2_SM and list(r.bad_sm[:r.bad_sms]) == [f.smid]
    assert (f.element, f.iteration, f.word, f.cta, f.writer_cta) == (5, 0, w, l2.owner(b, 5, r.ctas), l2.owner(b, 4, r.ctas))
    assert f.expected == l2.expected_read(r.seed, 5, w) and f.actual == f.expected ^ BIT
    print("l2 W %d B (%s, L2 %d B): march %.1f GB/s" % (nbytes, size, l2_bytes, r.march_bytes / max(r.march_ns, 1)))


# ---- 3. max_rounds at 64 under a hold: every probe with coverage rounds -----------------------------------------------
ROUNDS_MAX = {"compute": "COMPUTE_MAX_ROUNDS", "precision": "PRECISION_MAX_ROUNDS", "sparse": "SPARSE_MAX_ROUNDS",
              "warpmma": "WARPMMA_MAX_ROUNDS", "sram": "SRAM_MAX_ROUNDS", "regfile": "REGFILE_MAX_ROUNDS",
              "xlane": "XLANE_MAX_ROUNDS", "alu": "ALU_MAX_ROUNDS", "barrier-bar": "BARRIER_MAX_ROUNDS",
              "barrier-mbar": "BARRIER_MAX_ROUNDS"}


def held_call(cro, ctx, name, smid, rounds):
    """One call at 1 iteration and max_rounds = rounds, with an injection into SM smid (None: none)."""
    if name in TENSOR:
        P = _sm_legs_probes(cro)[name]
        inj = None if smid is None else (0, smid, 0) + P["rc"] + (P["mask"],)
        return P["call"](ctx, iterations=1, legs=1, max_rounds=rounds, inject=inj, cap=4096)
    if name in ("xlane", "alu"):
        P = _lane_probes(cro)[name]
        return P["call"](ctx, iterations=1, legs=1 << 2, max_rounds=rounds, inject=None if smid is None else P["inject"](2, smid, 0),
                         cap=4096)
    if name == "sram":
        inj = None if smid is None else (cro.SRAM_SMEM, smid, 3, 0, 7, BIT)
        return ctx.probe_sram(0, legs=cro.SRAM_LEG_SMEM, iterations=1, max_rounds=rounds, inject=inj, cap=4096)
    if name == "regfile":
        return ctx.probe_regfile(0, iterations=1, max_rounds=rounds, inject=None if smid is None else (smid, 3, 17, 100, 0, 0, 1 << 19),
                                 cap=4096)
    from test_barrier_probe import INJECT, MASK
    leg = {"barrier-bar": 0, "barrier-mbar": 1}[name]
    return ctx.probe_barrier(0, iterations=1, legs=1 << leg, max_rounds=rounds,
                             inject=None if smid is None else (leg, smid, 3, 17, INJECT[leg], 0, MASK), cap=cro.BARRIER_RECORDS)


@pytest.mark.parametrize("where", ["clean", "free", "held"])
@pytest.mark.parametrize("name", list(ROUNDS_MAX))
@gpu
def test_64_rounds_under_a_hold(cro, ctx, holder, coracle, n, every_sm, name, where):
    rounds = getattr(cro, ROUNDS_MAX[name])
    # the first launch of a kernel loads its module, which waits for the device: load them before the hold
    held_call(cro, ctx, name, None, 1)
    with holder.hold(K) as H:
        smid = {"clean": None, "free": max(every_sm - H), "held": min(H)}[where]
        (r, sms, faults), t = timed(lambda: held_call(cro, ctx, name, smid, rounds))
    # The call returns only once the hold ends: freeing its per-call buffers waits for this process's work on the
    # device, the holding kernel included, so wall_ns is the hold's length.  That every round ran inside the hold shows
    # in the rounds' own device time, and in a coverage that never reaches a held SM.
    T = r.leg[0] if hasattr(r, "leg") else r
    assert 0 < T.timer_ns < HOLD_NS // 4 and 0 < T.ns < HOLD_NS // 4, (T.timer_ns, T.ns)
    free, clean = every_sm - H, where != "free"
    if name in TENSOR:
        P = _sm_legs_probes(cro)[name]
        per = check_sm_legs_coverage(P, r, sms, H, every_sm, n, K, 0, rounds)
        L = r.leg[0]
        assert L.fold_mismatches == (0 if clean else per[smid])
        if clean:
            assert r.status == cro.OK and r.verdict == NONE and not faults and L.mismatches == L.failed_sms == 0
            assert L.fold == L.expect_fold == P["fold"](r.seed, 0, 1)
        else:
            assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid]
            assert L.failed_sms == 1 and L.mismatches == L.recorded == per[smid]
            assert [(f.leg, f.smid, f.row, f.col) for f in faults] == [(0, smid) + P["rc"]] * per[smid]
        assert json.loads(P["emit"](r)) == P["mod"].annotations(test_compute_abi.as_dict(r))
    elif name in ("xlane", "alu"):
        P = _lane_probes(cro)[name]
        per = check_lane_coverage(P, r, sms, H, every_sm, n, K, 1 << 2, rounds)
        if clean:
            assert r.status == cro.OK and r.verdict == NONE and not faults and r.failed_sms == 0 and r.mismatches[2] == 0
            assert tuple(r.fold[2]) == tuple(r.expect[2]) == P["fold"](r.seed, 2, 1)
        else:
            w = P["want"](r, 2, 0)
            lanes = set(w) if isinstance(w, dict) else {(3, 17)}
            assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid]
            assert r.failed_legs == 1 << 2 and r.fold_mismatches[2] == per[smid] and r.mismatches[2] == per[smid] * len(lanes)
            assert all((f.leg, f.smid, f.iteration) == (2, smid, 0) for f in faults)
            got = {}
            for f in faults:
                got[(f.warp, f.lane)] = got.get((f.warp, f.lane), 0) + 1
            assert got == {wl: per[smid] for wl in lanes}
        assert json.loads(P["emit"](r)) == P["mod"].annotations(lane_dict(r))
    elif name == "sram":
        import sram
        import test_sram_abi
        L = r.leg[0]
        per = {s.smid: s.leg[0].ctas for s in sms if s.leg[0].ctas}
        assert set(per) == free and L.sms_covered == n - K and L.complete == 0 and L.rounds == rounds
        assert L.ctas == rounds * n == sum(per.values()) and L.unpublished == 0
        assert L.fold == L.expect == sram.m5_fold(coracle.checksum, r.seed, r.bytes_per_sm // 8, 1)
        if clean:
            assert r.status == cro.OK and r.verdict == sram.NONE and not faults and list(L.mismatches) == [0] * 6
        else:
            e = sram_expected_word(r.seed, 3, 7)
            assert r.status == cro.ERR_CHECKSUM and r.verdict == sram.SM and list(r.bad_sm[:r.bad_sms]) == [smid]
            assert list(L.mismatches) == [per[smid] if x == 3 else 0 for x in range(6)] and L.recorded == per[smid]
            assert [(f.element, f.iteration, f.smid, f.word, f.expected, f.actual) for f in faults] == [(3, 0, smid, 7, e, e ^ BIT)] * per[smid]
        assert json.loads(cro.emit_sram_annotations_json(r)) == sram.annotations(test_sram_abi.as_dict(r))
    elif name == "regfile":
        import regfile
        import test_regfile_abi
        per = {s.smid: s.ctas for s in sms if s.ctas}
        assert set(per) == free and r.sms_covered == n - K and r.complete == 0 and r.rounds == rounds
        assert r.ctas == rounds * n == sum(per.values()) and r.unpublished == 0
        assert r.bits_checked == 32 * 224 * 256 * 2 * r.iterations * r.ctas
        if clean:
            assert r.status == cro.OK and r.verdict == NONE and not faults and r.fold == r.expect == regfile.fold(r.seed, 1)
        else:
            e = regfile.word(r.seed, 0, 32 * 3 + 17, 100)
            assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid]
            assert sum(r.mismatches) == per[smid] and [(f.element, f.iteration, f.smid, f.warp, f.lane, f.slot, f.expected, f.actual)
                                                       for f in faults] == [(0, 0, smid, 3, 17, 100, e, e ^ (1 << 19))] * per[smid]
        assert json.loads(cro.emit_regfile_annotations_json(r)) == regfile.annotations(test_regfile_abi.as_dict(r))
    else:
        import barrier
        from test_barrier_probe import INJECT, MASK
        leg = {"barrier-bar": 0, "barrier-mbar": 1}[name]
        per = {s.smid: s.ctas for s in sms if s.ctas}
        assert set(per) == free and r.sms_covered == n - K and r.complete == 0 and r.rounds == rounds
        assert r.ctas == rounds * n == sum(per.values()) and r.unpublished == 0 and r.threads_unpublished == 0 and r.timeouts == 0
        assert r.ops_checked[leg] == cro.BARRIER_OPS[leg] * 256 * rounds * n
        if clean:
            assert r.status == cro.OK and r.verdict == NONE and not faults and r.failed_sms == 0
            assert tuple(r.fold[leg]) == tuple(r.expect[leg]) == barrier.fold(leg, r.seed)
        else:
            want = barrier.injected(leg, r.seed, INJECT[leg], 3, 17, MASK)
            kept = min(len(want), cro.BARRIER_THREAD_RECORDS)
            assert r.status == cro.ERR_CHECKSUM and r.verdict == SM and list(r.bad_sm[:r.bad_sms]) == [smid]
            assert r.mismatches[leg] == len(want) * per[smid] and r.fold_mismatches[leg] == per[smid]
            assert [(f.smid, f.iteration, f.warp, f.lane, f.kind, f.bar, f.phase, f.slot, f.expected, f.actual) for f in faults] == \
                [(smid, 0, 3, 17) + w for _ in range(per[smid]) for w in want[:kept]]
        assert json.loads(cro.emit_barrier_annotations_json(r)) == barrier.annotations(barrier_dict(r))
    print("%s %s: %d rounds under a hold of %d SMs: %.1f ms of launches, %.1f ms the call, max CTAs on one SM %d"
          % (name, where, rounds, K, T.ns / 1e6, t * 1e3, max(per.values())))


# ---- 4. the scan's chunk cap ------------------------------------------------------------------------------------------
CHUNK_W = MIB + 16                 # test chunk: ragged against every power of two, so chunk k starts at an odd offset


def scan_capped(cro, ctx, **kw):
    return ctx.scan_hbm(0, max_bytes=(cro.SCAN_MAX_CHUNKS + 2) * CHUNK_W, chunk_bytes=CHUNK_W, seed=0x5CA9, cap=8192, **kw)


def complement(cf, nw):
    x, s, w = cf
    return (x ^ (U64 if nw & 1 else 0), (-nw - s) & U64, (-nw * nw - w) & U64)


@gpu
def test_scan_stops_at_its_chunk_cap(cro, ctx, coracle):
    import scan
    from test_hbm_scan import health
    rep, words = scan_capped(cro, ctx)
    C, cw = cro.SCAN_MAX_CHUNKS, CHUNK_W // 8
    # a scan the chunk cap stopped short of max_bytes covers the chunks it has and is otherwise an ordinary scan
    assert rep.status == cro.OK and rep.cuda_error == 0 and rep.complete == 1 and rep.elements_done == 4 and not words
    assert rep.n_chunks == C and rep.covered_bytes == C * CHUNK_W < (C + 2) * CHUNK_W
    for k in range(C):
        K_ = rep.chunk[k]
        assert (K_.word0, K_.bytes) == (k * cw, CHUNK_W), k
        want = coracle.checksum((rep.seed + K_.word0) & U64, 0, cw)
        assert K_.expect == want and K_.fold(0) == want and K_.fold(1) == complement(want, cw), k
    for p in range(2):
        assert rep.pass_[p].words_scanned == C * cw and rep.pass_[p].mismatches == rep.pass_[p].granules == 0
    assert rep.health == scan.health_bits(health(rep.before), health(rep.after))


@pytest.mark.parametrize("where", ["126|127", "last-word"])
@gpu
def test_scan_force_in_the_last_chunks(cro, ctx, scan_oracle, where):
    """A stuck-at-0 bit, so each word fails in exactly one pass: every count, flip, granule and record is the
    restatement's, each record in the chunk its index says, and nothing lies past the covered bytes."""
    C, cw = cro.SCAN_MAX_CHUNKS, CHUNK_W // 8
    first, count = {"126|127": ((C - 1) * cw - 300, 600), "last-word": (C * cw - 1, 1)}[where]
    stuck = ~(1 << 5) & U64
    rep, words = scan_capped(cro, ctx, force=(first, count, stuck, 0))
    want = scan_oracle.forced_mismatches(0x5CA9, first, count, stuck, 0)
    assert rep.status == cro.ERR_CHECKSUM and rep.n_chunks == C and rep.covered_bytes == C * CHUNK_W and rep.complete == 1
    for p in range(2):
        P = rep.pass_[p]
        assert P.mismatches == P.recorded == want[p]["mismatches"] and P.granules == want[p]["granules"], p
        assert list(P.bit_flips) == want[p]["bit_flips"], p
    assert rep.pass_[0].mismatches + rep.pass_[1].mismatches == count and rep.flip_or == 1 << 5
    expect = sorted([(w["word"], w["expected"], w["actual"], 1 << p) for p in range(2) for w in want[p]["words"]])
    assert [(w.word_index, w.expected, w.actual, w.passes) for w in words] == expect
    assert rep.located == len(words) == count and all(w.word_index < C * cw for w in words)
    for w in words:
        assert w.reserved == w.word_index // cw and rep.place(w) == (w.word_index // cw, w.word_index % cw), w.word_index


@gpu
def test_scan_refuses_a_force_past_its_covered_words(cro, ctx):
    C, cw = cro.SCAN_MAX_CHUNKS, CHUNK_W // 8
    with pytest.raises(cro.ProbeError) as e:
        scan_capped(cro, ctx, force=(C * cw - 1, 2, 0, 0))
    assert e.value.code == cro.ERR_INVALID_ARG


@pytest.fixture(scope="module")
def scan_oracle(_built):
    import scan
    return scan


# ---- 5. the host link at L = S and 2^24 hops --------------------------------------------------------------------------
LINK_S = 512 * MIB
LINK_MAX_HOPS = 1 << 24


@pytest.fixture(scope="module")
def link_ctx(cro):
    with cro.ProbeContext(sweep_bytes=LINK_S, devices=[0], read_sweeps=2, copy_sweeps=1) as c:
        yield c


@gpu
def test_host_link_at_the_sweep_size(cro, coracle, link_ctx):
    from test_host_link import CHECK_PATTERN
    nw = LINK_S // 8
    r, faults = link_ctx.probe_host_link(0, bytes=LINK_S)
    assert r.status == cro.OK and r.first_fail == cro.LINK_NO_FAIL and not faults and r.bytes == LINK_S
    want = [coracle.checksum(r.seed[j], 0, nw, threads=16) for j in range(3)]
    for k in range(cro.LINK_WORD_CHECKS):
        c = r.check[k]
        assert (c.words, c.mismatches, c.recorded) == (nw, 0, 0) and c.fold == c.expect == want[CHECK_PATTERN[k]], k
    mask = (1 << 63) | (1 << 17) | 1
    r, faults = link_ctx.probe_host_link(0, bytes=LINK_S, inject=(2, nw - 1, mask))
    (f,) = faults
    e = coracle.pattern_word(r.seed[CHECK_PATTERN[2]], nw - 1)
    assert r.status == cro.ERR_CHECKSUM and r.first_fail == 2
    assert [r.check[k].mismatches for k in range(cro.LINK_WORD_CHECKS)] == [0, 0, 1, 0, 0]
    assert (f.check, f.word_index, f.expected, f.actual, f.host_value) == (2, nw - 1, e, e ^ mask, e ^ mask)


@gpu
def test_host_link_chase_at_its_hop_maximum(cro, coracle, link_ctx):
    m = link_ctx.own_devices()[0].device_minor
    (r, _), t = timed(lambda: link_ctx.probe_host_link(0, bytes=MIB, hops=LINK_MAX_HOPS))
    want = coracle.chase_end(m, m, LINK_MAX_HOPS)
    assert r.status == cro.OK and (r.chase_hops, r.chase_end, r.chase_expect) == (LINK_MAX_HOPS, want, want)
    print("link chase of %d hops: %.1f s, %.0f ns per hop" % (LINK_MAX_HOPS, t, r.chase_ns / LINK_MAX_HOPS))


# ---- 6. the guard: every option maximum in the header has a row above, or a named exemption ---------------------------
# maximum -> the test that runs a probe at it
EDGES = {
    "CRO_COMPUTE_MAX_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_COMPUTE_MAX_ALU_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_PRECISION_MAX_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_PRECISION_MAX_ALU_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_SPARSE_MAX_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_WARPMMA_MAX_ITERATIONS": "test_tensor_probe_clean_at_its_iteration_maxima",
    "CRO_ALU_MAX_ITERATIONS": "test_alu_clean_at_its_iteration_maximum",
    "CRO_BARRIER_MAX_ITERATIONS": "test_barrier_clean_at_its_iteration_maximum",
    "CRO_L2_MAX_ITERATIONS": "test_l2_at_its_iteration_maximum",
    "CRO_L2_MAX_A1_COUNTERS": "test_l2_a1_counter_counts",
    "CRO_L2_MAX_A2_COUNTERS": "test_l2_a2_counter_counts",
    "CRO_L2_MAX_L2_MULTIPLE": "test_l2_buffer_size_ends",
    "CRO_SCAN_MAX_CHUNKS": "test_scan_stops_at_its_chunk_cap",
    "link hops": "test_host_link_chase_at_its_hop_maximum",
    **{"CRO_" + v: "test_64_rounds_under_a_hold" for v in ROUNDS_MAX.values()},
}
# maximum -> why it needs no row here
EXEMPT = {
    "CRO_XLANE_MAX_ITERATIONS": "already run at its maximum (4096) by test_xlane_probe.py",
    "CRO_REGFILE_MAX_ITERATIONS": "already run at its maximum (4096) by test_regfile_probe.py",
    "CRO_SRAM_MAX_ITERATIONS": "already run at its maximum (4096) by test_sram_probe.py",
}
MAXIMUM = re.compile(r"^#define\s+(CRO_\w+_MAX_(?:ALU_)?ITERATIONS|CRO_\w+_MAX_ROUNDS|CRO_L2_MAX_A1_COUNTERS|CRO_L2_MAX_A2_COUNTERS|"
                     r"CRO_L2_MAX_L2_MULTIPLE|CRO_SCAN_MAX_CHUNKS)\b", re.M)
LINK_HOPS = re.compile(r"uint32_t\s+hops;\s*/\*.*at most 2\^(\d+)")


def header_maxima(text):
    """{name: value} of every option maximum the header declares, the link's hop limit (a field comment) included."""
    out = {m.group(1): None for m in MAXIMUM.finditer(text)}
    hops = LINK_HOPS.findall(text)
    assert len(hops) == 1, hops
    out["link hops"] = 1 << int(hops[0])
    return out


def unmatched(text, edges=EDGES, exempt=EXEMPT):
    """Maxima with neither a row nor an exemption, and rows or exemptions naming no maximum."""
    have = set(header_maxima(text))
    named = set(edges) | set(exempt)
    return sorted(have - named), sorted(named - have)


def test_every_option_maximum_has_an_edge_row():
    with open(HEADER) as f:
        text = f.read()
    assert unmatched(text) == ([], [])
    assert not set(EDGES) & set(EXEMPT)
    assert header_maxima(text)["link hops"] == LINK_MAX_HOPS
    here = globals()
    for name, test in EDGES.items():
        fn = here.get(test)
        assert callable(fn) and any(m.name == "gpu" for m in getattr(fn, "pytestmark", [])), (name, test)
    for name, why in EXEMPT.items():
        path = os.path.join(ROOT, "tests", re.search(r"test_\w+\.py", why).group(0))
        with open(path) as f:
            assert "[1, 4096]" in f.read(), (name, path)


def test_the_guard_fails_for_a_new_maximum_or_a_missing_row():
    with open(HEADER) as f:
        text = f.read()
    assert unmatched(text + "\n#define CRO_FOO_MAX_ROUNDS 64\n") == (["CRO_FOO_MAX_ROUNDS"], [])
    assert unmatched(text + "\n#define CRO_FOO_MAX_ALU_ITERATIONS 8\n") == (["CRO_FOO_MAX_ALU_ITERATIONS"], [])
    for name in EDGES:
        fewer = {k: v for k, v in EDGES.items() if k != name}
        assert unmatched(text, edges=fewer) == ([name], []), name
    assert unmatched(text.replace("#define CRO_SCAN_MAX_CHUNKS", "#define CRO_SCAN_CHUNK_LIMIT")) == ([], ["CRO_SCAN_MAX_CHUNKS"])


def test_the_rows_use_the_header_values(cro):
    """The GPU rows take their maxima from the binding; the binding's constants are the header's."""
    with open(HEADER) as f:
        text = f.read()
    for name in header_maxima(text):
        if name.startswith("CRO_"):
            m = re.search(r"^#define\s+%s\s+\(?(\d+)u?(?:\s*<<\s*(\d+))?\)?" % name, text, re.M)
            value = int(m.group(1)) << int(m.group(2) or 0)
            assert getattr(cro, name[4:]) == value, name
