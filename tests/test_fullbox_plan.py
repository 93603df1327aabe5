"""The full-box probe's schedule (cro_probe_all) against a restatement, on the CPU: the plan the library walks
(cro_selftest_p2p_plan) equals oracle/fullbox.py field by field; its event graph orders every leg after what it
depends on; and the slots a healthy box would hold under it pass oracle/verdict.py's p2p_finalize, while each
corrupted leg fails naming that leg and that peer.  On one GPU the same slots go through the device's p2p_finalize.

The NVLink phase needs two or more GPUs to run, so this is where its host decisions are tested: unequal sweep sizes
(one prefix per call), odd device counts (every device records its round events, byes included) and one-way peer
access (such a pair is neither scheduled nor checked)."""
import ctypes
import functools
import itertools
import random

import pytest

import fullbox as FB
import verdict as V

M = V.MASK64
MiB = 1 << 20
HOPS = 1024


# ---- inputs -------------------------------------------------------------------------------------------------------------
def full_access(n):
    """Every device reaches every other it has a p2p_access column for (columns 0..7, as the template holds them)."""
    return [[int(j != i and j < n) for j in range(8)] for i in range(n)]


def one_way(n, a, b):
    """a reaches b, b does not reach a."""
    acc = full_access(n)
    if b < len(acc) and a < 8:
        acc[b][a] = 0
    return acc


def missing_pair(n, a, b):
    acc = full_access(n)
    if a < n and b < n:
        acc[a][b] = acc[b][a] = 0
    return acc


def random_access(n, rng, p=0.8):
    return [[int(j != i and j < n and rng.random() < p) for j in range(8)] for i in range(n)]


def sizes_equal(n, S=4 * MiB):
    return [S] * n


def sizes_one_halved(n, S=4 * MiB):
    return [S // 2 if i == n // 2 else S for i in range(n)]


def sizes_all_different(n, S=4 * MiB):
    return [S - 16 * 4096 * i for i in range(n)]


FLAG_SETS = [dict(flags=f, unidir=u, write_variant=w) for f, u, w in
             itertools.product([0, FB.F_SKIP_P2P_WRITE], [False, True], [FB.COPY_TMA_FUSED, 1])]


def p_values(sizes):
    """p2p_bytes below, at and above the smallest S (p2p_bytes never exceeds the options' S)."""
    lo = min(sizes) if sizes else 4 * MiB
    return [lo // 4, lo, 4 * MiB]


def library_plan(cro, sizes, P, access, flags=0, unidir=False, write_variant=FB.COPY_TMA_FUSED):
    cp = cro.selftest_p2p_plan(sizes, P, access, flags, unidir, write_variant)
    rounds = [[(cp.pair[r][2 * k], cp.pair[r][2 * k + 1]) for k in range(cp.n_pairs[r])] for r in range(cp.n_rounds)]
    ops = [FB.Op(o.kind, o.dev, o.peer, o.event, o.round, o.slot, o.bytes) for o in cp.op[:cp.n_ops]]
    fin = [FB.Fin(f.n, f.self, f.have_push, f.push_folded, f.p2p_bytes, f.peer_mask, f.chase_mask) for f in cp.fin]
    return FB.Plan(cp.p2p_bytes, rounds, ops, fin)


def assert_same_plan(got, want, what):
    assert got.p2p_bytes == want.p2p_bytes, (what, "p2p_bytes", got.p2p_bytes, want.p2p_bytes)
    assert got.rounds == want.rounds, (what, "rounds")
    for k, (g, w) in enumerate(zip(got.ops, want.ops)):
        assert g == w, (what, "op %d" % k, g, w)
    assert len(got.ops) == len(want.ops), (what, "op count", len(got.ops), len(want.ops))
    for i, (g, w) in enumerate(zip(got.fin, want.fin)):
        assert g == w, (what, "finalize of device %d" % i, g, w)


def cases_for(n):
    """Sampled access matrices x size sets x prefix lengths, the option flags rotating over the cases."""
    accesses = [("full", full_access(n)), ("one-way 0->1", one_way(n, 0, 1)), ("one-way 2->0", one_way(n, 2, 0)),
                ("missing 0-1", missing_pair(n, 0, 1)), ("random", random_access(n, random.Random(n)))]
    sizes = [("equal", sizes_equal(n)), ("one halved", sizes_one_halved(n)), ("all different", sizes_all_different(n))]
    k = 0
    for (an, acc), (sn, sz) in itertools.product(accesses, sizes):
        for P in p_values(sz):
            fl = FLAG_SETS[k % len(FLAG_SETS)]
            k += 1
            yield "n=%d %s %s P=%d %s" % (n, an, sn, P, fl), sz, P, acc, fl
    for fl in FLAG_SETS + [dict(flags=FB.F_SKIP_P2P, unidir=False, write_variant=FB.COPY_TMA_FUSED)]:
        yield "n=%d full equal %s" % (n, fl), sizes_equal(n), 4 * MiB, full_access(n), fl


def seeded_cases(count, seed=20261018):
    rng = random.Random(seed)
    for k in range(count):
        n = rng.randrange(0, 17)
        base = 16 * rng.randrange(1 << 10, 1 << 18)
        sz = [base if rng.random() < 0.5 else 16 * rng.randrange(1 << 10, 1 << 18) for _ in range(n)]
        P = 16 * rng.randrange(1, 1 << 18)
        acc = random_access(n, rng, rng.choice([1.0, 0.9, 0.6]))
        fl = dict(flags=rng.choice([0, 0, FB.F_SKIP_P2P_WRITE, FB.F_SKIP_P2P]), unidir=rng.random() < 0.2,
                  write_variant=rng.choice([1, 2, 3, 3]))
        yield "seeded case %d n=%d" % (k, n), sz, P, acc, fl


# ---- properties -------------------------------------------------------------------------------------------------------
def violations(p, access, unidir=False, push=True):
    """Every way plan p breaks the schedule's ordering and coverage rules, as short strings."""
    ops, out = p.ops, []
    n = len([i for i in range(FB.MAX_DEVICES) if any(o.dev == i for o in ops)])
    g = FB.Graph(ops)
    out += ["unbound wait at op %d %s" % (k, ops[k]) for k in g.unbound]
    if p.p2p_bytes == 0:
        return out
    legs = {(o.kind, o.dev, o.peer, o.round): k for k, o in enumerate(ops) if o.kind in FB.LEGS}
    # every reachable unordered pair meets once in each direction (one direction under unidir)
    for a in range(n):
        for b in range(n):
            if a == b:
                continue
            reads = [k for (kind, d, q, _), k in legs.items() if kind == FB.OP_READ and (d, q) == (a, b)]
            pushes = [k for (kind, d, q, _), k in legs.items() if kind == FB.OP_PUSH and (d, q) == (a, b)]
            want = int(FB.linked(access, a, b))
            if unidir and want:
                want = int(any((a, b) in rd for rd in p.rounds))
            if len(reads) != want or len(pushes) != (want if push else 0):
                out.append("pair %d->%d: %d reads, %d pushes, want %d" % (a, b, len(reads), len(pushes), want))
    # no device is in two pairs in a round
    for r, rd in enumerate(p.rounds):
        seen = [x for pr in rd for x in pr]
        if len(seen) != len(set(seen)):
            out.append("round %d: a device in two pairs %s" % (r, rd))
    hbm = {o.dev: k for k, o in enumerate(ops) if o.kind == FB.OP_HBM}
    prefix = {o.dev: k for k, o in enumerate(ops) if o.kind == FB.OP_PREFIX}
    for (kind, d, q, r), k in legs.items():
        if kind == FB.OP_PUSH:
            # into q's half B: after q's own HBM probe and after every earlier re-read of q's half B
            deps = [hbm[q]] + [j for (kk, dd, _, rr), j in legs.items() if kk == FB.OP_REREAD and dd == q and rr < r]
            out += ["push %d->%d round %d not after op %d %s" % (d, q, r, j, ops[j]) for j in deps
                    if not g.happens_before(j, k)]
        if kind == FB.OP_READ:
            out += ["read %d<-%d round %d not after op %d %s" % (d, q, r, j, ops[j]) for j in (hbm[q], prefix[q])
                    if not g.happens_before(j, k)]
        if kind == FB.OP_REREAD:
            j = legs.get((FB.OP_PUSH, q, d, r))
            if j is None or not g.happens_before(j, k):
                out.append("re-read on %d of %d's push round %d not after that push" % (d, q, r))
    for k, o in enumerate(ops):
        if o.kind == FB.OP_CHASE:
            out += ["chase on %d not after leg %s" % (o.dev, ops[j]) for j in legs.values() if not g.happens_before(j, k)]
        if o.kind == FB.OP_FINALIZE:
            f = p.fin[o.dev]
            peers = [j for j in range(n) if f.peer_mask >> j & 1]
            deps = [prefix[o.dev]] + [prefix[j] for j in peers]
            deps += [x for (kind, d, q, _), x in legs.items() if d == o.dev and q in peers]
            deps += [x for x, oo in enumerate(ops) if oo.kind == FB.OP_CHASE and oo.dev == o.dev]
            out += ["finalize on %d not after %s" % (o.dev, ops[j]) for j in deps if not g.happens_before(j, k)]
    return out


# ---- the plan equals the restatement ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", range(17))
def test_plan_equals_restatement(cro, n):
    count = 0
    for what, sz, P, acc, fl in cases_for(n):
        assert_same_plan(library_plan(cro, sz, P, acc, **fl), FB.plan(sz, P, acc, **fl), what)
        count += 1
    assert count >= 45


def test_plan_equals_restatement_seeded_sweep(cro):
    count = 0
    for what, sz, P, acc, fl in seeded_cases(600):
        assert_same_plan(library_plan(cro, sz, P, acc, **fl), FB.plan(sz, P, acc, **fl), what)
        count += 1
    assert count >= 500


def test_plan_hook_refuses_null_and_out_of_range(cro):
    lib, plan = cro.lib, cro.P2PPlan()
    S = (ctypes.c_uint64 * 17)(*[MiB] * 17)
    A = (ctypes.c_uint8 * (8 * 17))()
    assert lib.cro_selftest_p2p_plan(17, S, MiB, A, 0, 0, 3, ctypes.byref(plan)) == cro.ERR_INVALID_ARG
    assert lib.cro_selftest_p2p_plan(2, None, MiB, A, 0, 0, 3, ctypes.byref(plan)) == cro.ERR_INVALID_ARG
    assert lib.cro_selftest_p2p_plan(2, S, MiB, None, 0, 0, 3, ctypes.byref(plan)) == cro.ERR_INVALID_ARG
    assert lib.cro_selftest_p2p_plan(2, S, MiB, A, 0, 0, 3, None) == cro.ERR_INVALID_ARG
    assert lib.cro_selftest_p2p_plan(16, S, MiB, A, 0, 0, 3, ctypes.byref(plan)) == cro.OK
    assert lib.cro_selftest_p2p_plan(0, S, MiB, A, 0, 0, 3, ctypes.byref(plan)) == cro.OK and plan.n_ops == 0


# ---- what the fixes change, stated on the plan --------------------------------------------------------------------------
def test_unequal_sizes_move_one_prefix_everywhere(cro):
    sz = [4 * MiB, 2 * MiB, 4 * MiB, 3 * MiB]
    p = library_plan(cro, sz, 4 * MiB, full_access(4))
    assert p.p2p_bytes == 2 * MiB
    moved = {o.bytes for o in p.ops if o.kind in FB.LEGS + (FB.OP_PREFIX,)}
    assert moved == {2 * MiB}
    assert {f.p2p_bytes for f in p.fin[:4]} == {2 * MiB}


@pytest.mark.parametrize("n", [3, 5, 7, 15])
def test_odd_counts_record_every_round_event_on_every_device(cro, n):
    p = library_plan(cro, sizes_equal(n), MiB, full_access(n))
    for r in range(len(p.rounds)):
        for ev in (FB.EV_PUSH, FB.EV_REREAD):
            assert sorted(o.dev for o in p.ops if o.kind == FB.OP_RECORD and o.event == ev and o.round == r) == list(range(n))
    assert FB.Graph(p.ops).unbound == []


def test_one_way_access_is_neither_scheduled_nor_checked(cro):
    acc = one_way(4, 0, 1)                  # 0 reaches 1, 1 does not reach 0
    p = library_plan(cro, sizes_equal(4), MiB, acc)
    assert not [o for o in p.ops if o.kind in FB.LEGS and {o.dev, o.peer} == {0, 1}]
    assert not p.fin[0].peer_mask & 2 and not p.fin[1].peer_mask & 1
    assert not p.fin[0].chase_mask & 2 and not p.fin[1].chase_mask & 1
    assert p.fin[0].peer_mask == 0b1100 and p.fin[1].peer_mask == 0b1100


# ---- properties on the plan --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", range(17))
def test_plan_orders_every_leg(cro, n):
    for what, sz, P, acc, fl in itertools.islice(cases_for(n), 0, None, 4):
        p = library_plan(cro, sz, P, acc, **fl)
        bad = violations(p, acc, fl["unidir"], not fl["flags"] & FB.F_SKIP_P2P_WRITE)
        assert not bad, (what, bad[:5])


def test_plan_orders_every_leg_seeded(cro):
    for what, sz, P, acc, fl in seeded_cases(120, seed=7):
        p = library_plan(cro, sz, P, acc, **fl)
        bad = violations(p, acc, fl["unidir"], not fl["flags"] & FB.F_SKIP_P2P_WRITE)
        assert not bad, (what, bad[:5])


def _drop(p, pred):
    return p._replace(ops=[o for o in p.ops if not pred(o)])


def _hand_built():
    """One broken plan per property: the property check must name it."""
    acc4, acc3 = full_access(4), full_access(3)
    p4, p3 = FB.plan(sizes_equal(4), MiB, acc4), FB.plan(sizes_equal(3), MiB, acc3)
    first_read = next(o for o in p4.ops if o.kind == FB.OP_READ)
    late_prefix = [o for o in p4.ops if not (o.kind == FB.OP_PREFIX and o.dev == 1)] + [
        next(o for o in p4.ops if o.kind == FB.OP_PREFIX and o.dev == 1)]
    # the bye's re-read event not recorded: what recording it only for receivers does at an odd count
    byes = {(r, i) for r, rd in enumerate(p3.rounds) for i in range(3) if all(i not in pr for pr in rd)}
    return {
        "a pair meets once in each direction": (_drop(p4, lambda o: o == first_read), acc4, "reads"),
        "no device in two pairs": (p4._replace(rounds=[[(0, 1), (1, 2)]] + p4.rounds[1:]), acc4, "two pairs"),
        "push after the receiver's previous re-read": (
            _drop(p3, lambda o: o.kind == FB.OP_RECORD and o.event == FB.EV_REREAD and (o.round, o.dev) in byes), acc3, "push"),
        "read after the peer's HBM phase": (_drop(p4, lambda o: o.kind == FB.OP_WAIT and o.event == FB.EV_HBM), acc4, "read"),
        "re-read after the push": (_drop(p4, lambda o: o.kind == FB.OP_WAIT and o.event == FB.EV_PUSH), acc4, "re-read"),
        "chase after every leg": (_drop(p4, lambda o: o.kind == FB.OP_WAIT and o.event == FB.EV_CHASE), acc4, "chase"),
        "finalize after every slot it reads": (p4._replace(ops=late_prefix), acc4, "finalize"),
    }


@pytest.mark.parametrize("prop", list(_hand_built()))
def test_each_property_catches_its_hand_built_break(prop):
    p, acc, word = _hand_built()[prop]
    bad = violations(p, acc)
    assert any(word in b for b in bad), (prop, bad[:5])
    assert not violations(FB.plan([MiB] * len(acc), MiB, acc), acc)


# ---- the healthy box ---------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _fold(coracle, seed, words):
    return coracle.checksum(seed, 0, words)


def healthy_box(coracle, p, n, rng):
    seeds = [rng.randrange(1 << 64) for _ in range(n)]
    nonces = [rng.randrange(1 << 64) for _ in range(n)]
    chase_expect = [[rng.randrange(65536) for _ in range(n)] for _ in range(n)]
    slots, chase = FB.healthy_slots(p, seeds, nonces, lambda s, w: _fold(coracle, s, w), chase_expect)
    res = V.Result(bytes(rng.randrange(256) for _ in range(512)))
    for k, v in (("status", 0), ("fail_code", 0), ("fail_index", 0)):
        res.set(k, v)
    return slots, chase, chase_expect, nonces, res.bytes()


def corruptions(p, i, inputs):
    """(name, leg, peer, inputs with that one leg of that peer corrupted) for every leg device i's verdict checks."""
    f = p.fin[i]
    for j in range(f.n):
        if not f.peer_mask >> j & 1:
            continue
        legs = [(FB.OP_READ, 0), (FB.OP_PREFIX, None), (FB.OP_CHASE, None)]
        if f.have_push:
            legs += [(FB.OP_REREAD, 2)] + ([(FB.OP_PUSH, 1)] if f.push_folded else [])
        for leg, k in legs:
            st = dict(inputs, slots=list(inputs["slots"]), peer_slots=list(inputs["peer_slots"]),
                      chase_out=list(inputs["chase_out"]))
            if k is not None:
                s = st["slots"][V.SLOT_P2P0 + 3 * j + k]
                st["slots"][V.SLOT_P2P0 + 3 * j + k] = s._replace(w=s.w ^ (1 << 17))
            elif leg == FB.OP_PREFIX:
                st["peer_slots"][j] = list(st["peer_slots"][j])
                s = st["peer_slots"][j][V.SLOT_PREFIX]
                st["peer_slots"][j][V.SLOT_PREFIX] = s._replace(n_words=s.n_words - 1)
            else:
                st["chase_out"][2 * j] ^= 1
            yield leg, j, st


HEALTHY = [(n, sn, sz(n), an, acc(n), fl) for n in (2, 3, 4, 5, 8, 9)
           for (sn, sz), (an, acc), fl in zip(
               itertools.cycle([("equal", sizes_equal), ("one halved", sizes_one_halved), ("all different", sizes_all_different)]),
               [("full", full_access), ("one-way", lambda n: one_way(n, 0, n - 1)), ("missing", lambda n: missing_pair(n, 1, 2)),
                ("full", full_access)],
               [FLAG_SETS[0], FLAG_SETS[0], FLAG_SETS[4], FLAG_SETS[1]])]


@pytest.mark.parametrize("n,sn,sizes,an,access,fl", HEALTHY,
                         ids=["n=%d-%s-%s-%s" % (h[0], h[1], h[3], "".join("%s" % int(v) for v in h[5].values())) for h in HEALTHY])
def test_healthy_box_passes_and_each_corrupted_leg_is_named(cro, coracle, n, sn, sizes, an, access, fl):
    P = 4 * MiB
    p = library_plan(cro, sizes, P, access, **fl)
    assert p.p2p_bytes == min(sizes)
    rng = random.Random(n * 1000 + len(an))
    slots, chase, expect, nonces, res = healthy_box(coracle, p, n, rng)
    for i in range(n):
        inputs = FB.finalize_inputs(p, i, slots, chase, expect, nonces, access, HOPS, res)
        r = V.Result(V.p2p_finalize(**inputs))
        assert (r.get("status"), r.get("fail_code")) == (V.OK, V.FAIL_NONE), (i, r.get("fail_code"), r.get("fail_index"))
        assert r.get("p2p_ok") == p.fin[i].peer_mask & 0xFF and r.get("p2p_bytes") == min(sizes)
        for leg, j, st in corruptions(p, i, inputs):
            r = V.Result(V.p2p_finalize(**st))
            assert (r.get("status"), r.get("fail_code"), r.get("fail_index")) == (
                V.ERR_CHECKSUM, FB.expected_fail(leg, p.fin[i].push_folded), j), (i, leg, j)
            assert r.get("p2p_ok") == p.fin[i].peer_mask & ~(1 << j) & 0xFF


def test_a_one_way_peer_stays_unchecked_and_shows_why(cro, coracle):
    acc = one_way(3, 0, 2)                  # 0 reaches 2, 2 does not reach 0
    p = library_plan(cro, sizes_equal(3), MiB, acc)
    slots, chase, expect, nonces, res = healthy_box(coracle, p, 3, random.Random(5))
    for i, (ok, access) in enumerate([(0b010, [0, 1, 1]), (0b101, [1, 0, 1]), (0b010, [0, 1, 0])]):
        r = V.Result(V.p2p_finalize(**FB.finalize_inputs(p, i, slots, chase, expect, nonces, acc, HOPS, res)))
        assert r.get("status") == V.OK and r.get("p2p_ok") == ok and r.get("p2p_access")[:3] == access, i


# ---- on one GPU: the device's verdict on the healthy box ----------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as c:
        yield c


def _device(ctx, st):
    return ctx.selftest_p2p_finalize(0, st["result"], V.pack_slots(st["slots"]),
                                     [V.pack_slots(q) if q is not None else None for q in st["peer_slots"]],
                                     st["peer_stamp"], st["chase_out"], st["chase_expect"], st["n"], st["self_index"], st["hops"],
                                     int(st["have_push"]), int(st["push_folded"]), st["p2p_bytes"], st["stamp"])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_device_verdict_on_the_healthy_box(cro, coracle, ctx, n):
    cases = 0
    for sizes, acc, fl in [(sizes_all_different(n), full_access(n), FLAG_SETS[0]),
                           (sizes_one_halved(n), one_way(n, 0, n - 1), FLAG_SETS[2])]:
        p = library_plan(cro, sizes, 4 * MiB, acc, **fl)
        slots, chase, expect, nonces, res = healthy_box(coracle, p, n, random.Random(n))
        for i in range(n):
            inputs = FB.finalize_inputs(p, i, slots, chase, expect, nonces, acc, HOPS, res)
            want = V.p2p_finalize(**inputs)
            assert V.Result(want).get("status") == V.OK
            got = _device(ctx, inputs)
            assert got == want, (n, i, V.diff_fields(got, want))
            for leg, j, st in corruptions(p, i, inputs):
                want = V.p2p_finalize(**st)
                got = _device(ctx, st)
                assert got == want, (n, i, leg, j, V.diff_fields(got, want))
                assert (V.Result(got).get("fail_code"), V.Result(got).get("fail_index")) == (
                    FB.expected_fail(leg, p.fin[i].push_folded), j)
                cases += 1
    assert cases >= 4 * n
