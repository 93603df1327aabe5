"""The device-side verdict on crafted inputs, on one GPU: probe_finalize_kernel and p2p_finalize_kernel byte for byte
against the host restatement (oracle/verdict.py), and chase_kernel against the C oracle's walk of the latency
permutation.  The kernels run through the cro_selftest_* hooks, on buffers of the hooks' own, so every branch of the
verdict is reached here without a fault in the hardware and without a second GPU."""
import random

import pytest

import verdict as V

pytestmark = pytest.mark.gpu

M = V.MASK64
SHAPES = [(0, 1), (1, 1), (2, 3), (3, 2), (29, 1), (30, 30)]      # (copy sweeps, read sweeps)
HOPS = [0, 1, 1024, 65536]


@pytest.fixture(scope="module")
def ctx(cro):
    with cro.ProbeContext(sweep_bytes=1 << 20, devices=[0], flags=cro.F_LAZY_ALLOC) as c:
        yield c


class Mismatches:
    """Collects the cases whose device bytes differ from the restatement; fails with the differing fields."""

    def __init__(self):
        self.cases, self.bad = 0, []

    def check(self, what, got, want):
        self.cases += 1
        if got != want and len(self.bad) < 8:
            self.bad.append("%s: %s" % (what, {k: (hex(a) if isinstance(a, int) else a, hex(b) if isinstance(b, int) else b)
                                               for k, (a, b) in V.diff_fields(got, want).items()}))
        elif got != want:
            self.bad.append(what)

    def done(self):
        print("crafted cases: %d" % self.cases)
        assert not self.bad, "%d of %d cases differ (device, restatement):\n%s" % (len(self.bad), self.cases, "\n".join(self.bad[:8]))


# ---- probe_finalize ---------------------------------------------------------------------------------------------------
def random_times(rng, k):
    """k sweep windows with ties and the odd huge or inverted one."""
    out = []
    for _ in range(k):
        t0 = rng.randrange(1 << 40)
        d = rng.choice([1000, 1000, 2500, 7, 0, 1 << 33, rng.randrange(1 << 20)])
        out.append((t0, (t0 + d) & M if rng.random() > 0.05 else rng.randrange(t0 + 1)))
    return out


def finalize_state(rng, C, R, fused):
    """A probe that passed: every slot it checks carries the nonce, the word count and (where it folds) the closed form;
    every slot it does not read holds garbage."""
    nonce = rng.choice([rng.randrange(1 << 32), rng.randrange(1 << 64)])
    S = 8 * rng.randrange(1, 1 << 40)
    E = tuple(rng.randrange(1 << 64) for _ in range(3))
    sl = [V.Slot(*(rng.randrange(1 << 64) for _ in range(8))) for _ in range(V.SLOT_COUNT)]
    times = random_times(rng, 2 + C + R)
    sl[V.SLOT_FILL] = V.Slot(0, 0, 0, *times[0], nonce, S // 8)
    sl[V.SLOT_EXPECT] = V.Slot(*E, *times[1], nonce, S // 8)
    for i in range(C):
        sl[V.SLOT_SWEEP0 + i] = V.Slot(*(E if fused else (0, 0, 0)), *times[2 + i], nonce, S // 8)
    for i in range(R):
        sl[V.SLOT_SWEEP0 + C + i] = V.Slot(*E, *times[2 + C + i], nonce, S // 8)
    tmpl = bytes(rng.randrange(256) for _ in range(512))
    return dict(tmpl=tmpl, slots=sl, seed=rng.randrange(1 << 64), nonce=nonce, sweep_bytes=S, read_sweeps=R, copy_sweeps=C,
                read_variant=rng.choice([1, 2, 3]), copy_variant=3 if fused else rng.choice([1, 2]))


PERTURB = {
    "stamp-1": lambda s, st: s._replace(stamp=(s.stamp - 1) & M),
    "stamp^2^32": lambda s, st: s._replace(stamp=s.stamp ^ (1 << 32)),          # the whole 64-bit stamp is compared
    "n_words+1": lambda s, st: s._replace(n_words=(s.n_words + 1) & M),
    "n_words-1": lambda s, st: s._replace(n_words=(s.n_words - 1) & M),
    "x": lambda s, st: s._replace(x=s.x ^ 1),
    "s": lambda s, st: s._replace(s=(s.s + (1 << 63)) & M),
    "w": lambda s, st: s._replace(w=(s.w + 2) & M),
    "armed": lambda s, st: V.ARMED,                                              # the kernel never ran
}


def run_finalize(ctx, st, mm, what):
    got = ctx.selftest_probe_finalize(0, st["tmpl"], V.pack_slots(st["slots"]), st["seed"], st["nonce"], st["sweep_bytes"],
                                      st["read_sweeps"], st["copy_sweeps"], st["read_variant"], st["copy_variant"])
    want = V.probe_finalize(**st)
    mm.check(what, got, want)
    return V.Result(want)


@pytest.mark.parametrize("fused", [True, False], ids=["checksumming-copy", "plain-copy"])
@pytest.mark.parametrize("C,R", SHAPES)
def test_probe_finalize_every_single_fault(ctx, C, R, fused):
    """Every slot the verdict reads, perturbed one way at a time: the device's 512 bytes equal the restatement's."""
    rng = random.Random(1000 * C + 10 * R + fused)
    base = finalize_state(rng, C, R, fused)
    mm = Mismatches()
    assert run_finalize(ctx, base, mm, "healthy").get("status") == 0
    positions = [V.SLOT_FILL, V.SLOT_EXPECT] + [V.SLOT_SWEEP0 + i for i in range(C + R)]
    codes = set()
    for p in positions:
        for name, f in PERTURB.items():
            st = dict(base, slots=list(base["slots"]))
            st["slots"][p] = f(st["slots"][p], st)
            codes.add(run_finalize(ctx, st, mm, "slot %d %s" % (p, name)).get("fail_code"))
    # a slot the verdict does not read changes nothing
    for p in [V.SLOT_SWEEP0 + C + R][:int(V.SLOT_SWEEP0 + C + R < V.SLOT_EXPECT)] + [V.SLOT_PREFIX, V.SLOT_P2P0]:
        st = dict(base, slots=list(base["slots"]))
        st["slots"][p] = V.ARMED
        assert run_finalize(ctx, st, mm, "unread slot %d" % p).get("status") == 0
    mm.done()
    assert mm.cases >= 1 + len(positions) * len(PERTURB)
    want = {V.FAIL_EXPECT, V.FAIL_STALE, V.FAIL_READ} | ({V.FAIL_COPY_SRC} if fused and C else set())
    assert want <= codes, codes


def test_probe_finalize_random_multi_fault_states(ctx):
    """Seeded random states: any shape, any variants, one to four faults at once."""
    rng = random.Random(20261015)
    mm = Mismatches()
    seen = set()
    for k in range(400):
        C, R = rng.randrange(V.MAX_SWEEPS_EACH + 1), rng.randrange(1, V.MAX_SWEEPS_EACH + 1)
        st = finalize_state(rng, C, R, rng.random() < 0.6)
        st["slots"] = list(st["slots"])
        readable = [V.SLOT_FILL, V.SLOT_EXPECT] + [V.SLOT_SWEEP0 + i for i in range(C + R)]
        for _ in range(rng.randrange(0, 5)):
            p = rng.choice(readable)
            st["slots"][p] = rng.choice(list(PERTURB.values()))(st["slots"][p], st)
        r = run_finalize(ctx, st, mm, "random state %d (C=%d R=%d cv=%d)" % (k, C, R, st["copy_variant"]))
        seen.add((r.get("fail_code"), r.get("copy_verified") > 0))
    mm.done()
    assert mm.cases == 400 and len(seen) >= 6, seen


def test_probe_finalize_rejects_more_sweeps_than_slots(cro, ctx):
    st = finalize_state(random.Random(3), 1, 1, True)
    with pytest.raises(cro.ProbeError) as e:
        ctx.selftest_probe_finalize(0, st["tmpl"], V.pack_slots(st["slots"]), 1, 1, 8, V.MAX_SWEEPS_EACH + 1, 1, 1, 3)
    assert e.value.code == cro.ERR_INVALID_ARG


# ---- p2p_finalize -----------------------------------------------------------------------------------------------------
def p2p_state(rng, n, self_index, have_push, push_folded, hops, hbm_failed, sparse=True):
    """A healthy NVLink state; `sparse` drops the odd peer's access or slot array."""
    PB = 8 * rng.randrange(1, 1 << 30)
    stamp = rng.randrange(1 << 64)
    res = V.Result(bytes(rng.randrange(256) for _ in range(512)))
    res.set("status", V.ERR_CHECKSUM if hbm_failed else 0)
    res.set("fail_code", V.FAIL_READ if hbm_failed else 0)
    res.set("fail_index", 2 if hbm_failed else 0)
    keep = (self_index + 1) % n                               # always checked, so every state has a peer to fail
    access = [0 if j == self_index else int(not sparse or j == keep or rng.random() < 0.85) for j in range(8)]
    res.set("p2p_access", access)
    garbage = lambda: V.Slot(*(rng.randrange(1 << 64) for _ in range(8)))  # noqa: E731
    mine = [garbage() for _ in range(V.SLOT_COUNT)]
    mine_prefix = tuple(rng.randrange(1 << 64) for _ in range(3))
    mine[V.SLOT_PREFIX] = V.Slot(*mine_prefix, 0, 5, stamp, PB // 8)
    peers, stamps = [None] * V.MAX_DEVICES, [rng.randrange(1 << 64) for _ in range(V.MAX_DEVICES)]
    chase, expect = [M] * (2 * V.MAX_DEVICES), [rng.randrange(65536) for _ in range(V.MAX_DEVICES)]
    for j in range(n):
        if j == self_index or (sparse and j != keep and rng.random() < 0.1):
            continue                                          # self, and the odd absent peer
        fold = tuple(rng.randrange(1 << 64) for _ in range(3))
        ps = [garbage() for _ in range(V.SLOT_COUNT)]
        ps[V.SLOT_PREFIX] = V.Slot(*fold, 0, 5, stamps[j], PB // 8)
        peers[j] = ps
        t = random_times(rng, 3)
        mine[V.SLOT_P2P0 + 3 * j] = V.Slot(*fold, *t[0], stamp, PB // 8)
        mine[V.SLOT_P2P0 + 3 * j + 1] = V.Slot(*(mine_prefix if push_folded else (0, 0, 0)), *t[1], stamp, PB // 8)
        mine[V.SLOT_P2P0 + 3 * j + 2] = V.Slot(*fold, *t[2], stamp, PB // 8)
        chase[2 * j], chase[2 * j + 1] = expect[j], rng.choice([hops * 700, rng.randrange(1 << 40), 0])
    return dict(result=res.bytes(), slots=mine, peer_slots=peers, peer_stamp=stamps, chase_out=chase, chase_expect=expect,
                n=n, self_index=self_index, hops=hops, have_push=have_push, push_folded=push_folded, p2p_bytes=PB, stamp=stamp)


def run_p2p(ctx, st, mm, what):
    got = ctx.selftest_p2p_finalize(0, st["result"], V.pack_slots(st["slots"]),
                                    [V.pack_slots(p) if p is not None else None for p in st["peer_slots"]],
                                    st["peer_stamp"], st["chase_out"], st["chase_expect"], st["n"], st["self_index"], st["hops"],
                                    int(st["have_push"]), int(st["push_folded"]), st["p2p_bytes"], st["stamp"])
    want = V.p2p_finalize(**st)
    mm.check(what, got, want)
    return V.Result(want)


def _mine(st, k, j, f):
    st["slots"][V.SLOT_P2P0 + 3 * j + k] = f(st["slots"][V.SLOT_P2P0 + 3 * j + k])


def _prefix(st, j, f):
    if st["peer_slots"][j] is not None:
        st["peer_slots"][j] = list(st["peer_slots"][j])
        st["peer_slots"][j][V.SLOT_PREFIX] = f(st["peer_slots"][j][V.SLOT_PREFIX])


def _chase(st, j, end=None, ns=None):
    if end is not None:
        st["chase_out"][2 * j] = end
    if ns is not None:
        st["chase_out"][2 * j + 1] = ns


PEER_FAULTS = {
    "read stale": lambda st, j: _mine(st, 0, j, lambda s: s._replace(stamp=s.stamp ^ 1)),
    "read off": lambda st, j: _mine(st, 0, j, lambda s: s._replace(w=s.w ^ (1 << 40))),
    "prefix stale": lambda st, j: _prefix(st, j, lambda s: s._replace(stamp=(s.stamp + 1) & M)),
    "prefix short": lambda st, j: _prefix(st, j, lambda s: s._replace(n_words=s.n_words - 1)),
    "push stale": lambda st, j: _mine(st, 1, j, lambda s: V.ARMED),
    "push off": lambda st, j: _mine(st, 1, j, lambda s: s._replace(x=s.x ^ 4)),
    "re-read stale": lambda st, j: _mine(st, 2, j, lambda s: s._replace(stamp=0)),
    "re-read off": lambda st, j: _mine(st, 2, j, lambda s: s._replace(s=(s.s + 1) & M)),
    "chase end wrong": lambda st, j: _chase(st, j, end=st["chase_out"][2 * j] ^ 1),
    "chase not run": lambda st, j: _chase(st, j, end=M, ns=M),
    "chase ns saturates": lambda st, j: _chase(st, j, ns=(1 << 60) + 12345),
    "chase ns at the edge": lambda st, j: _chase(st, j, ns=(0xFFFFFFFF * max(st["hops"], 1)) // 16 + 1),
}


@pytest.mark.parametrize("n", [2, 3, 8, 9, 16])
def test_p2p_finalize_every_fault_of_every_peer(ctx, n):
    mm = Mismatches()
    codes = set()
    for self_index in sorted({0, n // 2, n - 1}):
        for k, (have_push, push_folded) in enumerate([(1, 1), (1, 0), (0, 1), (0, 0)]):
            hops = HOPS[(k + self_index) % 4]
            for hbm_failed in (False, True):
                rng = random.Random(hash((n, self_index, k, hbm_failed)) & 0xFFFFFFFF)
                base = p2p_state(rng, n, self_index, have_push, push_folded, hops, hbm_failed)
                tag = "n=%d self=%d push=%d/%d hops=%d hbm_failed=%d" % (n, self_index, have_push, push_folded, hops, hbm_failed)
                r = run_p2p(ctx, base, mm, tag + " healthy")
                assert r.get("status") == (V.ERR_CHECKSUM if hbm_failed else 0)
                peers = range(n) if not hbm_failed else [j for j in range(n) if j != self_index][:2]
                for j in peers:
                    for name, f in PEER_FAULTS.items():
                        st = dict(base, slots=list(base["slots"]), peer_slots=list(base["peer_slots"]),
                                  chase_out=list(base["chase_out"]))
                        f(st, j)
                        codes.add(run_p2p(ctx, st, mm, "%s peer %d %s" % (tag, j, name)).get("fail_code"))
    mm.done()
    assert {V.FAIL_EXPECT, V.FAIL_P2P_READ, V.FAIL_P2P_PUSH, V.FAIL_P2P_CHASE, V.FAIL_READ} <= codes, codes


def test_an_unrun_chase_fails_at_every_hop_count(ctx):
    """The armed chase output is no legal end: at 65536 hops (a whole Sattolo cycle, which ends on slot 0) too."""
    mm = Mismatches()
    for hops in (1, 1024, 65535, 65536, 131072):
        st = p2p_state(random.Random(hops), 2, 0, 1, 1, hops, False, sparse=False)
        end = 0 if hops % 65536 == 0 else st["chase_expect"][1]       # a whole number of cycles ends on slot 0
        st["chase_expect"][1] = end
        _chase(st, 1, end=end)
        assert V.Result(V.p2p_finalize(**st)).get("p2p_ok") == 0b10
        _chase(st, 1, end=M, ns=M)
        r = run_p2p(ctx, st, mm, "hops=%d" % hops)
        assert (r.get("fail_code"), r.get("fail_index"), r.get("p2p_ok")) == (V.FAIL_P2P_CHASE, 1, 0), hops
    mm.done()


# ---- chase_kernel -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hops", [1, 2, 65535, 65536, 65537, 1 << 20])
def test_chase_kernel_ends_where_the_oracle_walk_ends(cro, coracle, ctx, hops):
    one = [(0, 1)]
    sixteen = [None if j % 5 == 2 else (j % 8, (j + 3) % 8) for j in range(16)]
    assert V.ARMED.x >= 65536                                  # the armed word is no legal end
    for pairs in (one, sixteen):
        out = ctx.selftest_chase(0, pairs, hops)
        assert len(out) == 2 * len(pairs)
        for j, p in enumerate(pairs):
            if p is None:
                assert out[2 * j] == out[2 * j + 1] == M, (j, out[2 * j], out[2 * j + 1])   # untouched: still armed
            else:
                want = coracle.chase_end(p[0], p[1], hops)
                assert out[2 * j] == want == cro.chase_end(p[0], p[1], hops), (p, hops, out[2 * j], want)
                assert 0 < out[2 * j + 1] < 10 ** 10, (p, hops, out[2 * j + 1])             # a measured time, not the armed value
